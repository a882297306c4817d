// Roofline denominators of the SpMM gather: random row gathers (256 B and 512 B rows, as prop_kernel issues them:
// one float4 per lane, 8 rows in flight per group) from tables that fit the L2 (16 .. 96 MB) and that do not
// (384 MB .. 6 GB).  Prints one JSON object per (row bytes, table size): GB/s of gathered bytes.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/gather_bench tools/gather_bench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

template <int G>   // lanes per row: 16 -> 256 B rows, 32 -> 512 B rows
__global__ void __launch_bounds__(256, 4) gather_kernel(const float4 *__restrict__ table, const int32_t *__restrict__ idx, int64_t n_gather,
                                                         float *__restrict__ sink) {
    constexpr int RPW = 32 / G, UNR = 8;
    const int lane = threadIdx.x & 31, gl = lane % G, grp = lane / G;
    const int64_t n_groups = (int64_t)gridDim.x * (blockDim.x / 32) * RPW;
    const int64_t g = ((int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5)) * RPW + grp;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    // each group walks a contiguous chunk of the index stream (like a CSR row's column list)
    const int64_t per = (n_gather + n_groups - 1) / n_groups;
    const int64_t lo = g * per, hi = min(n_gather, lo + per);
    for (int64_t b = lo; b < hi; b += UNR) {
        float4 x[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int64_t p = b + u;
            x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < hi) x[u] = __ldg(table + (size_t)__ldg(idx + p) * G + gl);
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) { acc.x += x[u].x; acc.y += x[u].y; acc.z += x[u].z; acc.w += x[u].w; }
    }
    if (acc.x + acc.y + acc.z + acc.w == 123456.789f) sink[0] = acc.x;
}

template <int G>
void run(size_t table_mb, int64_t n_gather) {
    const size_t row_bytes = (size_t)G * 16, n_rows = table_mb * 1024 * 1024 / row_bytes;
    float4 *table; int32_t *idx; float *sink;
    CK(cudaMalloc(&table, n_rows * row_bytes)); CK(cudaMalloc(&idx, n_gather * 4)); CK(cudaMalloc(&sink, 4));
    CK(cudaMemset(table, 0, n_rows * row_bytes));
    int32_t *h = (int32_t *)malloc(n_gather * 4);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    for (int64_t i = 0; i < n_gather; ++i) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; h[i] = (int32_t)(s % n_rows); }
    CK(cudaMemcpy(idx, h, n_gather * 4, cudaMemcpyHostToDevice)); free(h);
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const int grid = 132 * 4 * 8;
    for (int i = 0; i < 3; ++i) gather_kernel<G><<<grid, 256>>>(table, idx, n_gather, sink);
    CK(cudaDeviceSynchronize());
    float best = 1e30f, tot = 0.f;
    for (int i = 0; i < 5; ++i) {
        CK(cudaEventRecord(e0)); gather_kernel<G><<<grid, 256>>>(table, idx, n_gather, sink); CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); best = ms < best ? ms : best; tot += ms;
    }
    printf("{\"row_bytes\": %zu, \"table_mb\": %zu, \"gathers\": %lld, \"ms_best\": %.4f, \"ms_mean\": %.4f, \"GBps_best\": %.1f, \"GBps_mean\": %.1f}\n",
           row_bytes, table_mb, (long long)n_gather, best, tot / 5, n_gather * row_bytes / (best * 1e-3) / 1e9, n_gather * row_bytes / (tot / 5 * 1e-3) / 1e9);
    CK(cudaFree(table)); CK(cudaFree(idx)); CK(cudaFree(sink));
}

int main() {
    const size_t sizes[] = {16, 40, 64, 96, 123, 384, 768, 6144};
    for (size_t mb : sizes) run<16>(mb, 8 << 20);
    for (size_t mb : sizes) run<32>(mb, 8 << 20);
    return 0;
}
