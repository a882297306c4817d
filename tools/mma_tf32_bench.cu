// Microbenchmark: legacy mma.sync TF32 (m16n8k8) and FP32 FFMA issue rates on this GPU.
// Decides whether a 3xTF32 error-compensated InfoNCE contraction on the legacy tensor path can beat the FFMA kernel.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void mma_loop(float *out, int iters) {
    float c[8][4] = {};
    unsigned a[4] = {threadIdx.x, threadIdx.x * 3u, 7u, 11u}, b[2] = {threadIdx.x * 5u, 13u};
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c[j][0]), "+f"(c[j][1]), "+f"(c[j][2]), "+f"(c[j][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    float s = 0; for (int j = 0; j < 8; ++j) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void mma_bf16_loop(float *out, int iters) {
    float c[8][4] = {};
    unsigned a[4] = {threadIdx.x, threadIdx.x * 3u, 7u, 11u}, b[2] = {threadIdx.x * 5u, 13u};
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c[j][0]), "+f"(c[j][1]), "+f"(c[j][2]), "+f"(c[j][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    float s = 0; for (int j = 0; j < 8; ++j) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void ffma_loop(float *out, int iters) {
    float c[32]; for (int j = 0; j < 32; ++j) c[j] = threadIdx.x + j;
    float a = 1.0001f + threadIdx.x * 1e-9f, b = 0.5f;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 32; ++j) c[j] = fmaf(c[j], a, b);
    }
    float s = 0; for (int j = 0; j < 32; ++j) s += c[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
    float *out; cudaMalloc(&out, 132 * 8 * 256 * 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int threads : {128, 256, 512}) for (int bps : {1, 2, 4}) {
        int iters = 20000; float ms;
        mma_loop<<<132 * bps, threads>>>(out, 100); cudaDeviceSynchronize();
        cudaEventRecord(e0); mma_loop<<<132 * bps, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        double fl = 132.0 * bps * (threads / 32) * (double)iters * 8 * 2.0 * 16 * 8 * 8;
        printf("mma.sync tf32 m16n8k8 : %3d thr x %d blk/SM: %.1f TFLOP/s\n", threads, bps, fl / ms / 1e9);
        cudaEventRecord(e0); mma_bf16_loop<<<132 * bps, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        fl = 132.0 * bps * (threads / 32) * (double)iters * 8 * 2.0 * 16 * 8 * 16;
        printf("mma.sync bf16 m16n8k16: %3d thr x %d blk/SM: %.1f TFLOP/s\n", threads, bps, fl / ms / 1e9);
        cudaEventRecord(e0); ffma_loop<<<132 * bps, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        fl = 132.0 * bps * threads * (double)iters * 32 * 2.0;
        printf("ffma                  : %3d thr x %d blk/SM: %.1f TFLOP/s\n", threads, bps, fl / ms / 1e9);
    }
    printf("cuda error: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
