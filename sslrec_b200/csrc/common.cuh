// Shared helpers for the sslrec_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sslrec_b200.h"

namespace ssl {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);
extern int g_kmeans_rows_per_round;   // ssl_set_option("kmeans_rows_per_round", v): 4 (default) or 1 -- kmeans_assign_kernel<R>, bit-identical results
extern int g_predict_tiled;   // ssl_set_option("predict_tiled", v): 1 (default) = predict_tile_kernel, 0 = the warp-per-item kernel

#define SSL_CHECK_ARG(cond, ...)                \
    do {                                        \
        if (!(cond)) {                          \
            ssl::set_error(__VA_ARGS__);        \
            return SSL_E_ARG;                   \
        }                                       \
    } while (0)

#define SSL_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            ssl::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return SSL_E_CUDA;                                                                 \
        }                                                                                      \
    } while (0)

#define SSL_LAUNCH_CHECK(name)                                                                 \
    do {                                                                                       \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess) {                                                              \
            ssl::set_error("launch of %s failed: %s", name, cudaGetErrorString(e__));          \
            return SSL_E_CUDA;                                                                 \
        }                                                                                      \
        ssl::count_launch();                                                                   \
    } while (0)

constexpr int kNumSM = 132;   // H100 SXM

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG.  One call -> 4 x 32 random bits, keyed by a 64-bit seed and a
// 128-bit counter, so a mask / noise value is a pure function of (seed, stream, row, col): the
// forward and the transposed backward evaluate the same draw without storing it.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = mulhi32(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = mulhi32(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0;
        key.y += W1;
    }
    return ctr;
}

// 24-bit mantissa uniform in [0, 1), the granularity torch.rand(float32) has.
__host__ __device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

__host__ __device__ __forceinline__ uint2 seed_key(uint64_t seed) {
    return make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
}

// keep test of EdgeDrop / NodeDrop: floor(U + keep) == 1  <=>  U >= 1 - keep  (aug_utils.py:28,49)
__host__ __device__ __forceinline__ bool edge_keep_rng(uint64_t seed, uint32_t stream, uint32_t row, uint32_t col,
                                                       float keep) {
    uint4 r = philox4x32_10(make_uint4(row, col, stream, 0x45444745u /*"EDGE"*/), seed_key(seed));
    return u01(r.x) + keep >= 1.0f;
}
__host__ __device__ __forceinline__ bool node_keep_rng(uint64_t seed, uint32_t row, float keep) {
    uint4 r = philox4x32_10(make_uint4(row, 0u, 0u, 0x4E4F4445u /*"NODE"*/), seed_key(seed));
    return u01(r.x) + keep >= 1.0f;
}
// four consecutive uniforms of row `row`, elements 4*quad .. 4*quad+3
__host__ __device__ __forceinline__ float4 noise_u4_rng(uint64_t seed, uint32_t stream, uint32_t row, uint32_t quad) {
    uint4 r = philox4x32_10(make_uint4(row, quad, stream, 0x4E4F4953u /*"NOIS"*/), seed_key(seed));
    return make_float4(u01(r.x), u01(r.y), u01(r.z), u01(r.w));
}

// 3xTF32 split: hi = round-to-nearest tf32(x), lo = round-to-nearest tf32(x - hi).  Rounding (not
// truncating) both parts keeps the residual |x - hi - lo| <= 2^-22 |x| and unbiased.
__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t y;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(y) : "f"(x));
    return __uint_as_float(y);
}
__device__ __forceinline__ void tf32_split(float x, float &hi, float &lo) {
    hi = tf32_rna(x);
    lo = tf32_rna(x - hi);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the live count of a device-bounded launch (the *_live entry points): *n_live clamped to [0, cap]
__device__ __forceinline__ int64_t live_count(const int64_t *n_live, int64_t cap) {
    const int64_t v = *n_live;
    return v < 0 ? 0 : (v > cap ? cap : v);
}

__device__ __forceinline__ float4 ldg4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ void fma4(float4 &a, float w, const float4 &x) {
    a.x = fmaf(w, x.x, a.x);
    a.y = fmaf(w, x.y, a.y);
    a.z = fmaf(w, x.z, a.z);
    a.w = fmaf(w, x.w, a.w);
}
__device__ __forceinline__ void add4(float4 &a, const float4 &x) {
    a.x += x.x;
    a.y += x.y;
    a.z += x.z;
    a.w += x.w;
}

}  // namespace ssl
