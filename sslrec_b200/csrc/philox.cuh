// Philox4x32-10 and the seed / uniform helpers every kernel RNG draws with (common.cuh includes it).
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <stdint.h>

namespace ssl {

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

}  // namespace ssl
