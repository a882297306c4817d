// Popularity-proportional negative candidates (ssl_neg_candidates_pop; optional key train.neg_popularity = beta with
// train.dns_candidates = M >= 2).
//
// Input: the alias table of the item weights V_i (integers, sum n_item 2^32; built on the host, engine.pop_tables): one
// uint2 {thr, alias} per column c, column c holding item c with share thr[c] / 2^32 and alias[c] with the rest; a column
// with alias[c] == c is item c alone (every draw accepts it).  Candidate (b, j >= 1) reads the Philox4x32-10 blocks keyed
// (seed; b, j, blk, "DNSP"), blk = 0 .. 63, two draws (x, y) = (r.x, r.y), (r.z, r.w) per block, in this order:
//
//     c    = (x * n_item) >> 32                                   (sample_negs_kernel's multiply-shift)
//     item = c if alias[c] == c || y < thr[c], else alias[c]
//     the draw is rejected while item is in u's sorted training-CSR row; after 128 rejected draws the last one is kept
//
// so an accepted draw is item i with probability V_i / (n_item 2^32) restricted to u's non-positives.  cands[b, 0] = negs[b]
// (the loader's uniform negative).  With bias != null the kernel also writes, in fp32 and in this order,
//
//     bias[b, 0] = ln_m - lz_uni[u]                  bias[b, j] = (ln_m + lp[cands[b, j]]) - lz_pop[u]     (j >= 1)
//
// with lp[i] = log(V_i / (n_item 2^32)), lz_pop[u] = log(1 - sum_{i in P_u} V_i / (n_item 2^32)), lz_uni[u] = log(n_item - deg_u)
// (both 0 for a user who has every item) and ln_m = log M: bias[b, j] = ln(M q_j(c_j)), q_j candidate j's proposal restricted
// to u's non-positives, the logQ correction of the sampled softmax (ssm.cuh, ssm_fwd_logq_kernel).  It ignores the 128-draw
// cap.  A pure function of (seed, b, j): one thread per (b, j), no shared state.  The seed is read from *seed_ptr when it is
// given (a CUDA-graph replay reads the seed the host wrote there before it).
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <stdint.h>

#include "csr_contains.cuh"
#include "philox.cuh"

namespace ssl_pop {

constexpr int kThreadsPerBlock = 256;
constexpr uint32_t kTagCandidates = 0x444E5350u;   // "DNSP"

// the item of one draw (x, y) from column c = (x * n_item) >> 32
__device__ __forceinline__ uint32_t alias_draw(const uint2 *__restrict__ table, int64_t n_item, uint32_t x, uint32_t y) {
    const uint32_t c = (uint32_t)(((uint64_t)x * (uint64_t)n_item) >> 32);
    const uint2 t = __ldg(table + c);
    return (t.y == c || y < t.x) ? c : t.y;
}

static __global__ void __launch_bounds__(kThreadsPerBlock)
    neg_candidates_pop_kernel(const int64_t *__restrict__ users, const int64_t *__restrict__ negs, int64_t n_pairs, int M,
                              const int32_t *__restrict__ rowptr, const int32_t *__restrict__ cols, int64_t n_item,
                              const uint2 *__restrict__ table, const float *__restrict__ lp, const float *__restrict__ lz_pop,
                              const float *__restrict__ lz_uni, float ln_m, uint64_t seed, const uint64_t *__restrict__ seed_ptr,
                              int64_t *__restrict__ cands, float *__restrict__ bias) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_pairs * M) return;
    const int64_t b = e / M;
    const int j = (int)(e - b * M);
    const int64_t u = __ldg(users + b);
    if (j == 0) {
        cands[e] = __ldg(negs + b);
        if (bias != nullptr) bias[e] = ln_m - __ldg(lz_uni + u);
        return;
    }
    const uint2 key = ssl::seed_key(seed_ptr != nullptr ? __ldg(seed_ptr) : seed);
    const int lo = __ldg(rowptr + u), hi = __ldg(rowptr + u + 1);
    uint32_t neg = 0;
    for (uint32_t blk = 0; blk < 64; ++blk) {
        const uint4 r = ssl::philox4x32_10(make_uint4((uint32_t)b, (uint32_t)j, blk, kTagCandidates), key);
        neg = alias_draw(table, n_item, r.x, r.y);
        if (!ssl::csr_contains(cols, lo, hi, (int)neg)) break;
        neg = alias_draw(table, n_item, r.z, r.w);
        if (!ssl::csr_contains(cols, lo, hi, (int)neg)) break;
    }
    cands[e] = neg;
    if (bias != nullptr) bias[e] = (ln_m + __ldg(lp + neg)) - __ldg(lz_pop + u);
}

}  // namespace ssl_pop
