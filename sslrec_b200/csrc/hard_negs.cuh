// Score-argmax selection of dynamic negative sampling (ssl_neg_select; optional key train.dns_candidates).
//
// Input: the anchor rows U[ancs[b]] and the candidate item rows I[cands[b, j]], j = 0 .. M-1, of B batch pairs.  For every
// pair the kernel writes the candidate whose score is largest:
//
//     s_j = fma(u[d-1], c_j[d-1], ... fma(u[1], c_j[1], fma(u[0], c_j[0], 0)) ...)      one sequential fp32 FMA chain over k
//     negs_out[b] = cands[b, j*]   j* = the lowest j with the largest s_j; a NaN s_j never wins; all NaN -> j* = 0
//
// "Largest" is fp32 comparison, so +0 and -0 tie and the lower j wins.  Work split: one warp per pair; lane l scores the
// candidates j = l, l + 32, ... in ascending j and keeps its best (a later j replaces it only on a strictly larger score);
// a 5-step xor-shuffle butterfly then combines the 32 lane bests with the same rule (larger score, else lower j), which
// selects the maximum of a total order, so the result does not depend on the combination order.  Lane 0 writes the one
// output of the pair: no atomics.  Rows are read through their strides (elements), so a view of an interleaved [N, V, d]
// table and a plain [n, d] tensor both work; the item table pointer is the row of item 0.
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <stdint.h>

namespace ssl_dns {

constexpr int kWarpsPerBlock = 8;

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    neg_select_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                      const int64_t *__restrict__ ancs, const int64_t *__restrict__ cands, int64_t n_pairs, int M, int dim,
                      int64_t *__restrict__ negs_out) {
    const int lane = (int)threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (b >= n_pairs) return;                              // warp-uniform
    const float *u = u_tbl + __ldg(ancs + b) * u_stride;
    const int64_t *cb = cands + b * M;
    float best = 0.f;
    int best_j = M;                                        // M = no finite score yet
    for (int j = lane; j < M; j += 32) {
        const float *c = i_tbl + __ldg(cb + j) * i_stride;
        float s = 0.f;
#pragma unroll 4
        for (int k = 0; k < dim; ++k) s = fmaf(__ldg(u + k), __ldg(c + k), s);
        if (s == s && (best_j == M || s > best)) {         // s == s: not NaN
            best = s;
            best_j = j;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float s = __shfl_xor_sync(0xffffffffu, best, o);
        const int j = __shfl_xor_sync(0xffffffffu, best_j, o);
        if (j < M && (best_j == M || s > best || (s == best && j < best_j))) {
            best = s;
            best_j = j;
        }
    }
    if (lane == 0) negs_out[b] = __ldg(cb + (best_j == M ? 0 : best_j));
}

}  // namespace ssl_dns
