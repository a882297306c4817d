// Column backward of the in-batch sampled softmax (optional key train.ssm_in_batch): ssl_nce_bwd_cols.
//
// The term contracts every pair's user row against the batch's 2B item rows (the columns: the B positives, then the B
// loader negatives) with column weights w_c (include/sslrec_b200.h, a28).  Its column gradient comes from the swapped
// contraction (R = the normalised columns t^, C = the scaled users, colscale = g ln2 / rowsum), which cannot apply w_c: in
// that role the forward's column weight is a per-ROW factor.  This kernel applies it.  Per column c, every quantity fp32 and
// rounded after each operation, in exactly this order:
//
//     d[k]  = ((0 + dt_part[0, c, k]) + dt_part[1, c, k]) + ... + dt_part[n_split - 1, c, k]
//     d[k]  = d[k] * w[c]
//     proj  = tree(chain_l)   chain_l = fmaf(t[l + 96] d[l + 96], fmaf(t[l + 64] d[l + 64], fmaf(t[l + 32] d[l + 32],
//                                        fmaf(t[l] d[l], 0))))   (lane l = 0 .. 31; entries k >= dim are 0)
//             tree = the xor butterfly over the 32 lanes: for o = 16, 8, 4, 2, 1: v_l = v_l + v_{l xor o}
//     v[k]  = rinv[c] * fmaf(-t[k], proj, d[k])                       = rinv_c (dt^ - t^ (t^ . dt^)), the normalisation backward
//     sink[ids[c] * stride + k] += v[k]                               (float atomics; ids == NULL: row c, one add per element)
//
// with t = t_hat[c] (the normalised column, row-major [n, dim]) and rinv[c] its 1/norm.  Run with ids = NULL into a -0.0
// stage, it writes each column's contribution once, which train.deterministic scatters in position order
// (ssl_scatter_rows_ordered).  Unlike ssl_nce_bwd_table (contiguous rows 0 .. n-1, no ids, no weights) it addresses the
// sink through ids and scales by w.
//
// Work split: one warp per column, lane l holds entries l, l + 32, l + 64, l + 96.  A warp whose column is past n returns
// as a whole, so every shuffle runs with all 32 lanes.
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <math.h>
#include <stdint.h>

namespace ssl_inb {

constexpr int kWarpsPerBlock = 8;
constexpr int kPerLane = 4;          // SSL_MAX_DIM / 32

__device__ __forceinline__ float warp_tree(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = v + __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    nce_bwd_cols_kernel(const float *__restrict__ dt_part, int n_split, const float *__restrict__ t_hat, const float *__restrict__ rinv,
                        const float *__restrict__ colw, const int64_t *__restrict__ ids, int64_t n, int dim, float *sink,
                        int64_t stride) {
    const int lane = (int)threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * kWarpsPerBlock + ((int)threadIdx.x >> 5);
    if (c >= n) return;                                    // warp-uniform
    float d[kPerLane], t[kPerLane];
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) d[i] = 0.f;
    for (int s = 0; s < n_split; ++s) {
        const float *src = dt_part + ((size_t)s * n + c) * dim;
#pragma unroll
        for (int i = 0; i < kPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) d[i] = d[i] + __ldg(src + k);
        }
    }
    const float w = __ldg(colw + c);
    float chain = 0.f;
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) {
        const int k = lane + 32 * i;
        t[i] = k < dim ? __ldg(t_hat + c * dim + k) : 0.f;
        d[i] = d[i] * w;
        chain = fmaf(t[i], d[i], chain);
    }
    const float proj = warp_tree(chain);
    const float r = __ldg(rinv + c);
    float *dst = sink + (ids != nullptr ? __ldg(ids + c) : c) * stride;
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) atomicAdd(dst + k, r * fmaf(-t[i], proj, d[i]));
    }
}

}  // namespace ssl_inb
