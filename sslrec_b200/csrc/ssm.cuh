// Sampled softmax loss on cosine scores (optional key train.ssm_temperature): ssl_ssm_fwd / ssl_ssm_bwd.
//
// Input, per batch pair b: the user row u = U[ancs[b]], the positive c_0 = I[poss[b]] and the M candidates
// c_q = I[cands[b, q - 1]], q = 1 .. M (column q of every [B, M+1] output; q = 0 is the positive), temperature tau > 0.
// d is a multiple of 4; the row is cut into d/4 float4 slots, slot t holding elements 4t .. 4t+3.  G = the smallest power of
// two >= d/4 (1 .. 32).  Every quantity below is fp32, rounded after each operation, in exactly this order:
//
//     chain_t(x, y)  = fmaf(x[4t+3], y[4t+3], fmaf(x[4t+2], y[4t+2], fmaf(x[4t+1], y[4t+1], fmaf(x[4t], y[4t], 0))))
//                      (0 for a slot t >= d/4)
//     tree(v_0 .. v_{G-1}) = the xor butterfly: for o = 1, 2, 4, .. G/2: v_t = v_t + v_{t xor o}   (every t then holds the
//                      same value: ((v_0 + v_1) + (v_2 + v_3)) + ... for G = 4)
//     n_u = sqrtf(1e-8 + tree(chain_t(u, u)))         n_q = sqrtf(1e-8 + tree(chain_t(c_q, c_q)))
//     den_q = (n_u * n_q) * tau                        s_q = tree(chain_t(u, c_q)) / den_q
//     m = fmaxf(.. fmaxf(fmaxf(-inf, s_0), s_1) .., s_M)                       (a NaN score is skipped here ...)
//     S = tree(S_0 .. S_{G-1}),  S_t = ((0 + expf(s_t - m)) + expf(s_{t+G} - m)) + ...   over q = t, t + G, .. <= M
//                                                                               (... but makes S, and so loss_b, NaN)
//     loss_b = (m + logf(S)) - s_0           w_q = expf(s_q - m) / S - [q = 0]
//
// which is lse_q(s_q) - s_0 with x^ = x / sqrt(1e-8 + |x|^2) and s_q = x^_u . x^_q / tau.  The forward writes loss_b [B],
// s [B, M+1], w [B, M+1] and nrm [B, M+2] (column 0 n_u, column 1 + q n_q), which the backward reads instead of recomputing.
//
// logQ-corrected forward (ssm_fwd_logq_kernel, train.neg_popularity): with bias [B, M] (pop_negs.cuh), s^_0 = s_0 and
// s^_q = s_q - bias[b, q-1] for q >= 1 (one fp32 subtraction); m, S, loss_b and w are the lines above on s^ instead of s, and
// s is stored raw.  The backward below is then the correct backward unchanged.
//
// Backward, with g = scale * (*gscale) (gscale may be null: 1), per pair and in ascending q = 0 .. M:
//     gw_q = g * w_q      a_q = gw_q / den_q      e_q = (gw_q * s_q) / (n_q * n_q)
//     row c_q       += fmaf(a_q, u[k], -(e_q * c_q[k]))                        = g w_q (u^ / tau - s_q c^_q) / n_q
//     acc[k]         = fmaf(a_q, c_q[k], acc[k])        beta = fmaf(gw_q, s_q, beta)          (both from 0, in q order)
// and after the last q
//     row u         += fmaf(-(beta / (n_u * n_u)), u[k], acc[k])                = g sum_q w_q (c^_q / tau - s_q u^) / n_u
// The candidate and positive rows are added with float atomics as they come (one add per element and q); the user row is
// kept in registers across the pair and added once.  Duplicate candidates (a pair can draw an item twice or draw its positive)
// are separate terms that add into one row: no de-duplication; the logQ correction is the logq forward's alone.
// Run on gathered rows with identity ids (ancs = poss = 0 .. B-1, cands[b, j] = B + b M + j, the gathered item rows
// [I[poss]; I[cands]] as the item table) into -0.0 stages, it writes each position's contribution once, in this numbering:
// the user stage holds positions 0 .. B-1 (rows ancs), the item stage 0 .. B-1 (rows poss) and B + b M + j (rows cands[b, j]);
// train.deterministic scatters them in position order (ssl_scatter_rows_ordered).
//
// Work split: a group of G lanes per pair (lane t of the group owns slot t), 32 / G pairs per warp, so one load instruction
// reads 32 / G whole rows.  The forward's lane t writes s, w and nrm of the columns q = t (mod G), which it re-reads itself in
// the later passes; lane 0 of the group writes loss_b.  Rows are tbl + id * stride (elements; an item table pointer is item
// 0's row), 16-byte aligned with a stride that is a multiple of 4, so a view of an interleaved [N, V, d] table and a plain
// [n, d] tensor both work.
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <math.h>
#include <stdint.h>

namespace ssl_ssm {

constexpr int kWarpsPerBlock = 8;

// G: lanes per pair for a row of dim floats
__host__ __device__ __forceinline__ int group_lanes(int dim) {
    int g = 1;
    while (g * 4 < dim) g <<= 1;
    return g;
}

__device__ __forceinline__ float chain4(const float4 x, const float4 y) {
    return fmaf(x.w, y.w, fmaf(x.z, y.z, fmaf(x.y, y.y, fmaf(x.x, y.x, 0.f))));
}

__device__ __forceinline__ float tree(float v, int G) {
    for (int o = 1; o < G; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float4 load_row(const float *tbl, int64_t stride, int64_t id, int slot, bool live) {
    if (!live) return float4{0.f, 0.f, 0.f, 0.f};
    return __ldg(reinterpret_cast<const float4 *>(tbl + id * stride) + slot);
}

// the pair of this lane's group, whether the group has one (b < n_pairs), and its slot; lanes of a group past the batch read
// the last pair and write nothing, so every lane of the warp takes part in the shuffles
struct Lane {
    int64_t b;
    bool active;
    int slot;
};
__device__ __forceinline__ Lane lane_of(int64_t n_pairs, int G) {
    const int lane = (int)threadIdx.x & 31;
    const int64_t b = ((int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5)) * (32 / G) + lane / G;
    return Lane{b < n_pairs ? b : n_pairs - 1, b < n_pairs, lane % G};
}

// the forward of one pair; kLogQ: the softmax runs on s^_q = s_q - bias[b, q-1] (q >= 1, one fp32 subtraction; s^_0 = s_0)
// while s_out keeps the raw s_q (ssm_fwd_logq_kernel)
template <bool kLogQ>
__device__ __forceinline__ void ssm_fwd_body(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl,
                                             int64_t i_stride, const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss,
                                             const int64_t *__restrict__ cands, const float *__restrict__ bias, int64_t n_pairs, int M,
                                             int dim, float tau, float *__restrict__ loss_b, float *s_out, float *__restrict__ w_out,
                                             float *__restrict__ nrm_out) {
    const int G = group_lanes(dim);
    if (((int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5)) * (32 / G) >= n_pairs) return;   // warp-uniform
    const Lane ln = lane_of(n_pairs, G);
    const int64_t b = ln.b;
    const bool live = ln.slot * 4 < dim;
    const int64_t *cb = cands + b * M;
    const float *bb = kLogQ ? bias + b * M : nullptr;
    float *sb = s_out + b * (M + 1), *wb = w_out + b * (M + 1), *nb = nrm_out + b * (M + 2);
    const float4 u = load_row(u_tbl, u_stride, __ldg(ancs + b), ln.slot, live);
    const float nu = sqrtf(1e-8f + tree(chain4(u, u), G));
    float m = -INFINITY, s_pos = 0.f;
#pragma unroll 2
    for (int q = 0; q <= M; ++q) {
        const int64_t id = q == 0 ? __ldg(poss + b) : __ldg(cb + q - 1);
        const float4 c = load_row(i_tbl, i_stride, id, ln.slot, live);
        const float dt = tree(chain4(u, c), G);
        const float nq = sqrtf(1e-8f + tree(chain4(c, c), G));
        const float s = dt / ((nu * nq) * tau);
        m = fmaxf(m, kLogQ && q > 0 ? s - __ldg(bb + q - 1) : s);
        if (q == 0) s_pos = s;
        if (ln.active && q % G == ln.slot) {
            sb[q] = s;
            nb[1 + q] = nq;
        }
    }
    // s^_q, re-formed from the stored raw score by the same subtraction
    auto shat = [&](int q) { return kLogQ && q > 0 ? sb[q] - __ldg(bb + q - 1) : sb[q]; };
    float part = 0.f;
    if (ln.active)
        for (int q = ln.slot; q <= M; q += G) part += expf(shat(q) - m);
    const float S = tree(part, G);
    if (!ln.active) return;
    for (int q = ln.slot; q <= M; q += G) wb[q] = expf(shat(q) - m) / S - (q == 0 ? 1.f : 0.f);
    if (ln.slot == 0) {
        nb[0] = nu;
        loss_b[b] = (m + logf(S)) - s_pos;
    }
}

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    ssm_fwd_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                   const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss, const int64_t *__restrict__ cands,
                   int64_t n_pairs, int M, int dim, float tau, float *__restrict__ loss_b, float *s_out, float *__restrict__ w_out,
                   float *__restrict__ nrm_out) {
    ssm_fwd_body<false>(u_tbl, u_stride, i_tbl, i_stride, ancs, poss, cands, nullptr, n_pairs, M, dim, tau, loss_b, s_out, w_out,
                        nrm_out);
}

// the logQ-corrected forward (ssl_ssm_fwd_logq): bias [n_pairs, M] from ssl_neg_candidates_pop (pop_negs.cuh); the backward
// is ssm_bwd_kernel unchanged, since the derivative of every s_q needs only the raw s_q and the weight w_q
static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    ssm_fwd_logq_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                        const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss, const int64_t *__restrict__ cands,
                        const float *__restrict__ bias, int64_t n_pairs, int M, int dim, float tau, float *__restrict__ loss_b,
                        float *s_out, float *__restrict__ w_out, float *__restrict__ nrm_out) {
    ssm_fwd_body<true>(u_tbl, u_stride, i_tbl, i_stride, ancs, poss, cands, bias, n_pairs, M, dim, tau, loss_b, s_out, w_out,
                       nrm_out);
}

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    ssm_bwd_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                   const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss, const int64_t *__restrict__ cands,
                   int64_t n_pairs, int M, int dim, float tau, const float *__restrict__ s_in, const float *__restrict__ w_in,
                   const float *__restrict__ nrm_in, const float *__restrict__ gscale, float scale, float *g_users, int64_t gu_stride,
                   float *g_items, int64_t gi_stride) {
    const int G = group_lanes(dim);
    if (((int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5)) * (32 / G) >= n_pairs) return;   // warp-uniform
    const Lane ln = lane_of(n_pairs, G);
    if (!ln.active || ln.slot * 4 >= dim) return;          // no shuffles below: idle lanes may leave
    const int64_t b = ln.b;
    const int slot = ln.slot;
    const float g = scale * (gscale != nullptr ? __ldg(gscale) : 1.f);
    const int64_t *cb = cands + b * M;
    const float *sb = s_in + b * (M + 1), *wb = w_in + b * (M + 1), *nb = nrm_in + b * (M + 2);
    const int64_t ia = __ldg(ancs + b);
    const float4 u = load_row(u_tbl, u_stride, ia, slot, true);
    const float nu = __ldg(nb);
    float4 acc = float4{0.f, 0.f, 0.f, 0.f};
    float beta = 0.f;
#pragma unroll 2
    for (int q = 0; q <= M; ++q) {
        const int64_t id = q == 0 ? __ldg(poss + b) : __ldg(cb + q - 1);
        const float4 c = load_row(i_tbl, i_stride, id, slot, true);
        const float nq = __ldg(nb + 1 + q), s = __ldg(sb + q);
        const float gw = g * __ldg(wb + q);
        const float a = gw / ((nu * nq) * tau);
        const float e = (gw * s) / (nq * nq);
        atomicAdd(reinterpret_cast<float4 *>(g_items + id * gi_stride) + slot,
                  float4{fmaf(a, u.x, -(e * c.x)), fmaf(a, u.y, -(e * c.y)), fmaf(a, u.z, -(e * c.z)), fmaf(a, u.w, -(e * c.w))});
        acc = float4{fmaf(a, c.x, acc.x), fmaf(a, c.y, acc.y), fmaf(a, c.z, acc.z), fmaf(a, c.w, acc.w)};
        beta = fmaf(gw, s, beta);
    }
    const float r = -(beta / (nu * nu));
    atomicAdd(reinterpret_cast<float4 *>(g_users + ia * gu_stride) + slot,
              float4{fmaf(r, u.x, acc.x), fmaf(r, u.y, acc.y), fmaf(r, u.z, acc.z), fmaf(r, u.w, acc.w)});
}

}  // namespace ssl_ssm
