// MixGCF negatives fused with the BPR term (Huang et al., KDD 2021; optional key train.mixgcf): ssl_mixgcf_bpr_fwd /
// ssl_mixgcf_bpr_bwd.
//
// Input, per batch pair b: the user row u = U[ancs[b]] and positive row pbar = I[poss[b]] of the summed table the BPR term
// reads, the item rows X_l[.] of its layers l = 0 .. L (layer 0 = E0; n_layers = L + 1 <= 8) and M candidates c_j = cands[b, j].
//
//     alpha_l   = u01(Philox4x32-10(ctr = (b, l, 0, "MIXA"), key = seed_key(seed)).x)   or alpha_in[b, l] when injected
//     m_jl[k]   = fmaf(alpha_l, X_l[p][k], (1 - alpha_l) * X_l[c_j][k])                  (1 - alpha_l rounded to fp32)
//     s_jl      = fma(u[d-1], m_jl[d-1], ... fma(u[0], m_jl[0], 0) ...)                  one sequential fp32 FMA chain over k
//     j*_l      = the lowest j with the largest s_jl; a NaN s_jl never wins; all NaN -> j*_l = 0   (neg_select_kernel's rule)
//     nhat[k]   = ((m_{j*_0,0}[k] + m_{j*_1,1}[k]) + m_{j*_2,2}[k]) + ...                 sum pooling, layer order
//     z         = chain_k(u[k] * nhat[k]) - chain_k(u[k] * pbar[k])                       two sequential FMA chains
//     loss_b    = softplus(z) with torch's threshold-20 tail,  coef_b = sigmoid(z)          (bpr_fwd_kernel's epilogue)
//
// The forward writes loss_b, coef_b, picks[b, l] = c_{j*_l}, alpha[b, l] and nhat[b, :], which the backward reuses.  Work
// split: one warp per pair.  For each layer lane l scores the candidates j = l, l + 32, ... in ascending j and keeps its best;
// a 5-step xor-shuffle butterfly combines the 32 lane bests (larger score, else lower j): the maximum of a total order, so the
// pick does not depend on the combination order.  Lane k % 32 adds element k of the picked row into nhat (global memory, one
// writer per element); after __syncwarp lane 0 forms z.  Each output has one writer: no atomics.
//
// Backward (gradient through nhat only, none through the choice of j*): with g = scale * (*gscale) * coef_b[b] and
// gu[k] = g * u[k], it adds
//     user sink row ancs[b]       += g * (nhat[k] - pbar[k])
//     item sink row poss[b]       += -gu[k]
//     layer-l sink row poss[b]    += alpha_l * gu[k]
//     layer-l sink row picks[b,l] += (1 - alpha_l) * gu[k]
// with float atomics (batch ids repeat).  Run on gathered rows with identity ids (ancs = poss = 0 .. B-1, picks[b, l] = B + b)
// into stages filled with -0.0 it writes each position's contribution once, in this numbering: the user stage holds positions
// 0 .. B-1 (rows ancs), the item stage 0 .. B-1 (rows poss), the stage of layer l positions 0 .. B-1 (rows poss) and B .. 2B-1
// (rows picks[:, l]); train.deterministic scatters them in position order (ssl_scatter_rows_ordered).
//
// Rows are tbl + id * stride (elements; an item table pointer is item 0's row), so a view of an interleaved [N, V, d] layer
// and a plain [n, d] tensor both work.
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <math.h>
#include <stdint.h>

#include "philox.cuh"

namespace ssl_mix {

constexpr int kWarpsPerBlock = 8;
constexpr int kMaxLayers = 8;
constexpr uint32_t kTagAlpha = 0x4D495841u;   // "MIXA"

// the item rows of layers 0 .. n_layers-1; a __grid_constant__ kernel parameter, so indexing it by layer reads the parameter
// in place instead of copying it to local memory
struct LayerTables {
    const float *ptr[kMaxLayers];
    int64_t stride[kMaxLayers];
};
struct LayerSinks {
    float *ptr[kMaxLayers];
    int64_t stride[kMaxLayers];
};

__host__ __device__ __forceinline__ float alpha_draw(uint64_t seed, int64_t b, int l) {
    const uint4 r = ssl::philox4x32_10(make_uint4((uint32_t)b, (uint32_t)l, 0u, kTagAlpha), ssl::seed_key(seed));
    return ssl::u01(r.x);
}

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    mixgcf_fwd_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                      const __grid_constant__ LayerTables layers, int n_layers, const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss,
                      const int64_t *__restrict__ cands, int64_t n_pairs, int M, int dim, uint64_t seed,
                      const uint64_t *__restrict__ seed_ptr, const float *__restrict__ alpha_in, float *__restrict__ loss_b,
                      float *__restrict__ coef_b, int64_t *__restrict__ picks, float *__restrict__ alpha_out, float *nhat) {
    const int lane = (int)threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (b >= n_pairs) return;                              // warp-uniform
    const float *u = u_tbl + __ldg(ancs + b) * u_stride;
    const int64_t p = __ldg(poss + b);
    const int64_t *cb = cands + b * M;
    float *nb = nhat + b * dim;
    const uint64_t s = (alpha_in == nullptr && seed_ptr != nullptr) ? __ldg(seed_ptr) : seed;
    for (int l = 0; l < n_layers; ++l) {
        const float a = alpha_in != nullptr ? __ldg(alpha_in + b * n_layers + l) : alpha_draw(s, b, l);
        const float a1 = 1.f - a;
        const float *xl = layers.ptr[l];
        const int64_t xs = layers.stride[l];
        const float *xp = xl + p * xs;
        float best = 0.f;
        int best_j = M;                                    // M = no finite score yet
        for (int j = lane; j < M; j += 32) {
            const float *xc = xl + __ldg(cb + j) * xs;
            float sc = 0.f;
#pragma unroll 4
            for (int k = 0; k < dim; ++k) sc = fmaf(__ldg(u + k), fmaf(a, __ldg(xp + k), a1 * __ldg(xc + k)), sc);
            if (sc == sc && (best_j == M || sc > best)) {  // sc == sc: not NaN
                best = sc;
                best_j = j;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float so = __shfl_xor_sync(0xffffffffu, best, o);
            const int jo = __shfl_xor_sync(0xffffffffu, best_j, o);
            if (jo < M && (best_j == M || so > best || (so == best && jo < best_j))) {
                best = so;
                best_j = jo;
            }
        }
        const int64_t pick = __ldg(cb + (best_j == M ? 0 : best_j));
        const float *xc = xl + pick * xs;
        for (int k = lane; k < dim; k += 32) {
            const float m = fmaf(a, __ldg(xp + k), a1 * __ldg(xc + k));
            nb[k] = (l == 0) ? m : nb[k] + m;
        }
        if (lane == 0) {
            picks[b * n_layers + l] = pick;
            alpha_out[b * n_layers + l] = a;
        }
    }
    __syncwarp();                                          // nhat complete and visible to lane 0
    if (lane == 0) {
        const float *pb = i_tbl + p * i_stride;
        float zn = 0.f, zp = 0.f;
        for (int k = 0; k < dim; ++k) {
            const float uk = __ldg(u + k);
            zn = fmaf(uk, nb[k], zn);
            zp = fmaf(uk, __ldg(pb + k), zp);
        }
        const float z = zn - zp;
        loss_b[b] = (z > 20.f) ? z : log1pf(expf(z));
        coef_b[b] = 1.f / (1.f + expf(-z));
    }
}

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    mixgcf_bwd_kernel(const float *__restrict__ u_tbl, int64_t u_stride, const float *__restrict__ i_tbl, int64_t i_stride,
                      const int64_t *__restrict__ ancs, const int64_t *__restrict__ poss, const int64_t *__restrict__ picks,
                      int64_t n_pairs, int n_layers, int dim, const float *__restrict__ nhat, const float *__restrict__ alpha,
                      const float *__restrict__ coef_b, const float *__restrict__ gscale, float scale, float *g_users,
                      int64_t gu_stride, float *g_items, int64_t gi_stride, const __grid_constant__ LayerSinks g_layers) {
    const int lane = (int)threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (b >= n_pairs) return;
    const float g = scale * (gscale != nullptr ? __ldg(gscale) : 1.f) * __ldg(coef_b + b);
    const int64_t ia = __ldg(ancs + b), ip = __ldg(poss + b);
    const float *u = u_tbl + ia * u_stride, *pb = i_tbl + ip * i_stride, *nb = nhat + b * dim;
    for (int k = lane; k < dim; k += 32) {
        const float gu = g * __ldg(u + k);
        atomicAdd(g_users + ia * gu_stride + k, g * (__ldg(nb + k) - __ldg(pb + k)));
        atomicAdd(g_items + ip * gi_stride + k, -gu);
        for (int l = 0; l < n_layers; ++l) {
            const float a = __ldg(alpha + b * n_layers + l);
            float *gl = g_layers.ptr[l];
            const int64_t gs = g_layers.stride[l];
            atomicAdd(gl + ip * gs + k, a * gu);
            atomicAdd(gl + __ldg(picks + b * n_layers + l) * gs + k, (1.f - a) * gu);
        }
    }
}

}  // namespace ssl_mix
