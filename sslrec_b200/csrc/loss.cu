// Row-wise kernels around the InfoNCE contraction: gathers + BPR, normalisation with the K-major
// tile copy, the term's forward/backward epilogues, reductions, regulariser and Adam.
// All are HBM/L2-bound streaming kernels: one warp per embedding row, lanes over the dim.
#include <math_constants.h>

#include "common.cuh"
#include "f16x3.cuh"
#include "predict_tile.cuh"

namespace {

constexpr int kMaxPerLane = SSL_MAX_DIM / 32;   // 4 floats per lane at dim = 128
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ void load_row(const float *__restrict__ p, int dim, int lane, float (&x)[kMaxPerLane]) {
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        x[i] = (k < dim) ? __ldg(p + k) : 0.f;
    }
}
__device__ __forceinline__ float dot_rows(const float (&a)[kMaxPerLane], const float (&b)[kMaxPerLane]) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) s = fmaf(a[i], b[i], s);
    return ssl::warp_sum(s);
}

// ---------------------------------------------------------------------------------------------
// BPR
// ---------------------------------------------------------------------------------------------
__global__ void bpr_fwd_kernel(const float *users, int64_t us, const float *items, int64_t is, const int64_t *ancs,
                               const int64_t *poss, const int64_t *negs, int64_t batch, int dim, float *loss_b, float *coef_b) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float a[kMaxPerLane], p[kMaxPerLane], n[kMaxPerLane];
    load_row(users + ancs[b] * us, dim, lane, a);
    load_row(items + poss[b] * is, dim, lane, p);
    load_row(items + negs[b] * is, dim, lane, n);
    const float z = dot_rows(a, n) - dot_rows(a, p);
    if (lane == 0) {
        // softplus with torch's threshold-20 linear tail (F.softplus, loss_utils.py:10)
        loss_b[b] = (z > 20.f) ? z : log1pf(expf(z));
        coef_b[b] = 1.f / (1.f + expf(-z));
    }
}

__global__ void bpr_bwd_kernel(const float *users, int64_t us, const float *items, int64_t is, const int64_t *ancs,
                               const int64_t *poss, const int64_t *negs, int64_t batch, int dim, const float *coef_b,
                               const float *gscale, float scale, float *gu, int64_t gus, float *gi, int64_t gis) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    const float g = scale * (gscale ? __ldg(gscale) : 1.f) * coef_b[b];
    float a[kMaxPerLane], p[kMaxPerLane], n[kMaxPerLane];
    const int64_t ia = ancs[b], ip = poss[b], in = negs[b];
    load_row(users + ia * us, dim, lane, a);
    load_row(items + ip * is, dim, lane, p);
    load_row(items + in * is, dim, lane, n);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) {
            atomicAdd(gu + ia * gus + k, g * (n[i] - p[i]));
            atomicAdd(gi + ip * gis + k, -g * a[i]);
            atomicAdd(gi + in * gis + k, g * a[i]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// rows_normalize: one 64-row tile per block; row-major copy, K-major tile copy, 1/norm.
// The tile copy stores logical column c of the tile at physical slot 4*(c%16) + c/16 so that a
// thread of ssl_softmax_gemm reads its four columns {tx, tx+16, tx+32, tx+48} with one 16 B load.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rows_normalize_kernel(const float *__restrict__ x, int64_t stride, const int64_t *__restrict__ idx,
                                                           int64_t n, int dim, int mode, float alpha, float *__restrict__ out,
                                                           float *__restrict__ out_t, float *__restrict__ rinv,
                                                           float *__restrict__ out_hi, float *__restrict__ out_lo,
                                                           float *__restrict__ out_thi, float *__restrict__ out_tlo, int64_t t_pitch) {
    extern __shared__ float tile[];   // [64][dim + 1]
    const int pitch = dim + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t row0 = (int64_t)blockIdx.x * 64;
    for (int lr = warp; lr < 64; lr += 8) {
        const int64_t row = row0 + lr;
        float v[kMaxPerLane];
        float ri = 0.f;
        if (row < n) {
            const int64_t src = idx ? idx[row] : row;
            load_row(x + src * stride, dim, lane, v);
            if (mode == 1) {
#pragma unroll
                for (int i = 0; i < kMaxPerLane; ++i) if (lane + 32 * i < dim) v[i] += 1e-8f;    // F.normalize(x + 1e-8)
            }
            const float ss = dot_rows(v, v);
            ri = (mode == 0) ? (1.f / sqrtf(1e-8f + ss)) : (mode == 3) ? 1.f : (1.f / fmaxf(sqrtf(ss), 1e-12f));   // mode 3: raw rows
            if (lane == 0 && rinv) rinv[row] = ri;
        } else {
#pragma unroll
            for (int i = 0; i < kMaxPerLane; ++i) v[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) {
                const float y = v[i] * ri * alpha;
                tile[lr * pitch + k] = y;
                out[row * dim + k] = y;            // rows n .. ceil64(n) are written as zeros
                if (out_hi != nullptr) {           // tf32 split for the tensor-core contraction
                    float hi, lo;
                    ssl::tf32_split(y, hi, lo);
                    out_hi[row * dim + k] = hi;
                    out_lo[row * dim + k] = lo;
                }
            }
        }
    }
    if (out_t == nullptr && out_thi == nullptr) return;
    __syncthreads();
    if (out_t != nullptr) {
        float *dst = out_t + (size_t)blockIdx.x * dim * 64;
        for (int i = threadIdx.x; i < dim * 64; i += 256) {
            const int k = i >> 6, q = i & 63;
            const int c = (q >> 2) + 16 * (q & 3);
            dst[i] = tile[c * pitch + k];
        }
    }
    if (out_thi != nullptr) {       // transposed tf32 split: [dim, t_pitch], 64 columns per block
        // within every group of 8 columns, row 8j + 2t + c goes to column 8j + t + 4c: the order in which the tensor-core
        // contraction holds E in its accumulator fragment, so that fragment feeds the second GEMM's A operand unpermuted
        for (int i = threadIdx.x; i < dim * 64; i += 256) {
            const int k = i >> 6, c = i & 63;
            const int q = (c & ~7) | ((c & 7) >> 1) | ((c & 1) << 2);
            float hi, lo;
            ssl::tf32_split(tile[c * pitch + k], hi, lo);
            out_thi[(size_t)k * t_pitch + row0 + q] = hi;
            out_tlo[(size_t)k * t_pitch + row0 + q] = lo;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// rows_normalize_f16x3: the operands of ssl_softmax_gemm_f16x3.  rows_normalize's row-major copy and 1/norm (the same
// arithmetic, so ``out`` and ``rinv`` are bit-identical to it), plus the f16x3 split of the output (f16x3.cuh) as
// row-major fp16 hi / lo [ceil64(n), dim].  No transposed copy: the contraction reads the row-major tile both ways.
// One 64-row tile per block, one warp per row; rows n .. ceil64(n) are written as zeros.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rows_normalize_f16x3_kernel(const float *__restrict__ x, int64_t stride, const int64_t *__restrict__ idx,
                                                                 int64_t n, int dim, int mode, float alpha, float *__restrict__ out,
                                                                 float *__restrict__ rinv, __half *__restrict__ out_hi,
                                                                 __half *__restrict__ out_lo) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t row0 = (int64_t)blockIdx.x * 64;
    for (int lr = warp; lr < 64; lr += 8) {
        const int64_t row = row0 + lr;
        float v[kMaxPerLane];
        float ri = 0.f;
        if (row < n) {
            const int64_t src = idx ? idx[row] : row;
            load_row(x + src * stride, dim, lane, v);
            if (mode == 1) {
#pragma unroll
                for (int i = 0; i < kMaxPerLane; ++i) if (lane + 32 * i < dim) v[i] += 1e-8f;    // F.normalize(x + 1e-8)
            }
            const float ss = dot_rows(v, v);
            ri = (mode == 0) ? (1.f / sqrtf(1e-8f + ss)) : (1.f / fmaxf(sqrtf(ss), 1e-12f));
            if (lane == 0 && rinv) rinv[row] = ri;
        } else {
#pragma unroll
            for (int i = 0; i < kMaxPerLane; ++i) v[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) {
                const float y = v[i] * ri * alpha;
                out[row * dim + k] = y;
                ssl::f16x3_split1(y, out_hi[row * dim + k], out_lo[row * dim + k]);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// InfoNCE term epilogues
// ---------------------------------------------------------------------------------------------
__global__ void nce_finalize_kernel(const float *rowsum_part, const float *o_part, int n_split, int64_t batch, int dim,
                                    const float *a_hat, const float *p_hat, float tau, float deno_eps, float *rowsum,
                                    float *obar, float *loss_b) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float rs = 0.f;
    for (int s = 0; s < n_split; ++s) rs += rowsum_part[(size_t)s * batch + b];
    rs += deno_eps;
    float o[kMaxPerLane] = {0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < n_split; ++s) {
        const float *src = o_part + ((size_t)s * batch + b) * dim;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) o[i] += src[k];
        }
    }
    const float inv = 1.f / rs;
    float a[kMaxPerLane], p[kMaxPerLane];
    load_row(a_hat + b * dim, dim, lane, a);     // a_hat holds a^ * log2e / tau
    load_row(p_hat + b * dim, dim, lane, p);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) obar[b * dim + k] = o[i] * inv;
    }
    const float ap = dot_rows(a, p) * kLn2;       // = (a^ . p^) / tau
    if (lane == 0) {
        rowsum[b] = rs;
        loss_b[b] = -ap + 1.f / tau + logf(rs);
    }
}

// log-sum-exp epilogue without a positive pair (lightgcl.py:112-113): rowsum = sum of the split partials + eps,
// obar = o / rowsum (the softmax-weighted table average = gradient direction of the anchor), loss_b = log(rowsum)
__global__ void lse_finalize_kernel(const float *rowsum_part, const float *o_part, int n_split, int64_t batch, int dim, float eps,
                                    float *rowsum, float *obar, float *loss_b) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float rs = 0.f;
    for (int s = 0; s < n_split; ++s) rs += rowsum_part[(size_t)s * batch + b];
    rs += eps;
    const float inv = 1.f / rs;
    for (int k = lane; k < dim; k += 32) {
        float o = 0.f;
        for (int s = 0; s < n_split; ++s) o += o_part[((size_t)s * batch + b) * dim + k];
        obar[b * dim + k] = o * inv;
    }
    if (lane == 0) {
        rowsum[b] = rs;
        loss_b[b] = logf(rs);
    }
}

__global__ void nce_colscale_kernel(const float *rowsum, int64_t batch, const float *gscale, float scale, float *colscale) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    colscale[b] = scale * (gscale ? __ldg(gscale) : 1.f) * kLn2 / rowsum[b];
}
// ssl_nce_colscale_live: the mean over the first `live` anchors; 0 past them, so the swapped gemm sums nothing from a padding row
__global__ void nce_colscale_live_kernel(const float *rowsum, int64_t batch, const int64_t *n_live, const float *gscale, float scale,
                                         float *colscale) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    const int64_t live = ssl::live_count(n_live, batch);
    colscale[b] = (b < live) ? (scale / (float)live) * (gscale ? __ldg(gscale) : 1.f) * kLn2 / rowsum[b] : 0.f;
}

// d a^ = g/tau (obar - p^) ; d p^ = -g/tau a^ ; through x^ = x * rinv:  dx = rinv (dx^ - x^ (x^ . dx^))
// LIVE (ssl_nce_bwd_rows_live): rows past *n_live are skipped and g is divided by the live count
template <bool LIVE>
__global__ void nce_bwd_rows_kernel(const float *a_hat, const float *p_hat, const float *obar, const float *rinv1,
                                    const float *rinv2, const int64_t *idx, int64_t batch, int dim, float tau,
                                    const float *gscale, float scale, float *g1, int64_t g1s, float *g2, int64_t g2s,
                                    const int64_t *n_live) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    if (LIVE) {
        const int64_t live = ssl::live_count(n_live, batch);
        if (b >= live) return;
        scale /= (float)live;
    }
    const float g = scale * (gscale ? __ldg(gscale) : 1.f) / tau;
    const float unscale = tau * kLn2;             // a_hat rows are scaled by log2e / tau
    float a[kMaxPerLane], p[kMaxPerLane], ob[kMaxPerLane];
    load_row(a_hat + b * dim, dim, lane, a);
    load_row(p_hat + b * dim, dim, lane, p);
    load_row(obar + b * dim, dim, lane, ob);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) a[i] *= unscale;
    const int64_t row = idx[b];
    if (g1 != nullptr) {
        float d[kMaxPerLane];
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) d[i] = g * (ob[i] - p[i]);
        const float proj = dot_rows(a, d);
        const float r1 = rinv1[b];
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) atomicAdd(g1 + row * g1s + k, r1 * (d[i] - a[i] * proj));
        }
    }
    if (g2 != nullptr) {
        float d[kMaxPerLane];
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) d[i] = -g * a[i];
        const float proj = dot_rows(p, d);
        const float r2 = rinv2[b];
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) atomicAdd(g2 + row * g2s + k, r2 * (d[i] - p[i] * proj));
        }
    }
}

__global__ void nce_bwd_table_kernel(const float *dt_part, int n_split, const float *t_hat, const float *rinv, int64_t n,
                                     int dim, float *g_table, int64_t gs, int accumulate) {
    const int lane = threadIdx.x & 31;
    const int64_t j = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (j >= n) return;
    float d[kMaxPerLane] = {0.f, 0.f, 0.f, 0.f}, t[kMaxPerLane];
    for (int s = 0; s < n_split; ++s) {
        const float *src = dt_part + ((size_t)s * n + j) * dim;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) d[i] += src[k];
        }
    }
    load_row(t_hat + j * dim, dim, lane, t);
    const float proj = dot_rows(t, d);
    const float r = rinv[j];
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) {
            const float v = r * (d[i] - t[i] * proj);
            float *dst = g_table + j * gs + k;
            *dst = accumulate ? (*dst + v) : v;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// deterministic reductions, axpy, Adam
// ---------------------------------------------------------------------------------------------
constexpr int kRedBlocks = 592;   // 4 per SM

template <bool SQ>
__global__ void __launch_bounds__(256) reduce_stage1(const float *__restrict__ x, int64_t n, float *__restrict__ part) {
    __shared__ float sh[8];
    float s = 0.f;
    const int64_t n4 = n / 4;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
        const float4 v = ssl::ldg4(x + i * 4);
        s += SQ ? (v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w) : (v.x + v.y + v.z + v.w);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const float v = x[n4 * 4 + threadIdx.x];
        s += SQ ? v * v : v;
    }
    s = ssl::warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += sh[i];
        part[blockIdx.x] = t;
    }
}
// ssl_sum_live: sum of the first *n_live entries of a vector with room for n, times alpha / live
__global__ void __launch_bounds__(1024) sum_live_kernel(const float *__restrict__ x, int64_t n, const int64_t *__restrict__ n_live, float alpha,
                                                        float *__restrict__ out) {
    __shared__ float sh[32];
    const int64_t live = ssl::live_count(n_live, n);
    float s = 0.f;
    for (int64_t i = threadIdx.x; i < live; i += 1024) s += x[i];
    s = ssl::warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 32; ++i) t += sh[i];
        out[0] = live > 0 ? (alpha / (float)live) * t : 0.f;
    }
}
__global__ void __launch_bounds__(1024) reduce_stage2(const float *__restrict__ part, int n, float alpha, float *__restrict__ out) {
    __shared__ float sh[32];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += 1024) s += part[i];
    s = ssl::warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 32; ++i) t += sh[i];
        out[0] = alpha * t;
    }
}

__global__ void axpy_kernel(const float *__restrict__ x, float *__restrict__ y, int64_t n, const float *gscale, float alpha) {
    const float a = alpha * (gscale ? __ldg(gscale) : 1.f);
    const int64_t n4 = n / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 xv = ssl::ldg4(x + i * 4);
        float4 yv = *reinterpret_cast<float4 *>(y + i * 4);
        ssl::fma4(yv, a, xv);
        *reinterpret_cast<float4 *>(y + i * 4) = yv;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = n4 * 4 + threadIdx.x;
        y[i] = fmaf(a, x[i], y[i]);
    }
}

struct AdamK {
    float b1, b2, omb1, omb2, step_size, inv_bc2_sqrt, eps, wd;   // omb = 1 - beta evaluated in double on the host, as torch does
};
__device__ __forceinline__ void adam1(float &p, float g, float &m, float &v, const AdamK &k) {
    const float b1 = k.b1, b2 = k.b2, step_size = k.step_size, inv_bc2_sqrt = k.inv_bc2_sqrt, eps = k.eps, wd = k.wd;
    if (wd != 0.f) g = fmaf(wd, p, g);
    m = fmaf(b1, m, k.omb1 * g);                  // exp_avg.lerp_(grad, 1 - beta1)
    v = fmaf(b2, v, k.omb2 * g * g);              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) * inv_bc2_sqrt + eps;
    p -= step_size * (m / denom);
}
struct PeerPtrs {
    float *p[SSL_MAX_PEERS];
    int n;
};
// bias corrections from a device-resident step count (CUDA-graph replay): double precision like the host path
__global__ void adam_prepare_kernel(const int64_t *__restrict__ step_dev, double lr, double beta1, double beta2, float *__restrict__ out2) {
    const double step = (double)*step_dev;
    out2[0] = (float)(lr / (1.0 - pow(beta1, step)));
    out2[1] = (float)(1.0 / sqrt(1.0 - pow(beta2, step)));
}

__global__ void adam_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
                            int64_t n, AdamK k, PeerPtrs peers, const float *__restrict__ dyn) {
    if (dyn != nullptr) {
        k.step_size = __ldg(dyn);
        k.inv_bc2_sqrt = __ldg(dyn + 1);
    }
    const int64_t n4 = n / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 pv = *reinterpret_cast<float4 *>(p + i * 4), mv = *reinterpret_cast<float4 *>(m + i * 4),
               vv = *reinterpret_cast<float4 *>(v + i * 4);
        const float4 gv = ssl::ldg4(g + i * 4);
        adam1(pv.x, gv.x, mv.x, vv.x, k);
        adam1(pv.y, gv.y, mv.y, vv.y, k);
        adam1(pv.z, gv.z, mv.z, vv.z, k);
        adam1(pv.w, gv.w, mv.w, vv.w, k);
        *reinterpret_cast<float4 *>(p + i * 4) = pv;
        for (int q = 0; q < peers.n; ++q) *reinterpret_cast<float4 *>(peers.p[q] + i * 4) = pv;   // NVLink stores
        *reinterpret_cast<float4 *>(m + i * 4) = mv;
        *reinterpret_cast<float4 *>(v + i * 4) = vv;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = n4 * 4 + threadIdx.x;
        adam1(p[i], g[i], m[i], v[i], k);
        for (int q = 0; q < peers.n; ++q) peers.p[q][i] = p[i];
    }
}

// ---------------------------------------------------------------------------------------------
// full_predict + _mask_predict: one block per (user, 1024-item chunk); the user row sits in
// shared memory, each warp walks item rows (coalesced 4*dim-byte reads).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) predict_mask_kernel(const float *ut, int64_t us, const float *itab, int64_t is,
                                                         const int64_t *users, int64_t n_item, int dim, const int64_t *mask_dense,
                                                         const int32_t *trn_rowptr, const int32_t *trn_cols, float *preds) {
    __shared__ float urow[SSL_MAX_DIM];
    const int64_t b = blockIdx.y;
    const int64_t u = users[b];
    for (int k = threadIdx.x; k < dim; k += 256) urow[k] = ut[u * us + k];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float uq[kMaxPerLane];
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) uq[i] = (lane + 32 * i < dim) ? urow[lane + 32 * i] : 0.f;
    const int64_t i0 = (int64_t)blockIdx.x * 1024;
    const int64_t i1 = min(i0 + 1024, n_item);
    for (int64_t it = i0 + warp; it < i1; it += 8) {
        float row[kMaxPerLane];
        load_row(itab + it * is, dim, lane, row);
        const float s = dot_rows(uq, row);
        if (lane == 0) {
            float m = 0.f;
            if (mask_dense) m = (float)mask_dense[b * n_item + it];
            preds[b * n_item + it] = s * (1.f - m) - 1e8f * m;    // base_model.py:36
        }
    }
    if (mask_dense == nullptr && trn_rowptr != nullptr) {
        __syncthreads();   // the block's own score writes above are visible to its threads
        for (int e = trn_rowptr[u] + threadIdx.x; e < trn_rowptr[u + 1]; e += 256) {
            const int64_t it = trn_cols[e];
            if (it >= i0 && it < i1) preds[b * n_item + it] = preds[b * n_item + it] * 0.f - 1e8f;   // s*(1-1) - 1e8*1
        }
    }
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" int ssl_bpr_fwd(const float *users, int64_t u_stride, const float *items, int64_t i_stride, const int64_t *ancs,
                           const int64_t *poss, const int64_t *negs, int64_t batch, int32_t dim, float *loss_b, float *coef_b,
                           void *stream) {
    SSL_CHECK_ARG(users && items && ancs && poss && negs && loss_b && coef_b, "ssl_bpr_fwd: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_bpr_fwd: dim %d out of range", dim);
    if (batch == 0) return SSL_OK;
    bpr_fwd_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(users, u_stride, items, i_stride, ancs, poss, negs, batch, dim, loss_b, coef_b);
    SSL_LAUNCH_CHECK("bpr_fwd_kernel");
    return SSL_OK;
}

extern "C" int ssl_bpr_bwd(const float *users, int64_t u_stride, const float *items, int64_t i_stride, const int64_t *ancs,
                           const int64_t *poss, const int64_t *negs, int64_t batch, int32_t dim, const float *coef_b,
                           const float *gscale, float scale, float *g_users, int64_t gu_stride, float *g_items,
                           int64_t gi_stride, void *stream) {
    SSL_CHECK_ARG(users && items && ancs && poss && negs && coef_b && g_users && g_items, "ssl_bpr_bwd: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_bpr_bwd: dim %d out of range", dim);
    if (batch == 0) return SSL_OK;
    bpr_bwd_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(users, u_stride, items, i_stride, ancs, poss, negs, batch, dim, coef_b, gscale, scale, g_users, gu_stride, g_items, gi_stride);
    SSL_LAUNCH_CHECK("bpr_bwd_kernel");
    return SSL_OK;
}

extern "C" int ssl_rows_normalize(const float *x, int64_t stride, const int64_t *idx, int64_t n, int32_t dim, int32_t norm_mode,
                                  float alpha, float *out, float *out_t, float *rinv, float *out_hi, float *out_lo,
                                  float *out_thi, float *out_tlo, int64_t t_pitch, void *stream) {
    SSL_CHECK_ARG(x && out, "ssl_rows_normalize: null argument");
    SSL_CHECK_ARG((out_hi == nullptr) == (out_lo == nullptr) && (out_thi == nullptr) == (out_tlo == nullptr), "ssl_rows_normalize: hi and lo outputs go together");
    SSL_CHECK_ARG(out_thi == nullptr || (t_pitch >= (n + 63) / 64 * 64 && t_pitch % 4 == 0), "ssl_rows_normalize: t_pitch must be >= ceil64(n) and a multiple of 4");
    SSL_CHECK_ARG(dim >= 4 && dim <= SSL_MAX_DIM && dim % 4 == 0, "ssl_rows_normalize: dim %d must be a multiple of 4 <= %d", dim, SSL_MAX_DIM);
    SSL_CHECK_ARG(norm_mode >= 0 && norm_mode <= 3, "ssl_rows_normalize: bad norm_mode");
    if (n == 0) return SSL_OK;
    const size_t smem = sizeof(float) * 64 * (dim + 1);
    rows_normalize_kernel<<<(unsigned)((n + 63) / 64), 256, smem, STREAM>>>(x, stride, idx, n, dim, norm_mode, alpha, out, out_t, rinv, out_hi, out_lo, out_thi, out_tlo, t_pitch);
    SSL_LAUNCH_CHECK("rows_normalize_kernel");
    return SSL_OK;
}

extern "C" int ssl_rows_normalize_f16x3(const float *x, int64_t stride, const int64_t *idx, int64_t n, int32_t dim, int32_t norm_mode,
                                        float alpha, float *out, float *rinv, uint16_t *out_hi, uint16_t *out_lo, void *stream) {
    SSL_CHECK_ARG(x && out && out_hi && out_lo, "ssl_rows_normalize_f16x3: null argument");
    SSL_CHECK_ARG(dim == 32 || dim == 64, "ssl_rows_normalize_f16x3: dim %d not supported (32 or 64)", dim);
    SSL_CHECK_ARG(norm_mode >= 0 && norm_mode <= 2, "ssl_rows_normalize_f16x3: norm_mode %d (0, 1 or 2: unit rows only)", norm_mode);
    SSL_CHECK_ARG(fabsf(alpha) <= ssl::kF16MaxAlpha, "ssl_rows_normalize_f16x3: |alpha| = %g exceeds %g", (double)fabsf(alpha),
                  (double)ssl::kF16MaxAlpha);
    if (n == 0) return SSL_OK;
    rows_normalize_f16x3_kernel<<<(unsigned)((n + 63) / 64), 256, 0, STREAM>>>(x, stride, idx, n, dim, norm_mode, alpha, out, rinv,
                                                                               reinterpret_cast<__half *>(out_hi),
                                                                               reinterpret_cast<__half *>(out_lo));
    SSL_LAUNCH_CHECK("rows_normalize_f16x3_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim,
                                const float *a_hat, const float *p_hat, float tau, float deno_eps, float *rowsum, float *obar,
                                float *loss_b, void *stream) {
    SSL_CHECK_ARG(rowsum_part && o_part && a_hat && p_hat && rowsum && obar && loss_b, "ssl_nce_finalize: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && n_split >= 1 && tau > 0.f, "ssl_nce_finalize: bad argument");
    if (batch == 0) return SSL_OK;
    nce_finalize_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(rowsum_part, o_part, n_split, batch, dim, a_hat, p_hat, tau, deno_eps, rowsum, obar, loss_b);
    SSL_LAUNCH_CHECK("nce_finalize_kernel");
    return SSL_OK;
}

extern "C" int ssl_lse_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim, float eps,
                                float *rowsum, float *obar, float *loss_b, void *stream) {
    SSL_CHECK_ARG(rowsum_part && o_part && rowsum && obar && loss_b, "ssl_lse_finalize: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && n_split >= 1, "ssl_lse_finalize: bad argument");
    if (batch == 0) return SSL_OK;
    lse_finalize_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(rowsum_part, o_part, n_split, batch, dim, eps, rowsum, obar, loss_b);
    SSL_LAUNCH_CHECK("lse_finalize_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_colscale(const float *rowsum, int64_t batch, const float *gscale, float scale, float *colscale, void *stream) {
    SSL_CHECK_ARG(rowsum && colscale, "ssl_nce_colscale: null argument");
    if (batch == 0) return SSL_OK;
    nce_colscale_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, STREAM>>>(rowsum, batch, gscale, scale, colscale);
    SSL_LAUNCH_CHECK("nce_colscale_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_colscale_live(const float *rowsum, int64_t batch, const int64_t *n_live, const float *gscale, float scale,
                                     float *colscale, void *stream) {
    SSL_CHECK_ARG(rowsum && colscale && n_live, "ssl_nce_colscale_live: null argument");
    SSL_CHECK_ARG(batch >= 0, "ssl_nce_colscale_live: batch %lld < 0", (long long)batch);
    if (batch == 0) return SSL_OK;
    nce_colscale_live_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, STREAM>>>(rowsum, batch, n_live, gscale, scale, colscale);
    SSL_LAUNCH_CHECK("nce_colscale_live_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_bwd_rows(const float *a_hat, const float *p_hat, const float *obar, const float *rinv1, const float *rinv2,
                                const int64_t *idx, int64_t batch, int32_t dim, float tau, const float *gscale, float scale,
                                float *g1, int64_t g1_stride, float *g2, int64_t g2_stride, void *stream) {
    SSL_CHECK_ARG(a_hat && p_hat && obar && idx, "ssl_nce_bwd_rows: null argument");
    SSL_CHECK_ARG((g1 == nullptr || rinv1) && (g2 == nullptr || rinv2), "ssl_nce_bwd_rows: rinv missing");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && tau > 0.f, "ssl_nce_bwd_rows: bad argument");
    if (batch == 0 || (g1 == nullptr && g2 == nullptr)) return SSL_OK;
    nce_bwd_rows_kernel<false><<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(a_hat, p_hat, obar, rinv1, rinv2, idx, batch, dim, tau, gscale, scale, g1, g1_stride, g2, g2_stride, nullptr);
    SSL_LAUNCH_CHECK("nce_bwd_rows_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_bwd_rows_live(const float *a_hat, const float *p_hat, const float *obar, const float *rinv1, const float *rinv2,
                                     const int64_t *idx, int64_t batch, const int64_t *n_live, int32_t dim, float tau, const float *gscale,
                                     float scale, float *g1, int64_t g1_stride, float *g2, int64_t g2_stride, void *stream) {
    SSL_CHECK_ARG(a_hat && p_hat && obar && idx && n_live, "ssl_nce_bwd_rows_live: null argument");
    SSL_CHECK_ARG((g1 == nullptr || rinv1) && (g2 == nullptr || rinv2), "ssl_nce_bwd_rows_live: rinv missing");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && tau > 0.f && batch >= 0, "ssl_nce_bwd_rows_live: bad argument");
    if (batch == 0 || (g1 == nullptr && g2 == nullptr)) return SSL_OK;
    nce_bwd_rows_kernel<true><<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(a_hat, p_hat, obar, rinv1, rinv2, idx, batch, dim, tau, gscale, scale, g1, g1_stride, g2, g2_stride, n_live);
    SSL_LAUNCH_CHECK("nce_bwd_rows_kernel");
    return SSL_OK;
}

extern "C" int ssl_nce_bwd_table(const float *dt_part, int32_t n_split, const float *t_hat, const float *rinv, int64_t n,
                                 int32_t dim, float *g_table, int64_t g_stride, int32_t accumulate, void *stream) {
    SSL_CHECK_ARG(dt_part && t_hat && rinv && g_table, "ssl_nce_bwd_table: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && n_split >= 1, "ssl_nce_bwd_table: bad argument");
    if (n == 0) return SSL_OK;
    nce_bwd_table_kernel<<<(unsigned)((n + 7) / 8), 256, 0, STREAM>>>(dt_part, n_split, t_hat, rinv, n, dim, g_table, g_stride, accumulate);
    SSL_LAUNCH_CHECK("nce_bwd_table_kernel");
    return SSL_OK;
}

namespace {
float *reduce_scratch(cudaStream_t) {
    // one scratch per device, allocated once; stream-ordered use only (single host thread per GPU)
    static thread_local float *buf[16] = {nullptr};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 16) return nullptr;
    if (!buf[dev]) cudaMalloc(&buf[dev], sizeof(float) * kRedBlocks);
    return buf[dev];
}
template <bool SQ>
int reduce_impl(const float *x, int64_t n, float alpha, float *out, cudaStream_t st, const char *name) {
    SSL_CHECK_ARG(x && out, "%s: null argument", name);
    SSL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0, "%s: input must be 16-byte aligned", name);
    float *part = reduce_scratch(st);
    if (!part) {
        ssl::set_error("%s: scratch allocation failed", name);
        return SSL_E_ALLOC;
    }
    int blocks = (int)std::min<int64_t>(kRedBlocks, std::max<int64_t>(1, (n / 4 + 255) / 256));
    reduce_stage1<SQ><<<blocks, 256, 0, st>>>(x, n, part);
    SSL_LAUNCH_CHECK("reduce_stage1");
    reduce_stage2<<<1, 1024, 0, st>>>(part, blocks, alpha, out);
    SSL_LAUNCH_CHECK("reduce_stage2");
    return SSL_OK;
}
}  // namespace

extern "C" int ssl_sumsq(const float *x, int64_t n, float *out, void *stream) { return reduce_impl<true>(x, n, 1.f, out, STREAM, "ssl_sumsq"); }
extern "C" int ssl_sum(const float *x, int64_t n, float alpha, float *out, void *stream) { return reduce_impl<false>(x, n, alpha, out, STREAM, "ssl_sum"); }
extern "C" int ssl_sum_live(const float *x, int64_t n, const int64_t *n_live, float alpha, float *out, void *stream) {
    SSL_CHECK_ARG(x && n_live && out, "ssl_sum_live: null argument");
    SSL_CHECK_ARG(n >= 0, "ssl_sum_live: n %lld < 0", (long long)n);
    sum_live_kernel<<<1, 1024, 0, STREAM>>>(x, n, n_live, alpha, out);
    SSL_LAUNCH_CHECK("sum_live_kernel");
    return SSL_OK;
}

extern "C" int ssl_axpy(const float *x, float *y, int64_t n, const float *gscale, float alpha, void *stream) {
    SSL_CHECK_ARG(x && y, "ssl_axpy: null argument");
    SSL_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, "ssl_axpy: pointers must be 16-byte aligned");
    if (n == 0) return SSL_OK;
    const int blocks = (int)std::min<int64_t>(ssl::kNumSM * 8, (n / 4 + 255) / 256 + 1);
    axpy_kernel<<<blocks, 256, 0, STREAM>>>(x, y, n, gscale, alpha);
    SSL_LAUNCH_CHECK("axpy_kernel");
    return SSL_OK;
}

static int adam_launch(float *p, float *const *p_peers, int32_t n_peers, const float *g, float *m, float *v, int64_t n, int64_t step,
                       const int64_t *step_dev, float *scratch2, double lr, double beta1, double beta2, double eps, double weight_decay, void *stream) {
    SSL_CHECK_ARG(p && g && m && v && (step >= 1 || (step_dev != nullptr && scratch2 != nullptr)), "ssl_adam_step: bad argument");
    SSL_CHECK_ARG(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0,
                  "ssl_adam_step: pointers must be 16-byte aligned");
    SSL_CHECK_ARG(n_peers >= 0 && n_peers <= SSL_MAX_PEERS && (n_peers == 0 || p_peers != nullptr), "ssl_adam_step_peers: bad peer list");
    PeerPtrs peers{};
    peers.n = n_peers;
    for (int q = 0; q < n_peers; ++q) {
        SSL_CHECK_ARG(p_peers[q] != nullptr && (reinterpret_cast<uintptr_t>(p_peers[q]) & 15) == 0, "ssl_adam_step_peers: peer pointer %d null or unaligned", q);
        peers.p[q] = p_peers[q];
    }
    if (n == 0) return SSL_OK;
    float step_size = 0.f, inv_bc2_sqrt = 0.f;
    if (step_dev == nullptr) {
        const double bc1 = 1.0 - std::pow(beta1, (double)step);
        const double bc2 = 1.0 - std::pow(beta2, (double)step);
        step_size = (float)(lr / bc1);
        inv_bc2_sqrt = (float)(1.0 / std::sqrt(bc2));
    } else {
        adam_prepare_kernel<<<1, 1, 0, STREAM>>>(step_dev, lr, beta1, beta2, scratch2);
        SSL_LAUNCH_CHECK("adam_prepare_kernel");
    }
    const int blocks = (int)std::min<int64_t>(ssl::kNumSM * 8, (n / 4 + 255) / 256 + 1);
    const AdamK k{(float)beta1, (float)beta2, (float)(1.0 - beta1), (float)(1.0 - beta2), step_size, inv_bc2_sqrt, (float)eps, (float)weight_decay};
    adam_kernel<<<blocks, 256, 0, STREAM>>>(p, g, m, v, n, k, peers, step_dev != nullptr ? scratch2 : nullptr);
    SSL_LAUNCH_CHECK("adam_kernel");
    return SSL_OK;
}

extern "C" int ssl_adam_step_peers(float *p, float *const *p_peers, int32_t n_peers, const float *g, float *m, float *v, int64_t n,
                                   int64_t step, double lr, double beta1, double beta2, double eps, double weight_decay, void *stream) {
    SSL_CHECK_ARG(step >= 1, "ssl_adam_step: step must be >= 1");
    return adam_launch(p, p_peers, n_peers, g, m, v, n, step, nullptr, nullptr, lr, beta1, beta2, eps, weight_decay, stream);
}

extern "C" int ssl_adam_step_dev(float *p, float *const *p_peers, int32_t n_peers, const float *g, float *m, float *v, int64_t n,
                                 const int64_t *step_dev, float *scratch2, double lr, double beta1, double beta2, double eps, double weight_decay,
                                 void *stream) {
    SSL_CHECK_ARG(step_dev != nullptr && scratch2 != nullptr, "ssl_adam_step_dev: step_dev / scratch2 is null");
    return adam_launch(p, p_peers, n_peers, g, m, v, n, 0, step_dev, scratch2, lr, beta1, beta2, eps, weight_decay, stream);
}

extern "C" int ssl_adam_step(float *p, const float *g, float *m, float *v, int64_t n, int64_t step, double lr, double beta1,
                             double beta2, double eps, double weight_decay, void *stream) {
    return ssl_adam_step_peers(p, nullptr, 0, g, m, v, n, step, lr, beta1, beta2, eps, weight_decay, stream);
}

extern "C" int ssl_predict_mask(const float *users_tab, int64_t u_stride, const float *items_tab, int64_t i_stride,
                                const int64_t *users, int64_t n_b, int64_t n_item, int32_t dim, const int64_t *mask_dense,
                                const int32_t *trn_rowptr, const int32_t *trn_cols, float *preds, void *stream) {
    SSL_CHECK_ARG(users_tab && items_tab && users && preds, "ssl_predict_mask: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_predict_mask: dim %d out of range", dim);
    SSL_CHECK_ARG(n_b <= 65535, "ssl_predict_mask: at most 65535 users per call");
    if (n_b == 0 || n_item == 0) return SSL_OK;
    if (ssl::g_predict_tiled) {      // default: 128 x 128 score tiles, every item row read once per 128 users (predict_tile.cuh)
        namespace P = ssl_predict;
        dim3 grid((unsigned)((n_item + P::TN - 1) / P::TN), (unsigned)((n_b + P::TM - 1) / P::TM));
        P::predict_tile_kernel<<<grid, P::NT, 0, STREAM>>>(users_tab, u_stride, items_tab, i_stride, users, n_b, n_item, dim, mask_dense, trn_rowptr,
                                                          trn_cols, preds);
        SSL_LAUNCH_CHECK("predict_tile_kernel");
        return SSL_OK;
    }
    // ssl_set_option("predict_tiled", 0): the round-1 kernel (one warp per (user, item) dot product), kept as the cross-check
    dim3 grid((unsigned)((n_item + 1023) / 1024), (unsigned)n_b);
    predict_mask_kernel<<<grid, 256, 0, STREAM>>>(users_tab, u_stride, items_tab, i_stride, users, n_item, dim, mask_dense, trn_rowptr, trn_cols, preds);
    SSL_LAUNCH_CHECK("predict_mask_kernel");
    return SSL_OK;
}
