// HCCF's hyper-graph branch (models/general_cf/hccf.py:43-49,100-108) and its backward, without library GEMMs:
//
//   A   = E_side W mult                         [n, H]   incidence of the side's nodes to the H hyper-edges (:43-44)
//   H_k = dropout(A)                            [n, H]   fresh mask per layer (:48-49), kept values / keep
//   lat = act(H_k^T X)                          [H, d]   (:105)         act = LeakyReLU(slope)
//   Y   = act(H_k lat)                          [n, d]   (:106)
//
// Every product is skinny: one dimension is the node count n (80 k at the amazon shape), the other two are d <= 128 and
// H <= 128.  Two kernel shapes cover the forward and the backward:
//   rowgemm  Out[r, :] (op)= post( In1[r, :] M1 + In2[r, :] M2 )      -- row-local; the small matrices live in shared memory
//   colgemm  Part[cta]      = sum_r In1[r, :]^T (x) In2[r, :]          -- a reduction over the rows; per-CTA partials are
//                                                                         reduced in a fixed order by colgemm_finalize
// with the LeakyReLU derivative folded into the loads (dZ = dY * act'(Y)) and into the finalize (dlat = . * act'(lat)).
// FP32 FMA: at H = 128, d = 64 a row costs 16 k MACs per product against ~1 KB of traffic, i.e. the kernels sit between the
// FMA and the HBM roof and are far from dominant (the step's contraction is the InfoNCE term); bit-reproducible (no atomics).
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int TR = 64;            // rows per tile
constexpr int kT = 256;           // threads per CTA
constexpr int kMaxK = 128;        // inner / outer sizes (dim, hyper_num) up to 128

struct RowGemmArgs {
    const float *in1; int64_t in1_stride; int k1;
    const float *m1; int m1_trans;               // M1 [k1, n_out] row-major, or (trans) [n_out, k1]
    const float *in2; int64_t in2_stride; int k2;
    const float *m2; int m2_trans;
    const float *pre_ref; int64_t pre_stride; float pre_slope;   // optional: in1[r, j] *= (pre_ref[r, j] > 0 ? 1 : pre_slope)   (dZ = dY * act'(Y))
    float *out; int64_t out_stride; int n_out;
    float scale, slope;                          // out = leaky(acc * scale, slope); slope = 1: no activation
    int accumulate;                              // out += instead of out =
    int64_t n_rows;
    int vec;                                     // inputs allow 16-byte loads
    int vec_out;                                 // out allows 16-byte stores
};

__device__ __forceinline__ float leaky(float x, float slope) { return x > 0.f ? x : x * slope; }

// shared layout: M [K][NO] (row-major after the optional transpose), In tile [TR][K + 1] (padded).
// thread -> 4 rows x CPT contiguous columns of the [TR x NO] output tile (NO <= 16 * CPT)
template <int CPT>
__global__ void __launch_bounds__(kT) rowgemm_kernel(RowGemmArgs a) {
    extern __shared__ float sm[];
    const int K = a.k1 + a.k2, NO = a.n_out;
    const int ldm = 16 * CPT;                     // padded row of M (columns >= NO are zero)
    float *s_m = sm;                              // [K][ldm]
    float *s_in = sm + (size_t)K * ldm;           // [TR][K + 1]
    const int ldi = K + 1;
    // stage M1 | M2 as [K][ldm] (zero padded): global reads run along the SOURCE's fastest dimension in either orientation
    for (int i = threadIdx.x; i < K * (ldm - NO); i += kT) s_m[(i / (ldm - NO)) * ldm + NO + i % (ldm - NO)] = 0.f;
    for (int part = 0; part < 2; ++part) {
        const float *m = part ? a.m2 : a.m1;
        const int kk = part ? a.k2 : a.k1, k0 = part ? a.k1 : 0, trans = part ? a.m2_trans : a.m1_trans;
        if (m == nullptr || kk == 0) continue;
        if (trans) {            // m [NO][kk]
            for (int i = threadIdx.x; i < NO * kk; i += kT) {
                const int c = i / kk, k = i - c * kk;
                s_m[(size_t)(k0 + k) * ldm + c] = __ldg(m + i);
            }
        } else {                // m [kk][NO]
            for (int i = threadIdx.x; i < kk * NO; i += kT) {
                const int k = i / NO, c = i - k * NO;
                s_m[(size_t)(k0 + k) * ldm + c] = __ldg(m + i);
            }
        }
    }
    const int tc = threadIdx.x % 16, tr = threadIdx.x / 16;       // 16 column groups x 16 row groups (4 rows each)
    const int64_t n_tiles = (a.n_rows + TR - 1) / TR;
    const bool vec = a.vec != 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int64_t r0 = t * TR;
        __syncthreads();
        if (vec) {          // 16-byte global loads (rows are 16-byte aligned and k1, k2 multiples of 4)
            const int q1 = a.k1 >> 2, q2 = a.k2 >> 2;
            for (int i = threadIdx.x; i < TR * q1; i += kT) {
                const int r = i / q1, k = (i - r * q1) * 4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (r0 + r < a.n_rows) {
                    v = ssl::ldg4(a.in1 + (r0 + r) * a.in1_stride + k);
                    if (a.pre_ref != nullptr) {
                        const float4 y = ssl::ldg4(a.pre_ref + (r0 + r) * a.pre_stride + k);
                        v.x *= (y.x > 0.f) ? 1.f : a.pre_slope; v.y *= (y.y > 0.f) ? 1.f : a.pre_slope;
                        v.z *= (y.z > 0.f) ? 1.f : a.pre_slope; v.w *= (y.w > 0.f) ? 1.f : a.pre_slope;
                    }
                }
                float *d = s_in + r * ldi + k;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
            for (int i = threadIdx.x; i < TR * q2; i += kT) {
                const int r = i / q2, k = (i - r * q2) * 4;
                const float4 v = (r0 + r < a.n_rows) ? ssl::ldg4(a.in2 + (r0 + r) * a.in2_stride + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                float *d = s_in + r * ldi + a.k1 + k;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        } else {
            for (int i = threadIdx.x; i < TR * a.k1; i += kT) {
                const int r = i / a.k1, k = i % a.k1;
                float v = 0.f;
                if (r0 + r < a.n_rows) {
                    v = __ldg(a.in1 + (r0 + r) * a.in1_stride + k);
                    if (a.pre_ref != nullptr) v *= (__ldg(a.pre_ref + (r0 + r) * a.pre_stride + k) > 0.f) ? 1.f : a.pre_slope;
                }
                s_in[r * ldi + k] = v;
            }
            for (int i = threadIdx.x; i < TR * a.k2; i += kT) {
                const int r = i / a.k2, k = i % a.k2;
                s_in[r * ldi + a.k1 + k] = (r0 + r < a.n_rows) ? __ldg(a.in2 + (r0 + r) * a.in2_stride + k) : 0.f;
            }
        }
        __syncthreads();
        float acc[4][CPT];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < CPT; ++j) acc[i][j] = 0.f;
#pragma unroll 4
        for (int k = 0; k < K; ++k) {
            float x[4], m[CPT];
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = s_in[(tr * 4 + i) * ldi + k];
            const float *mr = s_m + (size_t)k * ldm + tc * CPT;
            if constexpr (CPT % 4 == 0) {
#pragma unroll
                for (int j = 0; j < CPT; j += 4) {
                    const float4 v = *reinterpret_cast<const float4 *>(mr + j);
                    m[j] = v.x; m[j + 1] = v.y; m[j + 2] = v.z; m[j + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int j = 0; j < CPT; ++j) m[j] = mr[j];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < CPT; ++j) acc[i][j] = fmaf(x[i], m[j], acc[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t r = r0 + tr * 4 + i;
            if (r >= a.n_rows) continue;
            if constexpr (CPT % 4 == 0) {
                if (a.vec_out && tc * CPT + CPT <= NO) {          // 16-byte stores: CPT contiguous columns of this thread
#pragma unroll
                    for (int j = 0; j < CPT; j += 4) {
                        float4 *o = reinterpret_cast<float4 *>(a.out + r * a.out_stride + tc * CPT + j);
                        float4 v = make_float4(leaky(acc[i][j] * a.scale, a.slope), leaky(acc[i][j + 1] * a.scale, a.slope),
                                               leaky(acc[i][j + 2] * a.scale, a.slope), leaky(acc[i][j + 3] * a.scale, a.slope));
                        if (a.accumulate) ssl::add4(v, *o);
                        *o = v;
                    }
                    continue;
                }
            }
#pragma unroll
            for (int j = 0; j < CPT; ++j) {
                const int c = tc * CPT + j;
                if (c >= NO) break;
                float *o = a.out + r * a.out_stride + c;
                const float v = leaky(acc[i][j] * a.scale, a.slope);
                *o = a.accumulate ? (*o + v) : v;
            }
        }
    }
}

struct ColGemmArgs {
    const float *in1; int64_t in1_stride; int k1;     // Part[k1, k2] = sum_r in1[r, :]^T (x) in2[r, :]
    const float *in2; int64_t in2_stride; int k2;
    const float *pre_ref; int64_t pre_stride;         // optional: in2[r, j] *= (pre_ref[r, j] > 0 ? 1 : slope)
    float slope;
    float *part;                                       // [gridDim.x, k1, k2]
    int64_t n_rows;
    int vec;                                           // inputs allow 16-byte loads
};

// thread -> N1 x N2 outputs: k1 = t1 * N1 + i, k2 = t2 * N2 + j (K1 <= 16 * N1, K2 <= 16 * N2; the shared rows are zero-padded)
template <int N1, int N2>
__global__ void __launch_bounds__(kT) colgemm_kernel(ColGemmArgs a) {
    extern __shared__ float sm[];
    const int K1 = a.k1, K2 = a.k2;
    constexpr int L1 = 16 * N1, L2 = 16 * N2;
    float *s1 = sm;                          // [TR][L1]
    float *s2 = sm + (size_t)TR * L1;        // [TR][L2]
    const int t1 = threadIdx.x / 16, t2 = threadIdx.x % 16;
    float acc[N1][N2];
#pragma unroll
    for (int i = 0; i < N1; ++i)
#pragma unroll
        for (int j = 0; j < N2; ++j) acc[i][j] = 0.f;
    const int64_t n_tiles = (a.n_rows + TR - 1) / TR;
    // contiguous chunk of tiles per CTA: the summation order of every output is fixed by (grid, n_rows) alone
    const int64_t per = (n_tiles + gridDim.x - 1) / gridDim.x;
    const int64_t tlo = (int64_t)blockIdx.x * per, thi = min(n_tiles, tlo + per);
    for (int64_t t = tlo; t < thi; ++t) {
        const int64_t r0 = t * TR;
        __syncthreads();
        if (a.vec) {        // 16-byte global loads and shared stores (K1, K2 multiples of 4, rows 16-byte aligned)
            for (int i = threadIdx.x; i < TR * (L1 / 4); i += kT) {
                const int r = i / (L1 / 4), k = (i % (L1 / 4)) * 4;
                const float4 v = (k < K1 && r0 + r < a.n_rows) ? ssl::ldg4(a.in1 + (r0 + r) * a.in1_stride + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                *reinterpret_cast<float4 *>(s1 + r * L1 + k) = v;
            }
            for (int i = threadIdx.x; i < TR * (L2 / 4); i += kT) {
                const int r = i / (L2 / 4), k = (i % (L2 / 4)) * 4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (k < K2 && r0 + r < a.n_rows) {
                    v = ssl::ldg4(a.in2 + (r0 + r) * a.in2_stride + k);
                    if (a.pre_ref != nullptr) {
                        const float4 y = ssl::ldg4(a.pre_ref + (r0 + r) * a.pre_stride + k);
                        v.x *= (y.x > 0.f) ? 1.f : a.slope; v.y *= (y.y > 0.f) ? 1.f : a.slope;
                        v.z *= (y.z > 0.f) ? 1.f : a.slope; v.w *= (y.w > 0.f) ? 1.f : a.slope;
                    }
                }
                *reinterpret_cast<float4 *>(s2 + r * L2 + k) = v;
            }
        } else {
            for (int i = threadIdx.x; i < TR * L1; i += kT) {
                const int r = i / L1, k = i % L1;
                s1[i] = (k < K1 && r0 + r < a.n_rows) ? __ldg(a.in1 + (r0 + r) * a.in1_stride + k) : 0.f;
            }
            for (int i = threadIdx.x; i < TR * L2; i += kT) {
                const int r = i / L2, k = i % L2;
                float v = 0.f;
                if (k < K2 && r0 + r < a.n_rows) {
                    v = __ldg(a.in2 + (r0 + r) * a.in2_stride + k);
                    if (a.pre_ref != nullptr) v *= (__ldg(a.pre_ref + (r0 + r) * a.pre_stride + k) > 0.f) ? 1.f : a.slope;
                }
                s2[i] = v;
            }
        }
        __syncthreads();
#pragma unroll 2
        for (int r = 0; r < TR; ++r) {
            float x[N1], y[N2];
            const float *p1 = s1 + r * L1 + t1 * N1, *p2 = s2 + r * L2 + t2 * N2;
            if constexpr (N1 % 4 == 0) {
#pragma unroll
                for (int i = 0; i < N1; i += 4) {
                    const float4 v = *reinterpret_cast<const float4 *>(p1 + i);
                    x[i] = v.x; x[i + 1] = v.y; x[i + 2] = v.z; x[i + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int i = 0; i < N1; ++i) x[i] = p1[i];
            }
            if constexpr (N2 % 4 == 0) {
#pragma unroll
                for (int j = 0; j < N2; j += 4) {
                    const float4 v = *reinterpret_cast<const float4 *>(p2 + j);
                    y[j] = v.x; y[j + 1] = v.y; y[j + 2] = v.z; y[j + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int j = 0; j < N2; ++j) y[j] = p2[j];
            }
#pragma unroll
            for (int i = 0; i < N1; ++i)
#pragma unroll
                for (int j = 0; j < N2; ++j) acc[i][j] = fmaf(x[i], y[j], acc[i][j]);
        }
    }
    float *p = a.part + (size_t)blockIdx.x * K1 * K2;
#pragma unroll
    for (int i = 0; i < N1; ++i) {
        const int k1 = t1 * N1 + i;
        if (k1 >= K1) break;
#pragma unroll
        for (int j = 0; j < N2; ++j) {
            const int k2 = t2 * N2 + j;
            if (k2 < K2) p[(size_t)k1 * K2 + k2] = acc[i][j];
        }
    }
}

// out[e] = post(sum_c part[c, e]);  post: * scale, then mode 0: identity (and out_act = leaky(out));
//                                          mode 1: * (ref[e] > 0 ? 1 : slope)   (derivative of the activation at the saved pre-activation)
// block = 32 elements x 8 lanes over the partials: lane l adds partials l, l + 8, ... in order, the 8 lane sums are added in lane
// order -- a fixed summation order for every element (bit-reproducible), 8-way parallel, 128-byte coalesced reads
__global__ void __launch_bounds__(256) colgemm_finalize_kernel(const float *__restrict__ part, int n_part, int64_t n_elem, float scale, int mode,
                                                               float slope, const float *__restrict__ ref, float *__restrict__ out,
                                                               float *__restrict__ out_act) {
    __shared__ float sh[8][33];
    const int ex = threadIdx.x & 31, lane = threadIdx.x >> 5;
    const int64_t e = (int64_t)blockIdx.x * 32 + ex;
    float s = 0.f;
    if (e < n_elem)
        for (int c = lane; c < n_part; c += 8) s += part[(size_t)c * n_elem + e];
    sh[lane][ex] = s;
    __syncthreads();
    if (lane != 0 || e >= n_elem) return;
    s = sh[0][ex];
#pragma unroll
    for (int l = 1; l < 8; ++l) s += sh[l][ex];
    s *= scale;
    if (mode == 1) s *= (ref[e] > 0.f) ? 1.f : slope;
    out[e] = s;
    if (out_act != nullptr) out_act[e] = leaky(s, slope);
}

// dropout of the incidence, forward (out = a * keep / p) and backward (out += g * keep / p); keep test: floor(U + p) as torch's
// Bernoulli(p) mask of F.dropout -- the in-kernel draw is keyed by (seed, stream; row, 4-column group)
__global__ void hyper_dropout_kernel(const float *__restrict__ x, float *__restrict__ out, int64_t n, int h, float keep, int mode,
                                     const float *__restrict__ mask, uint64_t seed, const uint64_t *__restrict__ seed_ptr, uint32_t stream, int accumulate) {
    const int quads = h / 4;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * quads) return;
    const int64_t r = i / quads;
    const int q = (int)(i % quads);
    float4 v = ssl::ldg4(x + r * h + q * 4);
    float4 k;
    if (mode == 2) k = ssl::ldg4(mask + r * h + q * 4);
    else {
        const uint4 u = ssl::philox4x32_10(make_uint4((uint32_t)r, (uint32_t)q, stream, 0x48595052u /*"HYPR"*/),
                                           ssl::seed_key(seed_ptr != nullptr ? __ldg(seed_ptr) : seed));
        k = make_float4(ssl::u01(u.x) + keep >= 1.f ? 1.f : 0.f, ssl::u01(u.y) + keep >= 1.f ? 1.f : 0.f,
                        ssl::u01(u.z) + keep >= 1.f ? 1.f : 0.f, ssl::u01(u.w) + keep >= 1.f ? 1.f : 0.f);
    }
    const float inv = 1.f / keep;
    v = make_float4(v.x * k.x * inv, v.y * k.y * inv, v.z * k.z * inv, v.w * k.w * inv);
    float4 *o = reinterpret_cast<float4 *>(out + r * h + q * 4);
    if (accumulate) {
        float4 c = *o;
        ssl::add4(c, v);
        *o = c;
    } else *o = v;
}

bool ok_dim(int k) { return k >= 4 && k <= kMaxK; }
int round_n(int k) { const int c = (k + 15) / 16; return c <= 1 ? 1 : (c <= 2 ? 2 : (c <= 4 ? 4 : 8)); }   // outputs per thread: 1, 2, 4, 8

template <int CPT>
int launch_rowgemm(const RowGemmArgs &a, cudaStream_t st) {
    const int K = a.k1 + a.k2;
    const size_t smem = sizeof(float) * ((size_t)K * 16 * CPT + (size_t)TR * (K + 1));
    static bool configured[64] = {};
    int dev = 0;
    SSL_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        SSL_CUDA(cudaFuncSetAttribute(rowgemm_kernel<CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)(sizeof(float) * (2 * kMaxK * 16 * CPT + TR * (2 * kMaxK + 1)))));
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    const int64_t n_tiles = (a.n_rows + TR - 1) / TR;
    const int grid = (int)std::min<int64_t>(n_tiles, 2 * ssl::kNumSM);
    rowgemm_kernel<CPT><<<grid, kT, smem, st>>>(a);
    SSL_LAUNCH_CHECK("rowgemm_kernel");
    return SSL_OK;
}

template <int N1, int N2>
int launch_colgemm(const ColGemmArgs &a, int grid, cudaStream_t st) {
    const size_t smem = sizeof(float) * (size_t)TR * 16 * (N1 + N2);
    static bool configured[64] = {};
    int dev = 0;
    SSL_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        SSL_CUDA(cudaFuncSetAttribute(colgemm_kernel<N1, N2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    colgemm_kernel<N1, N2><<<grid, kT, smem, st>>>(a);
    SSL_LAUNCH_CHECK("colgemm_kernel");
    return SSL_OK;
}

template <int N1>
int launch_colgemm1(const ColGemmArgs &a, int n2, int grid, cudaStream_t st) {
    switch (n2) {
        case 1: return launch_colgemm<N1, 1>(a, grid, st);
        case 2: return launch_colgemm<N1, 2>(a, grid, st);
        case 4: return launch_colgemm<N1, 4>(a, grid, st);
        default: return launch_colgemm<N1, 8>(a, grid, st);
    }
}

}  // namespace

extern "C" int ssl_rowgemm(const float *in1, int64_t in1_stride, int32_t k1, const float *m1, int32_t m1_trans, const float *in2,
                           int64_t in2_stride, int32_t k2, const float *m2, int32_t m2_trans, const float *pre_ref, int64_t pre_stride,
                           float pre_slope, float *out, int64_t out_stride, int32_t n_out, float scale, float slope, int32_t accumulate, int64_t n_rows,
                           void *stream) {
    // no rows: the row pointers may be null (torch gives an empty tensor data_ptr() == 0)
    SSL_CHECK_ARG(n_rows >= 0 && m1 && (n_rows == 0 || (in1 && out)), "ssl_rowgemm: null argument or n_rows < 0");
    SSL_CHECK_ARG(ok_dim(k1) && (in2 == nullptr ? true : (ok_dim(k2) && m2 != nullptr)), "ssl_rowgemm: inner sizes out of range (4..128)");
    SSL_CHECK_ARG(ok_dim(n_out), "ssl_rowgemm: n_out %d out of range (4..128)", n_out);
    if (n_rows == 0) return SSL_OK;
    auto al16 = [](const void *p, int64_t stride) { return p == nullptr || ((reinterpret_cast<uintptr_t>(p) & 15) == 0 && stride % 4 == 0); };
    const int vec = (k1 % 4 == 0 && (in2 == nullptr || k2 % 4 == 0) && al16(in1, in1_stride) && al16(in2, in2_stride) && al16(pre_ref, pre_stride)) ? 1 : 0;
    RowGemmArgs a{in1, in1_stride, k1, m1, m1_trans, in2, in2_stride, in2 ? k2 : 0, m2, m2_trans, pre_ref, pre_stride, pre_slope, out, out_stride, n_out,
                  scale, slope, accumulate, n_rows, vec, al16(out, out_stride) ? 1 : 0};
    cudaStream_t st = (cudaStream_t)stream;
    switch (round_n(n_out)) {
        case 1: return launch_rowgemm<1>(a, st);
        case 2: return launch_rowgemm<2>(a, st);
        case 4: return launch_rowgemm<4>(a, st);
        default: return launch_rowgemm<8>(a, st);
    }
}

extern "C" int ssl_colgemm_parts(int64_t n_rows) {
    const int64_t n_tiles = (n_rows + TR - 1) / TR;
    return (int)std::max<int64_t>(1, std::min<int64_t>(n_tiles, 3 * ssl::kNumSM));
}

extern "C" int ssl_colgemm(const float *in1, int64_t in1_stride, int32_t k1, const float *in2, int64_t in2_stride, int32_t k2,
                           const float *pre_ref, int64_t pre_stride, float slope, int64_t n_rows, float *part, float scale, int32_t mode,
                           const float *ref, float *out, float *out_act, void *stream) {
    // no rows: in1 / in2 may be null; the one partial is zero, so out = 0 and out_act = leaky(0)
    SSL_CHECK_ARG(n_rows >= 0 && part && out && (n_rows == 0 || (in1 && in2)), "ssl_colgemm: null argument or n_rows < 0");
    SSL_CHECK_ARG(ok_dim(k1) && ok_dim(k2), "ssl_colgemm: sizes %d x %d out of range (4..128)", k1, k2);
    SSL_CHECK_ARG(mode == 0 || (mode == 1 && ref != nullptr), "ssl_colgemm: mode 1 needs ref");
    const int grid = ssl_colgemm_parts(n_rows);
    auto al16 = [](const void *p, int64_t stride) { return p == nullptr || ((reinterpret_cast<uintptr_t>(p) & 15) == 0 && stride % 4 == 0); };
    const int vec = (k1 % 4 == 0 && k2 % 4 == 0 && al16(in1, in1_stride) && al16(in2, in2_stride) && al16(pre_ref, pre_stride)) ? 1 : 0;
    ColGemmArgs a{in1, in1_stride, k1, in2, in2_stride, k2, pre_ref, pre_stride, slope, part, n_rows, vec};
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    switch (round_n(k1)) {
        case 1: rc = launch_colgemm1<1>(a, round_n(k2), grid, st); break;
        case 2: rc = launch_colgemm1<2>(a, round_n(k2), grid, st); break;
        case 4: rc = launch_colgemm1<4>(a, round_n(k2), grid, st); break;
        default: rc = launch_colgemm1<8>(a, round_n(k2), grid, st); break;
    }
    if (rc != SSL_OK) return rc;
    const int64_t n_elem = (int64_t)k1 * k2;
    colgemm_finalize_kernel<<<(unsigned)((n_elem + 31) / 32), 256, 0, st>>>(part, grid, n_elem, scale, mode, slope, ref, out, out_act);
    SSL_LAUNCH_CHECK("colgemm_finalize_kernel");
    return SSL_OK;
}

static int hyper_dropout_launch(const float *x, float *out, int64_t n, int32_t h, float keep, int32_t mode, const float *mask, uint64_t seed,
                                const uint64_t *seed_ptr, uint32_t stream_id, int32_t accumulate, void *stream) {
    // no rows: x, out and mask may be null
    SSL_CHECK_ARG(n >= 0 && (n == 0 || (x && out)) && h >= 4 && h % 4 == 0 && keep > 0.f && keep <= 1.f, "ssl_hyper_dropout: bad argument");
    SSL_CHECK_ARG(mode == 1 || (mode == 2 && (mask != nullptr || n == 0)),
                  "ssl_hyper_dropout: mode 1 (in-kernel draw) or 2 (injected [n, h] float keep mask)");
    const int64_t total = n * (h / 4);
    if (total == 0) return SSL_OK;
    hyper_dropout_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, out, n, h, keep, mode, mask, seed, seed_ptr, stream_id, accumulate);
    SSL_LAUNCH_CHECK("hyper_dropout_kernel");
    return SSL_OK;
}

extern "C" int ssl_hyper_dropout(const float *x, float *out, int64_t n, int32_t h, float keep, int32_t mode, const float *mask, uint64_t seed,
                                 uint32_t stream_id, int32_t accumulate, void *stream) {
    return hyper_dropout_launch(x, out, n, h, keep, mode, mask, seed, nullptr, stream_id, accumulate, stream);
}

extern "C" int ssl_hyper_dropout_dev(const float *x, float *out, int64_t n, int32_t h, float keep, int32_t mode, const float *mask,
                                     const uint64_t *seed_ptr, uint32_t stream_id, int32_t accumulate, void *stream) {
    SSL_CHECK_ARG(mode == 2 || seed_ptr != nullptr, "ssl_hyper_dropout_dev: seed_ptr is null");
    return hyper_dropout_launch(x, out, n, h, keep, mode, mask, 0, seed_ptr, stream_id, accumulate, stream);
}
