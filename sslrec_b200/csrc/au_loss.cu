// DirectAU's alignment / uniformity losses (models/loss_utils.py:75-86) on unit rows produced by
// ssl_rows_normalize(norm_mode 2 = F.normalize).  The B x B pair sum of the uniformity term is the
// softmax contraction of nce_gemm*.cu with R = C = x^ (e_ij = exp(4 x^_i.x^_j - 4) = exp(-2 |x^_i - x^_j|^2));
// the kernels here are its epilogue, the direct pair sum used below 256 rows, the row-wise alignment
// term and the shared backward through the normalisation.  One warp per row, lanes over the dim.
#include "common.cuh"

namespace {

constexpr int kMaxPerLane = SSL_MAX_DIM / 32;

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

// loss_b[b] = |x^_b - y^_b|^2   (alignment with alpha = 2: norm(p=2).pow(2), loss_utils.py:79)
__global__ void align_fwd_kernel(const float *xhat, const float *yhat, int64_t batch, int dim, float *loss_b) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float x[kMaxPerLane], y[kMaxPerLane];
    load_row(xhat + b * dim, dim, lane, x);
    load_row(yhat + b * dim, dim, lane, y);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) x[i] -= y[i];
    const float s = dot_rows(x, x);
    if (lane == 0) loss_b[b] = s;
}

// Epilogue of the pair contraction: reduce the split partials, remove the i == j term
// (pdist runs over i < j only): pair_sum[i] = sum_{j != i} e_ij,  w[i,:] = sum_{j != i} e_ij x^_j.
// r_scaled = x^ * 4 log2(e) is the row operand the contraction used, offset = 4 log2(e).
__global__ void uniform_finalize_kernel(const float *rowsum_part, const float *o_part, int n_split, int64_t batch, int dim,
                                        const float *r_scaled, const float *xhat, float offset, float *pair_sum, float *w) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float rs = 0.f;
    for (int s = 0; s < n_split; ++s) rs += rowsum_part[(size_t)s * batch + b];
    float o[kMaxPerLane] = {0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < n_split; ++s) {
        const float *src = o_part + ((size_t)s * batch + b) * dim;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int k = lane + 32 * i;
            if (k < dim) o[i] += src[k];
        }
    }
    float r[kMaxPerLane], x[kMaxPerLane];
    load_row(r_scaled + b * dim, dim, lane, r);
    load_row(xhat + b * dim, dim, lane, x);
    const float e_ii = exp2f(dot_rows(r, x) - offset);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) w[b * dim + k] = o[i] - e_ii * x[i];
    }
    if (lane == 0) pair_sum[b] = rs - e_ii;
}

// Direct pair sums for small batches: the same pair_sum / w as uniform_finalize_kernel, but e_ij = exp(-2 |x^_i - x^_j|^2)
// from the difference vector over j != i in increasing order, as pdist does.  rowsum - e_ii cancels when the off-diagonal
// sum is small next to e_ii = 1 (B = 2-3, near-antipodal rows); this form has no such cancellation.  O(B^2 d) work.
__global__ void uniform_pairs_kernel(const float *xhat, int64_t batch, int dim, float *pair_sum, float *w) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    float x[kMaxPerLane], y[kMaxPerLane], df[kMaxPerLane], o[kMaxPerLane] = {0.f, 0.f, 0.f, 0.f};
    load_row(xhat + b * dim, dim, lane, x);
    float ps = 0.f;
    for (int64_t j = 0; j < batch; ++j) {
        if (j == b) continue;
        load_row(xhat + j * dim, dim, lane, y);
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) df[i] = x[i] - y[i];
        const float e = expf(-2.f * dot_rows(df, df));
        ps += e;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) o[i] = fmaf(e, y[i], o[i]);
    }
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) w[b * dim + k] = o[i];
    }
    if (lane == 0) pair_sum[b] = ps;
}

// dx^_b = g (c1 d1_b + c2 d2_b), g = scale * (*gscale); through x^ = x * rinv:
// de_b = rinv_b (dx^_b - x^_b (x^_b . dx^_b)), added to row idx[b] of the gradient view.
__global__ void unit_rows_bwd_kernel(const float *xhat, const float *rinv, const int64_t *idx, int64_t batch, int dim,
                                     const float *d1, float c1, const float *d2, float c2, const float *gscale, float scale,
                                     float *g_out, int64_t g_stride) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    const float g = scale * (gscale ? __ldg(gscale) : 1.f);
    float x[kMaxPerLane], d[kMaxPerLane], t[kMaxPerLane];
    load_row(xhat + b * dim, dim, lane, x);
    load_row(d1 + b * dim, dim, lane, d);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) d[i] *= g * c1;
    if (d2 != nullptr) {
        load_row(d2 + b * dim, dim, lane, t);
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) d[i] = fmaf(g * c2, t[i], d[i]);
    }
    const float proj = dot_rows(x, d);
    const float ri = rinv[b];
    const int64_t row = idx ? idx[b] : b;
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int k = lane + 32 * i;
        if (k < dim) atomicAdd(g_out + row * g_stride + k, ri * (d[i] - x[i] * proj));
    }
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" int ssl_align_fwd(const float *xhat, const float *yhat, int64_t batch, int32_t dim, float *loss_b, void *stream) {
    SSL_CHECK_ARG(xhat && yhat && loss_b, "ssl_align_fwd: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_align_fwd: bad dim");
    if (batch == 0) return SSL_OK;
    align_fwd_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(xhat, yhat, batch, dim, loss_b);
    SSL_LAUNCH_CHECK("align_fwd_kernel");
    return SSL_OK;
}

extern "C" int ssl_uniform_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim,
                                    const float *r_scaled, const float *xhat, float offset, float *pair_sum, float *w, void *stream) {
    SSL_CHECK_ARG(rowsum_part && o_part && r_scaled && xhat && pair_sum && w, "ssl_uniform_finalize: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && n_split >= 1, "ssl_uniform_finalize: bad argument");
    if (batch == 0) return SSL_OK;
    uniform_finalize_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(rowsum_part, o_part, n_split, batch, dim, r_scaled, xhat,
                                                                             offset, pair_sum, w);
    SSL_LAUNCH_CHECK("uniform_finalize_kernel");
    return SSL_OK;
}

extern "C" int ssl_uniform_pairs(const float *xhat, int64_t batch, int32_t dim, float *pair_sum, float *w, void *stream) {
    SSL_CHECK_ARG(xhat && pair_sum && w, "ssl_uniform_pairs: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_uniform_pairs: bad dim");
    if (batch == 0) return SSL_OK;
    uniform_pairs_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(xhat, batch, dim, pair_sum, w);
    SSL_LAUNCH_CHECK("uniform_pairs_kernel");
    return SSL_OK;
}

extern "C" int ssl_unit_rows_bwd(const float *xhat, const float *rinv, const int64_t *idx, int64_t batch, int32_t dim, const float *d1,
                                 float c1, const float *d2, float c2, const float *gscale, float scale, float *g_out,
                                 int64_t g_stride, void *stream) {
    SSL_CHECK_ARG(xhat && rinv && d1 && g_out, "ssl_unit_rows_bwd: null argument");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM && g_stride >= dim, "ssl_unit_rows_bwd: bad argument");
    if (batch == 0) return SSL_OK;
    unit_rows_bwd_kernel<<<(unsigned)((batch + 7) / 8), 256, 0, STREAM>>>(xhat, rinv, idx, batch, dim, d1, c1, d2, c2, gscale, scale,
                                                                          g_out, g_stride);
    SSL_LAUNCH_CHECK("unit_rows_bwd_kernel");
    return SSL_OK;
}
