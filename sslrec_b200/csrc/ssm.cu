// Sampled softmax loss for the BPR models, optional key train.ssm_temperature: ssl_ssm_fwd scores the positive and the M
// candidates of every pair by cosine over tau and takes the (M + 1)-way log-sum-exp; ssl_ssm_bwd sends the gradient to the
// user, positive and candidate rows (csrc/ssm.cuh).
#include "common.cuh"
#include "ssm.cuh"

namespace {
bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }
}  // namespace

extern "C" int ssl_ssm_fwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                           const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau, float *loss_b,
                           float *s, float *w, float *nrm, void *stream) {
    namespace X = ssl_ssm;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_ssm_fwd: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(M >= 1 && M <= SSL_MAX_CANDIDATES, "ssl_ssm_fwd: M = %d outside [1, %d]", M, SSL_MAX_CANDIDATES);
    SSL_CHECK_ARG(dim >= 4 && dim <= SSL_MAX_DIM && dim % 4 == 0, "ssl_ssm_fwd: dim %d is not a multiple of 4 in [4, %d]", dim, SSL_MAX_DIM);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim && u_stride % 4 == 0 && i_stride % 4 == 0,
                  "ssl_ssm_fwd: a stride is below dim %d or not a multiple of 4", dim);
    SSL_CHECK_ARG(tau > 0.f && tau <= 3.402823466e38f, "ssl_ssm_fwd: tau %g is not a finite number > 0", (double)tau);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && poss && cands && loss_b && s && w && nrm, "ssl_ssm_fwd: null pointer");
    SSL_CHECK_ARG(aligned16(u_tbl) && aligned16(i_tbl), "ssl_ssm_fwd: a table is not 16-byte aligned");
    const int per_block = X::kWarpsPerBlock * (32 / X::group_lanes(dim));
    X::ssm_fwd_kernel<<<(unsigned)((n_pairs + per_block - 1) / per_block), X::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, ancs, poss, cands, n_pairs, M, dim, tau, loss_b, s, w, nrm);
    SSL_LAUNCH_CHECK("ssm_fwd_kernel");
    return SSL_OK;
}

extern "C" int ssl_ssm_fwd_logq(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                                const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau,
                                float *loss_b, float *s, float *w, float *nrm, const float *bias, void *stream) {
    namespace X = ssl_ssm;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_ssm_fwd_logq: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(M >= 1 && M <= SSL_MAX_CANDIDATES, "ssl_ssm_fwd_logq: M = %d outside [1, %d]", M, SSL_MAX_CANDIDATES);
    SSL_CHECK_ARG(dim >= 4 && dim <= SSL_MAX_DIM && dim % 4 == 0, "ssl_ssm_fwd_logq: dim %d is not a multiple of 4 in [4, %d]", dim,
                  SSL_MAX_DIM);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim && u_stride % 4 == 0 && i_stride % 4 == 0,
                  "ssl_ssm_fwd_logq: a stride is below dim %d or not a multiple of 4", dim);
    SSL_CHECK_ARG(tau > 0.f && tau <= 3.402823466e38f, "ssl_ssm_fwd_logq: tau %g is not a finite number > 0", (double)tau);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && poss && cands && loss_b && s && w && nrm && bias, "ssl_ssm_fwd_logq: null pointer");
    SSL_CHECK_ARG(aligned16(u_tbl) && aligned16(i_tbl), "ssl_ssm_fwd_logq: a table is not 16-byte aligned");
    const int per_block = X::kWarpsPerBlock * (32 / X::group_lanes(dim));
    X::ssm_fwd_logq_kernel<<<(unsigned)((n_pairs + per_block - 1) / per_block), X::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, ancs, poss, cands, bias, n_pairs, M, dim, tau, loss_b, s, w, nrm);
    SSL_LAUNCH_CHECK("ssm_fwd_logq_kernel");
    return SSL_OK;
}

extern "C" int ssl_ssm_bwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                           const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau, const float *s,
                           const float *w, const float *nrm, const float *gscale, float scale, float *g_users, int64_t gu_stride,
                           float *g_items, int64_t gi_stride, void *stream) {
    namespace X = ssl_ssm;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_ssm_bwd: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(M >= 1 && M <= SSL_MAX_CANDIDATES, "ssl_ssm_bwd: M = %d outside [1, %d]", M, SSL_MAX_CANDIDATES);
    SSL_CHECK_ARG(dim >= 4 && dim <= SSL_MAX_DIM && dim % 4 == 0, "ssl_ssm_bwd: dim %d is not a multiple of 4 in [4, %d]", dim, SSL_MAX_DIM);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim && gu_stride >= dim && gi_stride >= dim && u_stride % 4 == 0 && i_stride % 4 == 0 &&
                      gu_stride % 4 == 0 && gi_stride % 4 == 0,
                  "ssl_ssm_bwd: a stride is below dim %d or not a multiple of 4", dim);
    SSL_CHECK_ARG(tau > 0.f && tau <= 3.402823466e38f, "ssl_ssm_bwd: tau %g is not a finite number > 0", (double)tau);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && poss && cands && s && w && nrm && g_users && g_items, "ssl_ssm_bwd: null pointer");
    SSL_CHECK_ARG(aligned16(u_tbl) && aligned16(i_tbl) && aligned16(g_users) && aligned16(g_items),
                  "ssl_ssm_bwd: a table or sink is not 16-byte aligned");
    const int per_block = X::kWarpsPerBlock * (32 / X::group_lanes(dim));
    X::ssm_bwd_kernel<<<(unsigned)((n_pairs + per_block - 1) / per_block), X::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, ancs, poss, cands, n_pairs, M, dim, tau, s, w, nrm, gscale, scale, g_users, gu_stride, g_items,
        gi_stride);
    SSL_LAUNCH_CHECK("ssm_bwd_kernel");
    return SSL_OK;
}
