// MixGCF negatives for the BPR models (Huang et al., KDD 2021), optional key train.mixgcf: ssl_mixgcf_bpr_fwd mixes each
// candidate with the positive layer by layer, keeps every layer's hardest mix and scores the pooled negative with the BPR
// term; ssl_mixgcf_bpr_bwd sends its gradient to the sum and layer sinks (csrc/mixgcf.cuh).
#include "common.cuh"
#include "mixgcf.cuh"

extern "C" int ssl_mixgcf_bpr_fwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride,
                                  const float *const *layer_tbls, const int64_t *layer_strides, int32_t n_layers, const int64_t *ancs,
                                  const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, uint64_t seed,
                                  const uint64_t *seed_ptr, const float *alpha_in, float *loss_b, float *coef_b, int64_t *picks,
                                  float *alpha_out, float *nhat, void *stream) {
    namespace X = ssl_mix;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_mixgcf_bpr_fwd: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(M >= 1 && M <= SSL_MAX_CANDIDATES, "ssl_mixgcf_bpr_fwd: M = %d outside [1, %d]", M, SSL_MAX_CANDIDATES);
    SSL_CHECK_ARG(n_layers >= 1 && n_layers <= X::kMaxLayers, "ssl_mixgcf_bpr_fwd: %d layers outside [1, %d]", n_layers, X::kMaxLayers);
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_mixgcf_bpr_fwd: dim %d out of range", dim);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim, "ssl_mixgcf_bpr_fwd: a stride is below dim %d", dim);
    SSL_CHECK_ARG(layer_tbls && layer_strides, "ssl_mixgcf_bpr_fwd: null layer list");
    X::LayerTables layers = {};
    for (int l = 0; l < n_layers; ++l) {
        SSL_CHECK_ARG(layer_strides[l] >= dim, "ssl_mixgcf_bpr_fwd: layer %d stride is below dim %d", l, dim);
        layers.ptr[l] = layer_tbls[l];
        layers.stride[l] = layer_strides[l];
    }
    if (n_pairs == 0) return SSL_OK;
    for (int l = 0; l < n_layers; ++l) SSL_CHECK_ARG(layers.ptr[l], "ssl_mixgcf_bpr_fwd: layer %d is null", l);
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && poss && cands && loss_b && coef_b && picks && alpha_out && nhat,
                  "ssl_mixgcf_bpr_fwd: null pointer");
    X::mixgcf_fwd_kernel<<<(unsigned)((n_pairs + X::kWarpsPerBlock - 1) / X::kWarpsPerBlock), X::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, layers, n_layers, ancs, poss, cands, n_pairs, M, dim, seed, seed_ptr, alpha_in, loss_b, coef_b,
        picks, alpha_out, nhat);
    SSL_LAUNCH_CHECK("mixgcf_fwd_kernel");
    return SSL_OK;
}

extern "C" int ssl_mixgcf_bpr_bwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                                  const int64_t *poss, const int64_t *picks, int64_t n_pairs, int32_t n_layers, int32_t dim,
                                  const float *nhat, const float *alpha, const float *coef_b, const float *gscale, float scale,
                                  float *g_users, int64_t gu_stride, float *g_items, int64_t gi_stride, float *const *g_layers,
                                  const int64_t *gl_strides, void *stream) {
    namespace X = ssl_mix;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_mixgcf_bpr_bwd: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(n_layers >= 1 && n_layers <= X::kMaxLayers, "ssl_mixgcf_bpr_bwd: %d layers outside [1, %d]", n_layers, X::kMaxLayers);
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_mixgcf_bpr_bwd: dim %d out of range", dim);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim && gu_stride >= dim && gi_stride >= dim, "ssl_mixgcf_bpr_bwd: a stride is below dim %d", dim);
    SSL_CHECK_ARG(g_layers && gl_strides, "ssl_mixgcf_bpr_bwd: null layer sink list");
    X::LayerSinks sinks = {};
    for (int l = 0; l < n_layers; ++l) {
        SSL_CHECK_ARG(gl_strides[l] >= dim, "ssl_mixgcf_bpr_bwd: layer %d sink stride is below dim %d", l, dim);
        sinks.ptr[l] = g_layers[l];
        sinks.stride[l] = gl_strides[l];
    }
    if (n_pairs == 0) return SSL_OK;
    for (int l = 0; l < n_layers; ++l) SSL_CHECK_ARG(sinks.ptr[l], "ssl_mixgcf_bpr_bwd: layer %d sink is null", l);
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && poss && picks && nhat && alpha && coef_b && g_users && g_items,
                  "ssl_mixgcf_bpr_bwd: null pointer");
    X::mixgcf_bwd_kernel<<<(unsigned)((n_pairs + X::kWarpsPerBlock - 1) / X::kWarpsPerBlock), X::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, ancs, poss, picks, n_pairs, n_layers, dim, nhat, alpha, coef_b, gscale, scale, g_users, gu_stride,
        g_items, gi_stride, sinks);
    SSL_LAUNCH_CHECK("mixgcf_bwd_kernel");
    return SSL_OK;
}
