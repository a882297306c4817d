// ssl_nce_bwd_cols: the column backward of the in-batch sampled softmax (csrc/ssm_in_batch.cuh).
#include <algorithm>

#include "common.cuh"
#include "ssm_in_batch.cuh"

extern "C" int ssl_nce_bwd_cols(const float *dt_part, int32_t n_split, const float *t_hat, const float *rinv, const float *colw,
                                const int64_t *ids, int64_t n, int32_t dim, float *sink, int64_t stride, void *stream) {
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_nce_bwd_cols: dim %d out of range", dim);
    SSL_CHECK_ARG(n_split >= 1, "ssl_nce_bwd_cols: n_split %d < 1", n_split);
    SSL_CHECK_ARG(n >= 0, "ssl_nce_bwd_cols: %lld columns", (long long)n);
    SSL_CHECK_ARG(stride >= dim, "ssl_nce_bwd_cols: stride %lld < dim %d", (long long)stride, dim);
    if (n == 0) return SSL_OK;
    SSL_CHECK_ARG(dt_part && t_hat && rinv && colw && sink, "ssl_nce_bwd_cols: null argument");
    namespace K = ssl_inb;
    const unsigned blocks = (unsigned)std::min<int64_t>((n + K::kWarpsPerBlock - 1) / K::kWarpsPerBlock, INT32_MAX);
    SSL_CHECK_ARG((int64_t)blocks * K::kWarpsPerBlock >= n, "ssl_nce_bwd_cols: %lld columns exceed one launch", (long long)n);
    K::nce_bwd_cols_kernel<<<blocks, K::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(dt_part, n_split, t_hat, rinv, colw, ids, n, dim,
                                                                                         sink, stride);
    SSL_LAUNCH_CHECK("nce_bwd_cols_kernel");
    return SSL_OK;
}
