// ssl_scatter_rows_ordered: batch-row gradients added into a sink in a fixed order (csrc/ordered_scatter.cuh).
#include <algorithm>

#include "common.cuh"
#include "ordered_scatter.cuh"

extern "C" int ssl_scatter_rows_ordered(const float *stage, const int64_t *ids, const int64_t *order, int64_t n_pos, int32_t dim,
                                        float *sink, int64_t stride, void *stream) {
    SSL_CHECK_ARG(sink, "ssl_scatter_rows_ordered: null sink");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_scatter_rows_ordered: dim %d out of range", dim);
    SSL_CHECK_ARG(stride >= dim, "ssl_scatter_rows_ordered: stride %lld < dim %d", (long long)stride, dim);
    SSL_CHECK_ARG(n_pos >= 0, "ssl_scatter_rows_ordered: %lld positions", (long long)n_pos);
    if (n_pos == 0) return SSL_OK;                 // an empty batch: its (empty) stage and id lists may be null
    SSL_CHECK_ARG(stage && ids && order, "ssl_scatter_rows_ordered: null argument");
    namespace S = ssl_scatter;
    const int64_t units = n_pos * ((dim + 31) / 32);
    const unsigned blocks = (unsigned)std::min<int64_t>((units + S::kWarpsPerBlock - 1) / S::kWarpsPerBlock, 1 << 30);
    S::ordered_scatter_kernel<<<blocks, S::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(stage, ids, order, n_pos, dim, sink, stride);
    SSL_LAUNCH_CHECK("ordered_scatter_kernel");
    return SSL_OK;
}
