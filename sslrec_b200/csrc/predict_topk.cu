// ssl_predict_topk: full_predict + _mask_predict + top-k (lightgcn.py:58-66, base_model.py:35-36, metrics.py:108) in two
// launches without the [n_b, n_item] score matrix (kernels and their argument in predict_topk.cuh).
#include "common.cuh"
#include "predict_topk.cuh"

namespace {

namespace P = ssl_predict;

// Item chunks per 128-user tile: enough CTAs for two per SM (the chunk kernel's occupancy at <= 128 registers), from the shape only.
// 1024 users -> 33 chunks, 256 users (HCCF's batch) -> 132; never more chunks than 128-item tiles.
int64_t topk_chunks(int64_t n_b, int64_t n_item) {
    const int64_t user_tiles = (n_b + P::TM - 1) / P::TM, item_tiles = (n_item + P::TN - 1) / P::TN;
    int64_t nc = (2 * ssl::kNumSM + user_tiles - 1) / user_tiles;
    if (nc > item_tiles) nc = item_tiles;
    if (nc > P::kTopkMaxChunks) nc = P::kTopkMaxChunks;
    return nc < 1 ? 1 : nc;
}

// candidate-list capacity per (user, chunk): k kept keys plus room for the survivors of at least one more tile
int64_t topk_cap(int k) { return 2 * (int64_t)k + P::TN; }

// [n_b][n_chunks][cap] uint64 keys, then [n_b][n_chunks] int32 counts
int64_t topk_ws_bytes(int64_t n_b, int64_t n_item, int k) {
    const int64_t rows = n_b * topk_chunks(n_b, n_item);
    return rows * topk_cap(k) * 8 + ((rows * 4 + 15) & ~(int64_t)15);
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" int ssl_predict_topk_workspace(int64_t n_b, int64_t n_item, int32_t k, int64_t *bytes) {
    SSL_CHECK_ARG(bytes, "ssl_predict_topk_workspace: null argument");
    SSL_CHECK_ARG(n_b >= 0 && n_b <= 65535, "ssl_predict_topk_workspace: n_b = %lld must be in [0, 65535]", (long long)n_b);
    SSL_CHECK_ARG(k >= 1 && k <= P::kTopkMaxK && k <= n_item, "ssl_predict_topk_workspace: k = %d must be in [1, min(%d, n_item)]", k,
                  P::kTopkMaxK);
    SSL_CHECK_ARG(n_item < (int64_t)0xffffffff, "ssl_predict_topk_workspace: too many items");
    *bytes = topk_ws_bytes(n_b, n_item, k);
    return SSL_OK;
}

extern "C" int ssl_predict_topk(const float *users_tab, int64_t u_stride, const float *items_tab, int64_t i_stride, const int64_t *users,
                                int64_t n_b, int64_t n_item, int32_t dim, const int64_t *mask_dense, const int32_t *trn_rowptr,
                                const int32_t *trn_cols, int32_t k, void *workspace, int64_t ws_bytes, int64_t *out_idx, float *out_val,
                                void *stream) {
    SSL_CHECK_ARG(users_tab && items_tab && users && out_idx, "ssl_predict_topk: null argument");
    SSL_CHECK_ARG(mask_dense || !trn_rowptr || trn_cols, "ssl_predict_topk: trn_rowptr without trn_cols");
    SSL_CHECK_ARG(k >= 1 && k <= P::kTopkMaxK && k <= n_item, "ssl_predict_topk: k = %d must be in [1, min(%d, n_item)]", k, P::kTopkMaxK);
    SSL_CHECK_ARG(n_item < (int64_t)0xffffffff, "ssl_predict_topk: too many items");
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_predict_topk: dim %d out of range", dim);
    SSL_CHECK_ARG(n_b >= 0 && n_b <= 65535, "ssl_predict_topk: n_b = %lld must be in [0, 65535]", (long long)n_b);
    const int64_t need = topk_ws_bytes(n_b, n_item, k);
    SSL_CHECK_ARG(ws_bytes >= need, "ssl_predict_topk: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
    SSL_CHECK_ARG(need == 0 || (workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0),
                  "ssl_predict_topk: workspace must be 16-byte aligned");
    if (n_b == 0) return SSL_OK;
    const int64_t nc = topk_chunks(n_b, n_item), cap = topk_cap(k);
    uint64_t *keys = static_cast<uint64_t *>(workspace);
    int32_t *cnt = reinterpret_cast<int32_t *>(keys + n_b * nc * cap);
    dim3 grid((unsigned)nc, (unsigned)((n_b + P::TM - 1) / P::TM));
    P::predict_topk_chunk_kernel<<<grid, P::NT, 0, STREAM>>>(users_tab, u_stride, items_tab, i_stride, users, n_b, n_item, dim, mask_dense,
                                                            trn_rowptr, trn_cols, k, (int)nc, (int)cap, keys, cnt);
    SSL_LAUNCH_CHECK("predict_topk_chunk_kernel");
    P::predict_topk_merge_kernel<<<(unsigned)n_b, P::kMergeThreads, 0, STREAM>>>(keys, cnt, (int)nc, (int)cap, k, out_idx, out_val);
    SSL_LAUNCH_CHECK("predict_topk_merge_kernel");
    return SSL_OK;
}
