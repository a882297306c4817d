// a17  KMeansClustering (models/aug_utils.py:142-157): Lloyd iterations, deterministic.
// a21  PairwiseTrnData.sample_negs (data_utils/datasets_general_cf.py:13-26): uniform rejection sampling.
#include "common.cuh"
#include "kmeans_assign.cuh"

namespace {

// centroids = newCents / (clustNums + 1e-6)   (aug_utils.py:156)
__global__ void kmeans_update_kernel(const float *__restrict__ part_sum, const float *__restrict__ part_cnt, int n_cta, int K,
                                     int dim, float *__restrict__ cents, float *__restrict__ counts) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= K * dim) return;
    const int k = e / dim;
    float s = 0.f, c = 0.f;
    for (int b = 0; b < n_cta; ++b) {
        s += part_sum[(size_t)b * K * dim + e];
        c += part_cnt[(size_t)b * K + k];
    }
    cents[e] = s / (c + 1e-6f);
    if (e % dim == 0) counts[k] = c;
}

// ---------------------------------------------------------------------------------------------
// Negative sampling: for the e-th training pair (u, i+) draw i- uniform over the items until u has
// not interacted with it (datasets_general_cf.py:17-23: randint + dok lookup).  Membership is a
// binary search in u's sorted training-CSR row; draw t of pair e in epoch `epoch` is the Philox
// block keyed (seed; e, t / 4, epoch), so the sample is a pure function of (seed, epoch, e).
// A user who interacted with every item would never terminate in the reference; here the draw is
// accepted after 64 blocks (256 rejected draws).
// ---------------------------------------------------------------------------------------------

__global__ void sample_negs_kernel(const int64_t *__restrict__ users, int64_t n_pairs, const int32_t *__restrict__ rowptr,
                                   const int32_t *__restrict__ cols, int64_t n_item, uint64_t seed, uint32_t epoch,
                                   int64_t *__restrict__ negs) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_pairs) return;
    const int64_t u = users[e];
    const int lo = rowptr[u], hi = rowptr[u + 1];
    uint32_t neg = 0;
    for (uint32_t blk = 0; blk < 64; ++blk) {
        const uint4 r = ssl::philox4x32_10(make_uint4((uint32_t)e, (uint32_t)((uint64_t)e >> 32), blk, epoch ^ 0x4E454753u /*"NEGS"*/),
                                           ssl::seed_key(seed));
        const uint32_t draw[4] = {r.x, r.y, r.z, r.w};
        bool done = false;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            if (done) continue;
            // unbiased enough for n_item << 2^32: multiply-shift maps the 32 random bits onto [0, n_item)
            neg = (uint32_t)(((uint64_t)draw[t] * (uint64_t)n_item) >> 32);
            done = !ssl::csr_contains(cols, lo, hi, (int)neg);
        }
        if (done) break;
    }
    negs[e] = neg;
}

}  // namespace

extern "C" int ssl_kmeans_workspace(int64_t n, int32_t dim, int32_t k, int32_t *n_cta, int32_t *n_warps) {
    SSL_CHECK_ARG(n > 0 && dim > 0 && k > 0 && n_cta && n_warps, "ssl_kmeans_workspace: bad arguments");
    int W = 8;
    // sized for the widest instantiation, whichever runs: the row partition (and with it every partial sum) does not depend on the option
    auto smem = [&](int w) { return sizeof(float) * ssl_kmeans::smem_floats(k, dim, w, ssl_kmeans::kMaxRowsPerRound); };
    while (W > 1 && smem(W) > 200 * 1024) W >>= 1;
    SSL_CHECK_ARG(smem(W) <= 200 * 1024, "ssl_kmeans: cluster_num * dim = %lld does not fit shared memory", (long long)k * dim);
    int64_t ctas = (n + (int64_t)W * 8 - 1) / ((int64_t)W * 8);      // at least ~8 rows per warp
    if (ctas > ssl::kNumSM) ctas = ssl::kNumSM;
    *n_cta = (int32_t)ctas;
    *n_warps = W;
    return SSL_OK;
}

extern "C" int ssl_kmeans_iter(const float *x, int64_t stride, int64_t n, int32_t dim, int32_t k, float *centroids, int64_t *assign,
                               float *part_sum, float *part_cnt, float *counts, int32_t *changed, void *stream) {
    SSL_CHECK_ARG(x && centroids && assign && part_sum && part_cnt && counts && changed, "ssl_kmeans_iter: null pointer");
    int32_t n_cta = 0, W = 0;
    int rc = ssl_kmeans_workspace(n, dim, k, &n_cta, &W);
    if (rc != SSL_OK) return rc;
    SSL_CHECK_ARG(stride >= dim, "ssl_kmeans_iter: stride < dim");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t rows_per_cta = (n + n_cta - 1) / n_cta;
    const int64_t rows_per_warp = (rows_per_cta + W - 1) / W;
    if (ssl::g_kmeans_rows_per_round > 1) {      // default: 4 rows per warp and round (4 independent distance chains per lane), results bit-identical
        constexpr int R = ssl_kmeans::kMaxRowsPerRound;
        const size_t smem = sizeof(float) * ssl_kmeans::smem_floats(k, dim, W, R);
        SSL_CUDA(cudaFuncSetAttribute(ssl_kmeans::kmeans_assign_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ssl_kmeans::kmeans_assign_kernel<R><<<n_cta, W * 32, smem, s>>>(x, stride, n, dim, k, centroids, assign, part_sum, part_cnt, changed,
                                                                       rows_per_cta, rows_per_warp);
    } else {
        const size_t smem = sizeof(float) * ssl_kmeans::smem_floats(k, dim, W, 1);
        SSL_CUDA(cudaFuncSetAttribute(ssl_kmeans::kmeans_assign_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ssl_kmeans::kmeans_assign_kernel<1><<<n_cta, W * 32, smem, s>>>(x, stride, n, dim, k, centroids, assign, part_sum, part_cnt, changed,
                                                                       rows_per_cta, rows_per_warp);
    }
    SSL_LAUNCH_CHECK("kmeans_assign_kernel");
    kmeans_update_kernel<<<(k * dim + 255) / 256, 256, 0, s>>>(part_sum, part_cnt, n_cta, k, dim, centroids, counts);
    SSL_LAUNCH_CHECK("kmeans_update_kernel");
    return SSL_OK;
}

extern "C" int ssl_sample_negs(const int64_t *users, int64_t n_pairs, const int32_t *trn_rowptr, const int32_t *trn_cols,
                               int64_t n_item, uint64_t seed, uint32_t epoch, int64_t *negs, void *stream) {
    SSL_CHECK_ARG(n_pairs >= 0 && n_item > 0 && n_item < (1ll << 31), "ssl_sample_negs: bad sizes");
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(users && trn_rowptr && trn_cols && negs, "ssl_sample_negs: null pointer");
    sample_negs_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(users, n_pairs, trn_rowptr, trn_cols,
                                                                                           n_item, seed, epoch, negs);
    SSL_LAUNCH_CHECK("sample_negs_kernel");
    return SSL_OK;
}
