// Dynamic negative sampling (DNS; Zhang et al., SIGIR 2013) for the BPR models, optional key train.dns_candidates = M:
// ssl_neg_candidates draws M - 1 extra negatives per batch pair, ssl_neg_select keeps the one the model scores highest
// (csrc/hard_negs.cuh).
#include "common.cuh"
#include "hard_negs.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// Candidates: cands[b, 0] = negs[b] (the loader's negative); cands[b, j >= 1] an item drawn uniformly until users[b] has
// not interacted with it, with sample_negs_kernel's rule: draw t = word t % 4 of the Philox block keyed (seed; b, j, t / 4,
// "DNSC"), multiply-shift onto [0, n_item), rejected while in u's sorted training-CSR row; after 64 blocks (256 rejected
// draws) the last draw is kept.  A pure function of (seed, b, j): one thread per (b, j), no shared state.  The seed is
// read from *seed_ptr when it is given (a CUDA-graph replay reads the seed the host wrote there before it).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kTagCandidates = 0x444E5343u;   // "DNSC"

__global__ void neg_candidates_kernel(const int64_t *__restrict__ users, const int64_t *__restrict__ negs, int64_t n_pairs, int M,
                                      const int32_t *__restrict__ rowptr, const int32_t *__restrict__ cols, int64_t n_item,
                                      uint64_t seed, const uint64_t *__restrict__ seed_ptr, int64_t *__restrict__ cands) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_pairs * M) return;
    const int64_t b = e / M;
    const int j = (int)(e - b * M);
    if (j == 0) {
        cands[e] = negs[b];
        return;
    }
    const uint2 key = ssl::seed_key(seed_ptr != nullptr ? __ldg(seed_ptr) : seed);
    const int64_t u = users[b];
    const int lo = rowptr[u], hi = rowptr[u + 1];
    uint32_t neg = 0;
    for (uint32_t blk = 0; blk < 64; ++blk) {
        const uint4 r = ssl::philox4x32_10(make_uint4((uint32_t)b, (uint32_t)j, blk, kTagCandidates), key);
        const uint32_t draw[4] = {r.x, r.y, r.z, r.w};
        bool done = false;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            if (done) continue;
            neg = (uint32_t)(((uint64_t)draw[t] * (uint64_t)n_item) >> 32);
            done = !ssl::csr_contains(cols, lo, hi, (int)neg);
        }
        if (done) break;
    }
    cands[e] = neg;
}

}  // namespace

extern "C" int ssl_neg_candidates(const int64_t *users, const int64_t *negs, int64_t n_pairs, int32_t M, const int32_t *trn_rowptr,
                                  const int32_t *trn_cols, int64_t n_item, uint64_t seed, const uint64_t *seed_ptr, int64_t *cands,
                                  void *stream) {
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31) && n_item > 0 && n_item < (1ll << 31), "ssl_neg_candidates: bad sizes");
    SSL_CHECK_ARG(M >= 2 && M <= SSL_MAX_CANDIDATES, "ssl_neg_candidates: M = %d outside [2, %d]", M, SSL_MAX_CANDIDATES);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(users && negs && trn_rowptr && trn_cols && cands, "ssl_neg_candidates: null pointer");
    const int64_t total = n_pairs * M;
    neg_candidates_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(users, negs, n_pairs, M, trn_rowptr, trn_cols,
                                                                                            n_item, seed, seed_ptr, cands);
    SSL_LAUNCH_CHECK("neg_candidates_kernel");
    return SSL_OK;
}

extern "C" int ssl_neg_select(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                              const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, int64_t *negs_out, void *stream) {
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31), "ssl_neg_select: %lld pairs", (long long)n_pairs);
    SSL_CHECK_ARG(M >= 2 && M <= SSL_MAX_CANDIDATES, "ssl_neg_select: M = %d outside [2, %d]", M, SSL_MAX_CANDIDATES);
    SSL_CHECK_ARG(dim >= 1 && dim <= SSL_MAX_DIM, "ssl_neg_select: dim %d out of range", dim);
    SSL_CHECK_ARG(u_stride >= dim && i_stride >= dim, "ssl_neg_select: a stride is below dim %d", dim);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(u_tbl && i_tbl && ancs && cands && negs_out, "ssl_neg_select: null pointer");
    namespace D = ssl_dns;
    D::neg_select_kernel<<<(unsigned)((n_pairs + D::kWarpsPerBlock - 1) / D::kWarpsPerBlock), D::kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(
        u_tbl, u_stride, i_tbl, i_stride, ancs, cands, n_pairs, M, dim, negs_out);
    SSL_LAUNCH_CHECK("neg_select_kernel");
    return SSL_OK;
}
