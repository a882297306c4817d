// Popularity-proportional negative candidates for the BPR models, optional key train.neg_popularity = beta:
// ssl_neg_candidates_pop draws the M - 1 extra candidates of every batch pair from an alias table of the item weights
// (deg_i + 1)^beta and optionally writes the logQ correction of the sampled softmax (csrc/pop_negs.cuh).
#include "common.cuh"
#include "pop_negs.cuh"

extern "C" int ssl_neg_candidates_pop(const int64_t *users, const int64_t *negs, int64_t n_pairs, int32_t M, const int32_t *trn_rowptr,
                                      const int32_t *trn_cols, int64_t n_item, const uint32_t *table, const float *lp,
                                      const float *lz_pop, const float *lz_uni, float ln_m, uint64_t seed, const uint64_t *seed_ptr,
                                      int64_t *cands, float *bias, void *stream) {
    namespace P = ssl_pop;
    SSL_CHECK_ARG(n_pairs >= 0 && n_pairs < (1ll << 31) && n_item > 0 && n_item < (1ll << 31), "ssl_neg_candidates_pop: bad sizes");
    SSL_CHECK_ARG(M >= 2 && M <= SSL_MAX_CANDIDATES, "ssl_neg_candidates_pop: M = %d outside [2, %d]", M, SSL_MAX_CANDIDATES);
    if (n_pairs == 0) return SSL_OK;
    SSL_CHECK_ARG(users && negs && trn_rowptr && trn_cols && table && cands, "ssl_neg_candidates_pop: null pointer");
    SSL_CHECK_ARG(bias == nullptr || (lp && lz_pop && lz_uni), "ssl_neg_candidates_pop: a bias needs lp, lz_pop and lz_uni");
    SSL_CHECK_ARG(((uintptr_t)table & 7u) == 0, "ssl_neg_candidates_pop: the alias table is not 8-byte aligned");
    const int64_t total = n_pairs * M;
    P::neg_candidates_pop_kernel<<<(unsigned)((total + P::kThreadsPerBlock - 1) / P::kThreadsPerBlock), P::kThreadsPerBlock, 0,
                                   (cudaStream_t)stream>>>(users, negs, n_pairs, M, trn_rowptr, trn_cols, n_item,
                                                           reinterpret_cast<const uint2 *>(table), lp, lz_pop, lz_uni, ln_m, seed,
                                                           seed_ptr, cands, bias);
    SSL_LAUNCH_CHECK("neg_candidates_pop_kernel");
    return SSL_OK;
}
