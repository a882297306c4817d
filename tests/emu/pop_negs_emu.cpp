// Host execution of sslrec_b200/csrc/pop_negs.cuh and of ssm_fwd_logq_kernel in csrc/ssm.cuh (the SAME sources the library
// compiles for sm_90a); tests/test_host_neg_popularity.py compares the outputs with tests/pop_oracle.py bit for bit.
// usage: pop_negs_emu draw in.bin out.bin
//   in:  int64 B, M, n_item, n_user, nnz; uint64 seed; float32 ln_m; int32 rowptr[n_user + 1], cols[nnz];
//        uint32 table[2 n_item]; float32 lp[n_item], lz_pop[n_user], lz_uni[n_user]; int64 users[B], negs[B]
//   out: int64 cands[B M], float32 bias[B M] (one launch with the bias), int64 cands[B M] (a second launch without it)
// usage: pop_negs_emu ssm in.bin out.bin
//   in:  int64 B, M, d, n_user_rows, n_item_rows; float32 tau; float32 u[n_user_rows d], i[n_item_rows d];
//        int64 ancs[B], poss[B], cands[B M]; float32 bias[B M]
//   out: float32 loss_b[B], s[B, M+1], w[B, M+1], nrm[B, M+2] of ssm_fwd_logq_kernel, then the same four of ssm_fwd_kernel
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

struct uint2 {
    uint32_t x, y;
};
struct uint4 {
    uint32_t x, y, z, w;
};
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct float4 {
    float x, y, z, w;
};
#include "cuda_emu.h"
static inline void atomicAdd(float4 *, float4) { abort(); }   // ssm.cuh's backward is not run here
#include "pop_negs.cuh"
#include "ssm.cuh"

// exactly n elements, 16-byte aligned: one element too far is an ASan error; freed at the end of main
static std::vector<void *> emu_buffers;
template <class T>
static T *buf(int64_t n) {
    void *p = nullptr;
    if (posix_memalign(&p, 16, (size_t)(n > 0 ? n : 1) * sizeof(T)) != 0) abort();
    emu_buffers.push_back(p);
    memset(p, 0xA5, (size_t)(n > 0 ? n : 1) * sizeof(T));
    return static_cast<T *>(p);
}

template <class T>
static T *rd(FILE *f, int64_t n) {
    T *p = buf<T>(n);
    if (n && fread(p, sizeof(T), (size_t)n, f) != (size_t)n) {
        fprintf(stderr, "short input\n");
        exit(2);
    }
    return p;
}

static int draw(FILE *in, FILE *out) {
    const int64_t *h = rd<int64_t>(in, 5);
    const int64_t B = h[0], n_item = h[2], n_user = h[3], nnz = h[4];
    const int M = (int)h[1];
    const uint64_t seed = *rd<uint64_t>(in, 1);
    const float ln_m = *rd<float>(in, 1);
    const int32_t *rowptr = rd<int32_t>(in, n_user + 1), *cols = rd<int32_t>(in, nnz);
    const uint2 *table = reinterpret_cast<const uint2 *>(rd<uint32_t>(in, 2 * n_item));
    const float *lp = rd<float>(in, n_item), *lz_pop = rd<float>(in, n_user), *lz_uni = rd<float>(in, n_user);
    const int64_t *users = rd<int64_t>(in, B), *negs = rd<int64_t>(in, B);
    int64_t *cands = buf<int64_t>(B * M), *cands2 = buf<int64_t>(B * M);
    float *bias = buf<float>(B * M);
    const dim3 grid((unsigned)((B * M + ssl_pop::kThreadsPerBlock - 1) / ssl_pop::kThreadsPerBlock)), block(ssl_pop::kThreadsPerBlock);
    emu_launch(grid, block, [&]() {
        ssl_pop::neg_candidates_pop_kernel(users, negs, B, M, rowptr, cols, n_item, table, lp, lz_pop, lz_uni, ln_m, seed, nullptr, cands,
                                           bias);
    });
    emu_launch(grid, block, [&]() {
        ssl_pop::neg_candidates_pop_kernel(users, negs, B, M, rowptr, cols, n_item, table, nullptr, nullptr, nullptr, ln_m, seed, &seed,
                                           cands2, nullptr);
    });
    fwrite(cands, 8, (size_t)(B * M), out);
    fwrite(bias, 4, (size_t)(B * M), out);
    fwrite(cands2, 8, (size_t)(B * M), out);
    return 0;
}

static int ssm(FILE *in, FILE *out) {
    const int64_t *h = rd<int64_t>(in, 5);
    const int64_t B = h[0], nu = h[3], ni = h[4];
    const int M = (int)h[1], d = (int)h[2];
    const float tau = *rd<float>(in, 1);
    const float *ut = rd<float>(in, nu * d), *it = rd<float>(in, ni * d);
    const int64_t *ancs = rd<int64_t>(in, B), *poss = rd<int64_t>(in, B), *cands = rd<int64_t>(in, B * M);
    const float *bias = rd<float>(in, B * M);
    const int64_t Q = M + 1;
    const int G = ssl_ssm::group_lanes(d);
    const int per_block = ssl_ssm::kWarpsPerBlock * (32 / G);
    const dim3 grid((unsigned)((B + per_block - 1) / per_block)), block(ssl_ssm::kWarpsPerBlock * 32);
    for (int logq = 1; logq >= 0; --logq) {
        float *loss = buf<float>(B), *s = buf<float>(B * Q), *w = buf<float>(B * Q), *nrm = buf<float>(B * (Q + 1));
        emu_launch(grid, block, [&]() {
            if (logq)
                ssl_ssm::ssm_fwd_logq_kernel(ut, d, it, d, ancs, poss, cands, bias, B, M, d, tau, loss, s, w, nrm);
            else
                ssl_ssm::ssm_fwd_kernel(ut, d, it, d, ancs, poss, cands, B, M, d, tau, loss, s, w, nrm);
        });
        fwrite(loss, 4, (size_t)B, out);
        fwrite(s, 4, (size_t)(B * Q), out);
        fwrite(w, 4, (size_t)(B * Q), out);
        fwrite(nrm, 4, (size_t)(B * (Q + 1)), out);
    }
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 4) return 2;
    FILE *in = fopen(argv[2], "rb"), *out = fopen(argv[3], "wb");
    if (!in || !out) return 2;
    const int rc = strcmp(argv[1], "draw") == 0 ? draw(in, out) : strcmp(argv[1], "ssm") == 0 ? ssm(in, out) : 2;
    fclose(in);
    fclose(out);
    for (void *p : emu_buffers) free(p);
    return rc;
}
