// Host execution of sslrec_b200/csrc/predict_tile.cuh (the SAME source the library compiles for sm_90a) against a float64
// restatement of base_model.py:35-36 + lightgcn.py:64.  usage: predict_emu n_b n_item dim u_stride i_stride mode seed
//   mode 0: no mask, 1: dense int64 mask, 2: training CSR
#include <stdio.h>
#include <stdlib.h>

#include "cuda_emu.h"
#include "predict_tile.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndf() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * 0.4f; }

int main(int argc, char **argv) {
    if (argc < 8) return 2;
    const int64_t n_b = atoll(argv[1]), n_item = atoll(argv[2]);
    const int dim = atoi(argv[3]);
    const int64_t us = atoll(argv[4]), is = atoll(argv[5]);
    const int mode = atoi(argv[6]);
    rng_state = (uint64_t)atoll(argv[7]) * 2654435761u + 12345u;
    const int64_t n_user = n_b / 2 + 3;                  // users repeat inside the batch
    // exact-size heap buffers: an index one element out of range is an ASan error
    std::vector<float> ut((size_t)((n_user - 1) * us + dim)), itab((size_t)((n_item - 1) * is + dim));
    for (auto &v : ut) v = rndf();
    for (auto &v : itab) v = rndf();
    std::vector<int64_t> users((size_t)n_b);
    for (auto &u : users) u = rnd() % n_user;
    std::vector<int64_t> mask;
    std::vector<int32_t> rowptr, cols;
    std::vector<char> is_masked((size_t)(n_user * n_item), 0);
    for (int64_t u = 0; u < n_user; ++u)
        for (int64_t i = 0; i < n_item; ++i)
            if (rnd() % 5 == 0) is_masked[u * n_item + i] = 1;
    if (mode == 1) {
        mask.resize((size_t)(n_b * n_item));
        for (int64_t b = 0; b < n_b; ++b)
            for (int64_t i = 0; i < n_item; ++i) mask[b * n_item + i] = is_masked[users[b] * n_item + i];
    } else if (mode == 2) {
        rowptr.push_back(0);
        for (int64_t u = 0; u < n_user; ++u) {
            for (int64_t i = 0; i < n_item; ++i)
                if (is_masked[u * n_item + i]) cols.push_back((int32_t)i);
            rowptr.push_back((int32_t)cols.size());
        }
        if (cols.empty()) cols.push_back(0);
    }
    std::vector<float> preds((size_t)(n_b * n_item), -7.f);
    const float *utp = ut.data(), *itp = itab.data();
    const int64_t *up = users.data(), *mp = mode == 1 ? mask.data() : nullptr;
    const int32_t *rp = mode == 2 ? rowptr.data() : nullptr, *cp = mode == 2 ? cols.data() : nullptr;
    float *pp = preds.data();
    using namespace ssl_predict;
    dim3 grid((unsigned)((n_item + TN - 1) / TN), (unsigned)((n_b + TM - 1) / TM));
    emu_launch(grid, dim3(NT), [&]() { predict_tile_kernel(utp, us, itp, is, up, n_b, n_item, dim, mp, rp, cp, pp); });

    double worst = 0.0;
    int64_t bad = 0, n_masked = 0;
    for (int64_t b = 0; b < n_b; ++b)
        for (int64_t i = 0; i < n_item; ++i) {
            double s = 0.0;
            float sf = 0.f;                              // the kernel's own order: one sequential fp32 FMA chain over k
            for (int k = 0; k < dim; ++k) {
                s += (double)ut[users[b] * us + k] * (double)itab[i * is + k];
                sf = fmaf(ut[users[b] * us + k], itab[i * is + k], sf);
            }
            const bool m = mode != 0 && is_masked[users[b] * n_item + i];
            const float got = preds[b * n_item + i];
            if (m) {
                ++n_masked;
                if (got != -1e8f) ++bad;
            } else {
                const double err = fabs((double)got - s);
                if (err > worst) worst = err;
                if (err > 1e-6 || got != sf) ++bad;      // fp64 agreement AND bit equality with the sequential fp32 chain
            }
        }
    printf("n_b=%lld n_item=%lld dim=%d mode=%d masked=%lld worst=%.3e bad=%lld\n", (long long)n_b, (long long)n_item, dim, mode,
           (long long)n_masked, worst, (long long)bad);
    return bad == 0 ? 0 : 1;
}
