// Host execution of sslrec_b200/csrc/predict_topk.cuh (the SAME source the library compiles for sm_90a) against a host restatement of
// ssl_predict_mask + ssl_topk: every score one sequential fp32 FMA chain, the mask formula, a sort by (value descending, item ascending).
// usage: predict_topk_emu n_b n_item dim u_stride i_stride mode k n_chunks cap seed
//   mode 0: no mask, 1: dense int64 mask, 2: training CSR (rows sorted ascending).  Item rows are duplicated at random (exact ties,
//   across chunks and at both ends of the catalogue), user 0's row is all zeros and user 1 has all but a few items masked.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

#include "cuda_emu.h"
#include "cuda_emu_warp.h"
#include "predict_topk.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndf() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * 0.4f; }
static inline uint32_t host_okey(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

int main(int argc, char **argv) {
    if (argc < 11) return 2;
    const int64_t n_b = atoll(argv[1]), n_item = atoll(argv[2]);
    const int dim = atoi(argv[3]);
    const int64_t us = atoll(argv[4]), is = atoll(argv[5]);
    const int mode = atoi(argv[6]), k = atoi(argv[7]), nc = atoi(argv[8]), cap = atoi(argv[9]);
    rng_state = (uint64_t)atoll(argv[10]) * 2654435761u + 12345u;
    const int64_t n_user = n_b / 2 + 3;                  // users repeat inside the batch
    std::vector<float> ut((size_t)((n_user - 1) * us + dim)), itab((size_t)((n_item - 1) * is + dim));
    for (auto &v : ut) v = rndf();
    for (auto &v : itab) v = rndf();
    for (int q = 0; q < dim; ++q) ut[q] = 0.f;           // user 0: every score is +0 -> ties decided by the item id alone
    for (int64_t i = 1; i < n_item; ++i)
        if (rnd() % 4 == 0) {
            const int64_t src = (rnd() % 2) ? rnd() % i : (int64_t)(rnd() % 3);
            for (int q = 0; q < dim; ++q) itab[i * is + q] = itab[src * is + q];
        }
    for (int q = 0; q < dim; ++q) itab[(n_item - 1) * is + q] = itab[q];     // the last item ties the first
    std::vector<int64_t> users((size_t)n_b);
    for (auto &u : users) u = rnd() % n_user;
    if (n_b > 2) users[1] = 1, users[2] = 0;
    std::vector<char> is_masked((size_t)(n_user * n_item), 0);
    for (int64_t u = 0; u < n_user; ++u)
        for (int64_t i = 0; i < n_item; ++i)
            if (u == 1 ? (i % 97 != 5) : (rnd() % 5 == 0)) is_masked[u * n_item + i] = 1;
    std::vector<int64_t> mask;
    std::vector<int32_t> rowptr, cols;
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
    // exact-size workspace holding garbage: the kernels must not read what they did not write
    std::vector<uint64_t> ws_keys((size_t)(n_b * nc * cap), 0xabababababababab);
    std::vector<int32_t> ws_cnt((size_t)(n_b * nc), -77);
    std::vector<int64_t> out_idx((size_t)(n_b * k), -1);
    std::vector<float> out_val((size_t)(n_b * k), -7.f);
    const float *utp = ut.data(), *itp = itab.data();
    const int64_t *up = users.data(), *mp = mode == 1 ? mask.data() : nullptr;
    const int32_t *rp = mode == 2 ? rowptr.data() : nullptr, *cp = mode == 2 ? cols.data() : nullptr;
    uint64_t *wk = ws_keys.data();
    int32_t *wc = ws_cnt.data();
    int64_t *oi = out_idx.data();
    float *ov = out_val.data();
    using namespace ssl_predict;
    emu_launch(dim3((unsigned)nc, (unsigned)((n_b + TM - 1) / TM)), dim3(NT),
               [&]() { predict_topk_chunk_kernel(utp, us, itp, is, up, n_b, n_item, dim, mp, rp, cp, k, nc, cap, wk, wc); });
    emu_launch(dim3((unsigned)n_b), dim3(kMergeThreads), [&]() { predict_topk_merge_kernel(wk, wc, nc, cap, k, oi, ov); });

    int64_t bad = 0, n_masked_top = 0;
    std::vector<std::pair<uint64_t, int64_t>> row((size_t)n_item);
    for (int64_t b = 0; b < n_b; ++b) {
        for (int64_t i = 0; i < n_item; ++i) {
            float s = 0.f;
            for (int q = 0; q < dim; ++q) s = fmaf(ut[users[b] * us + q], itab[i * is + q], s);
            float m = 0.f;
            if (mode == 1) m = (float)mask[b * n_item + i];
            float v = s * (1.f - m) - 1e8f * m;                                // base_model.py:36
            if (mode == 2 && is_masked[users[b] * n_item + i]) v = v * 0.f - 1e8f;
            uint32_t bits;
            memcpy(&bits, &v, 4);
            row[i] = {((uint64_t)host_okey(v) << 32) | (0xffffffffu - (uint32_t)i), (int64_t)bits};
        }
        std::sort(row.begin(), row.end(), [](const std::pair<uint64_t, int64_t> &x, const std::pair<uint64_t, int64_t> &y) { return x.first > y.first; });
        for (int q = 0; q < k; ++q) {
            const int64_t want_i = (int64_t)(0xffffffffu - (uint32_t)row[q].first);
            uint32_t got_bits;
            memcpy(&got_bits, &out_val[b * k + q], 4);
            if (out_idx[b * k + q] != want_i || got_bits != (uint32_t)row[q].second) ++bad;
            if (mode != 0 && is_masked[users[b] * n_item + want_i]) ++n_masked_top;
        }
    }
    printf("n_b=%lld n_item=%lld dim=%d mode=%d k=%d chunks=%d cap=%d masked_in_top=%lld bad=%lld\n", (long long)n_b, (long long)n_item, dim,
           mode, k, nc, cap, (long long)n_masked_top, (long long)bad);
    return bad == 0 ? 0 : 1;
}
