// Host execution of sslrec_b200/csrc/hard_negs.cuh (the SAME source the library compiles for sm_90a) against a sequential
// float32 restatement of its contract, bit for bit:  s_j = one fp32 FMA chain over k = 0 .. dim-1 of u[k] * c_j[k];
// negs_out[b] = cands[b, j*], j* the lowest j with the largest non-NaN s_j, 0 when every s_j is NaN.
// usage: neg_select_emu B M dim u_extra i_extra view pattern seed
//   u_extra / i_extra: row stride - dim of the user / item table;  view 1: both tables are view 1 of an interleaved
//   [rows, 3, stride] block (Rows of a 3-view layer sum), item 0 at row n_user
//   pattern 0 random rows | 1 exact ties (twin candidates: other ids of identical rows, so equal scores at several j) | 2 NaN rows among the candidates
//   | 3 every candidate row NaN for some pairs
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#define SSL_HOST_EMU 1
#include "cuda_emu.h"
#include "cuda_emu_warp.h"
#include "hard_negs.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndv() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * (float)(1u << (rnd() % 6)); }

int main(int argc, char **argv) {
    if (argc < 9) return 2;
    const int64_t B = atoll(argv[1]);
    const int M = atoi(argv[2]), dim = atoi(argv[3]), u_extra = atoi(argv[4]), i_extra = atoi(argv[5]), view = atoi(argv[6]);
    const int pattern = atoi(argv[7]);
    rng_state = (uint64_t)atoll(argv[8]) * 2654435761u + 11u;
    const int64_t n_user = 37, n_item = 53 + M;
    const int64_t us = view ? 3 * (dim + u_extra) : dim + u_extra, is = view ? 3 * (dim + i_extra) : dim + i_extra;
    if (view && u_extra != i_extra) return 2;            // one interleaved table: one stride
    // view: one [n_user + n_item, 3, dim + extra] block, the tables are its view 1 (offset dim + extra) at row 0 / row n_user
    std::vector<float> ublk, iblk;
    const float *u_tbl, *i_tbl;
    if (view) {
        ublk.resize((size_t)(n_user + n_item - 1) * us + (dim + u_extra) + dim);       // exact end: one float too far is an ASan error
        for (auto &v : ublk) v = rndv();
        u_tbl = ublk.data() + (dim + u_extra);
        i_tbl = u_tbl + n_user * us;
    } else {
        ublk.resize((size_t)(n_user - 1) * us + dim);
        iblk.resize((size_t)(n_item - 1) * is + dim);
        for (auto &v : ublk) v = rndv();
        for (auto &v : iblk) v = rndv();
        u_tbl = ublk.data();
        i_tbl = iblk.data();
    }
    const float nan = __builtin_nanf("");
    float *it = const_cast<float *>(i_tbl);
    const int64_t H = n_item / 2;                          // pattern 1: item H + r is a copy of item r, so twins score the same
    if (pattern == 1)
        for (int64_t r = 0; r < H; ++r)
            for (int k = 0; k < dim; ++k) it[(H + r) * is + k] = it[r * is + k];
    if (pattern >= 2)                                      // items 0 .. 7 score NaN for every user
        for (int64_t r = 0; r < 8; ++r) it[r * is + (int)(rnd() % (uint32_t)dim)] = nan;

    std::vector<int64_t> ancs((size_t)std::max<int64_t>(B, 1)), cands((size_t)std::max<int64_t>(B * M, 1));
    for (int64_t b = 0; b < B; ++b) {
        ancs[b] = rnd() % (uint32_t)n_user;
        for (int j = 0; j < M; ++j) {
            int64_t c = rnd() % (uint32_t)n_item;
            if (pattern == 1 && j > 0 && rnd() % 2) {      // the twin of an earlier candidate: another id, the same score
                const int64_t e = cands[b * M + rnd() % (uint32_t)j];
                c = e < H ? e + H : (e < 2 * H ? e - H : e);
            }
            if (pattern == 3 && b % 3 == 0) c = rnd() % 8;                                     // every score NaN
            cands[b * M + j] = c;
        }
    }
    std::vector<int64_t> want((size_t)std::max<int64_t>(B, 1)), got((size_t)std::max<int64_t>(B, 1), -7);
    int64_t ties = 0, all_nan = 0;
    for (int64_t b = 0; b < B; ++b) {
        const float *u = u_tbl + ancs[b] * us;
        int best_j = -1, n_best = 0;
        float best = 0.f;
        for (int j = 0; j < M; ++j) {
            const float *c = i_tbl + cands[b * M + j] * is;
            float s = 0.f;
            for (int k = 0; k < dim; ++k) s = fmaf(u[k], c[k], s);
            if (s != s) continue;
            if (best_j < 0 || s > best) {
                best = s;
                best_j = j;
                n_best = 1;
            } else if (s == best) {
                ++n_best;
            }
        }
        ties += n_best > 1;
        all_nan += best_j < 0;
        want[b] = cands[b * M + (best_j < 0 ? 0 : best_j)];
    }

    const int64_t *ap = ancs.data(), *cp = cands.data();
    int64_t *op = got.data();
    const unsigned grid = (unsigned)((B + ssl_dns::kWarpsPerBlock - 1) / ssl_dns::kWarpsPerBlock);
    if (B > 0)
        emu_launch(dim3(grid), dim3(ssl_dns::kWarpsPerBlock * 32),
                   [&]() { ssl_dns::neg_select_kernel(u_tbl, us, i_tbl, is, ap, cp, B, M, dim, op); });

    int64_t bad = 0;
    for (int64_t b = 0; b < B; ++b) bad += got[b] != want[b];
    printf("B=%lld M=%d dim=%d us=%lld is=%lld view=%d pattern=%d ties=%lld all_nan=%lld bad=%lld\n", (long long)B, M, dim,
           (long long)us, (long long)is, view, pattern, (long long)ties, (long long)all_nan, (long long)bad);
    if (pattern == 1 && B >= 8 && ties == 0) return 3;     // the case must exercise what it names
    if (pattern == 3 && B >= 3 && all_nan == 0) return 3;
    return bad == 0 ? 0 : 1;
}
