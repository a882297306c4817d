// Host execution of sslrec_b200/csrc/mixgcf.cuh (the SAME source the library compiles for sm_90a) against a sequential float32
// restatement of its contract, bit for bit: picks, alpha, nhat, loss_b, coef_b of the forward, and every per-position
// contribution of the backward run on identity ids into -0.0 stages (the train.deterministic route; numbering in mixgcf.cuh).
// usage: mixgcf_emu B M n_layers dim extra view pattern alpha_mode seed
//   extra: row stride - dim of every table;  view 1: every table is view 1 of an interleaved [rows, 3, dim + extra] block
//   pattern 0 random rows | 1 exact ties (twin items: other ids with identical rows in every layer) | 2 NaN rows among the
//   candidates | 3 every candidate row NaN for some pairs
//   alpha_mode 0 drawn from the seed | 1 injected random | 2 injected 0 | 3 injected the largest float below 1
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#define SSL_HOST_EMU 1
struct uint2 {
    uint32_t x, y;
};
struct uint4 {
    uint32_t x, y, z, w;
};
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
#include "cuda_emu.h"
#define __grid_constant__
static inline float atomicAdd(float *p, float v) {        // the tests' stages get one add per element: order never matters
    float old = *p;
    *p = old + v;
    return old;
}
#include "mixgcf.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndv() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * (float)(1u << (rnd() % 6)); }

// bit for bit, except that any two NaNs match (x86 and the GPU may give a NaN result another sign or payload)
static bool same(float a, float b) { return memcmp(&a, &b, 4) == 0 || (a != a && b != b); }

int main(int argc, char **argv) {
    if (argc < 10) return 2;
    const int64_t B = atoll(argv[1]);
    const int M = atoi(argv[2]), L1 = atoi(argv[3]), dim = atoi(argv[4]), extra = atoi(argv[5]), view = atoi(argv[6]);
    const int pattern = atoi(argv[7]), amode = atoi(argv[8]);
    rng_state = (uint64_t)atoll(argv[9]) * 2654435761u + 11u;
    const uint64_t seed = ((uint64_t)rnd() << 32) | rnd();
    const int64_t n_user = 37, n_item = 53 + M, N = n_user + n_item;
    const int64_t rs = view ? 3 * (dim + extra) : dim + extra;
    // tables: the sum table (users and items) and L1 layer tables, each its own block; a view is offset dim + extra into it
    const int64_t blk_floats = (N - 1) * rs + (view ? dim + extra : 0) + dim;     // exact end: one float too far is an ASan error
    std::vector<std::vector<float>> blocks(1 + L1, std::vector<float>((size_t)blk_floats));
    for (auto &bl : blocks)
        for (auto &v : bl) v = rndv();
    auto base = [&](int t) { return blocks[t].data() + (view ? dim + extra : 0); };
    const float *u_tbl = base(0), *i_tbl = base(0) + n_user * rs;
    std::vector<const float *> lt(L1);
    std::vector<int64_t> ls(L1, rs);
    for (int l = 0; l < L1; ++l) lt[l] = base(1 + l) + n_user * rs;
    const float nan = __builtin_nanf("");
    const int64_t H = n_item / 2;                          // pattern 1: item H + r is a copy of item r in every layer
    for (int l = 0; l < L1; ++l) {
        float *it = const_cast<float *>(lt[l]);
        if (pattern == 1)
            for (int64_t r = 0; r < H; ++r)
                for (int k = 0; k < dim; ++k) it[(H + r) * rs + k] = it[r * rs + k];
        if (pattern >= 2)                                  // items 0 .. 7 score NaN for every user (and every alpha < 1)
            for (int64_t r = 0; r < 8; ++r) it[r * rs + (int)(rnd() % (uint32_t)dim)] = nan;
    }
    const size_t Bs = (size_t)std::max<int64_t>(B, 1);
    std::vector<int64_t> ancs(Bs), poss(Bs), cands(Bs * M);
    for (int64_t b = 0; b < B; ++b) {
        ancs[b] = rnd() % (uint32_t)n_user;
        poss[b] = 8 + rnd() % (uint32_t)(n_item - 8);      // the positive is never a NaN row
        for (int j = 0; j < M; ++j) {
            int64_t c = 8 + rnd() % (uint32_t)(n_item - 8);
            if (pattern == 1 && j > 0 && rnd() % 2) {
                const int64_t e = cands[b * M + rnd() % (uint32_t)j];
                c = e < H ? e + H : (e < 2 * H ? e - H : e);
            }
            if (pattern == 2 && rnd() % 4 == 0) c = rnd() % 8;
            if (pattern == 3 && b % 3 == 0) c = rnd() % 8;
            cands[b * M + j] = c;
        }
    }
    std::vector<float> ain;
    if (amode != 0) {
        ain.resize(Bs * L1);
        for (auto &a : ain) a = amode == 1 ? (float)(rnd() >> 8) * (1.0f / 16777216.0f) : (amode == 2 ? 0.f : nextafterf(1.f, 0.f));
    }

    // ---- sequential restatement ----
    std::vector<int64_t> w_picks(Bs * L1);
    std::vector<float> w_alpha(Bs * L1), w_nhat(Bs * dim), w_loss(Bs), w_coef(Bs);
    int64_t ties = 0, all_nan = 0;
    for (int64_t b = 0; b < B; ++b) {
        const float *u = u_tbl + ancs[b] * rs;
        for (int l = 0; l < L1; ++l) {
            const float a = amode ? ain[b * L1 + l] : ssl_mix::alpha_draw(seed, b, l), a1 = 1.f - a;
            const float *xp = lt[l] + poss[b] * rs;
            int best_j = -1, n_best = 0;
            float best = 0.f;
            for (int j = 0; j < M; ++j) {
                const float *xc = lt[l] + cands[b * M + j] * rs;
                float s = 0.f;
                for (int k = 0; k < dim; ++k) s = fmaf(u[k], fmaf(a, xp[k], a1 * xc[k]), s);
                if (s != s) continue;
                if (best_j < 0 || s > best) {
                    best = s, best_j = j, n_best = 1;
                } else if (s == best) {
                    ++n_best;
                }
            }
            ties += n_best > 1;
            all_nan += best_j < 0;
            const int64_t pick = cands[b * M + (best_j < 0 ? 0 : best_j)];
            w_picks[b * L1 + l] = pick;
            w_alpha[b * L1 + l] = a;
            const float *xc = lt[l] + pick * rs;
            for (int k = 0; k < dim; ++k) {
                const float m = fmaf(a, xp[k], a1 * xc[k]);
                w_nhat[b * dim + k] = l == 0 ? m : w_nhat[b * dim + k] + m;
            }
        }
        const float *pb = i_tbl + poss[b] * rs;
        float zn = 0.f, zp = 0.f;
        for (int k = 0; k < dim; ++k) zn = fmaf(u[k], w_nhat[b * dim + k], zn), zp = fmaf(u[k], pb[k], zp);
        const float z = zn - zp;
        w_loss[b] = z > 20.f ? z : log1pf(expf(z));
        w_coef[b] = 1.f / (1.f + expf(-z));
    }

    // ---- the kernel ----
    ssl_mix::LayerTables tabs = {};
    for (int l = 0; l < L1; ++l) tabs.ptr[l] = lt[l], tabs.stride[l] = ls[l];
    std::vector<int64_t> g_picks(Bs * L1, -7);
    std::vector<float> g_alpha(Bs * L1, -7.f), g_nhat(Bs * dim, -7.f), g_loss(Bs, -7.f), g_coef(Bs, -7.f);
    const unsigned grid = (unsigned)((B + ssl_mix::kWarpsPerBlock - 1) / ssl_mix::kWarpsPerBlock);
    const float *aip = amode ? ain.data() : nullptr;
    if (B > 0)
        emu_launch(dim3(grid), dim3(ssl_mix::kWarpsPerBlock * 32), [&]() {
            ssl_mix::mixgcf_fwd_kernel(u_tbl, rs, i_tbl, rs, tabs, L1, ancs.data(), poss.data(), cands.data(), B, M, dim, seed, nullptr,
                                       aip, g_loss.data(), g_coef.data(), g_picks.data(), g_alpha.data(), g_nhat.data());
        });
    int64_t bad_fwd = 0;
    for (int64_t b = 0; b < B; ++b) {
        bad_fwd += !same(g_loss[b], w_loss[b]) + !same(g_coef[b], w_coef[b]);
        for (int l = 0; l < L1; ++l) bad_fwd += (g_picks[b * L1 + l] != w_picks[b * L1 + l]) + !same(g_alpha[b * L1 + l], w_alpha[b * L1 + l]);
        for (int k = 0; k < dim; ++k) bad_fwd += !same(g_nhat[b * dim + k], w_nhat[b * dim + k]);
    }

    // ---- backward, staged: gathered rows, identity ids, -0.0 stages ----
    const float gscale = 0.75f, scale = 1.f / 3.f;
    std::vector<float> ug(Bs * dim), pg(Bs * dim);
    for (int64_t b = 0; b < B; ++b)
        for (int k = 0; k < dim; ++k) ug[b * dim + k] = u_tbl[ancs[b] * rs + k], pg[b * dim + k] = i_tbl[poss[b] * rs + k];
    std::vector<int64_t> ar(Bs), idp(Bs * L1);
    for (int64_t b = 0; b < B; ++b) {
        ar[b] = b;
        for (int l = 0; l < L1; ++l) idp[b * L1 + l] = B + b;
    }
    std::vector<float> su(Bs * dim, -0.f), si(Bs * dim, -0.f);
    std::vector<std::vector<float>> sl(L1, std::vector<float>(2 * Bs * dim, -0.f));
    ssl_mix::LayerSinks sinks = {};
    for (int l = 0; l < L1; ++l) sinks.ptr[l] = sl[l].data(), sinks.stride[l] = dim;
    if (B > 0)
        emu_launch(dim3(grid), dim3(ssl_mix::kWarpsPerBlock * 32), [&]() {
            ssl_mix::mixgcf_bwd_kernel(ug.data(), dim, pg.data(), dim, ar.data(), ar.data(), idp.data(), B, L1, dim, g_nhat.data(),
                                       g_alpha.data(), g_coef.data(), &gscale, scale, su.data(), dim, si.data(), dim, sinks);
        });
    int64_t bad_bwd = 0;
    for (int64_t b = 0; b < B; ++b) {
        const float g = scale * gscale * w_coef[b];
        for (int k = 0; k < dim; ++k) {
            const float gu = g * ug[b * dim + k];
            bad_bwd += !same(su[b * dim + k], g * (w_nhat[b * dim + k] - pg[b * dim + k])) + !same(si[b * dim + k], -gu);
            for (int l = 0; l < L1; ++l) {
                const float a = w_alpha[b * L1 + l];
                bad_bwd += !same(sl[l][b * dim + k], a * gu) + !same(sl[l][(B + b) * dim + k], (1.f - a) * gu);
            }
        }
    }
    printf("B=%lld M=%d L1=%d dim=%d rs=%lld view=%d pattern=%d alpha=%d ties=%lld all_nan=%lld bad_fwd=%lld bad_bwd=%lld\n",
           (long long)B, M, L1, dim, (long long)rs, view, pattern, amode, (long long)ties, (long long)all_nan, (long long)bad_fwd,
           (long long)bad_bwd);
    if (pattern == 1 && B >= 8 && M >= 2 && ties == 0) return 3;      // the case must exercise what it names
    if (pattern == 3 && B >= 3 && all_nan == 0) return 3;
    return bad_fwd == 0 && bad_bwd == 0 ? 0 : 1;
}
