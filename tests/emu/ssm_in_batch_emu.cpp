// Host execution of sslrec_b200/csrc/ssm_in_batch.cuh (the SAME source the library compiles for sm_90a) against a sequential
// float32 restatement of its documented order, bit for bit:
//     d[k] = ((0 + part[0, c, k]) + part[1, c, k]) + ...;  d[k] = d[k] * w[c];
//     proj = the xor butterfly over the 32 lanes of chain_l = fmaf(t[l + 96] d[l + 96], .. fmaf(t[l] d[l], 0));
//     sink[row_c] += rinv[c] * fmaf(-t[k], proj, d[k])
// usage: ssm_in_batch_emu n n_split dim stride_extra mode seed
//   mode 0: ids = NULL into a -0.0 stage (row c)        1: ids a permutation of the sink rows, onto a random prior sink
//        2: ids with repeats (atomic order free: checked against the restatement's per-row sums to 1e-6 of the
//        magnitudes summed)
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "cuda_emu.h"
#include "cuda_emu_warp.h"
static std::mutex emu_atomic_mutex;
static inline float atomicAdd(float *p, float v) {
    std::lock_guard<std::mutex> lk(emu_atomic_mutex);
    const float old = *p;
    *p = old + v;
    return old;
}
#include "ssm_in_batch.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndv() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * (float)(1u << (rnd() % 8)); }

int main(int argc, char **argv) {
    if (argc < 7) return 2;
    const int64_t n = atoll(argv[1]);
    const int n_split = atoi(argv[2]), dim = atoi(argv[3]), extra = atoi(argv[4]), mode = atoi(argv[5]);
    rng_state = (uint64_t)atoll(argv[6]) * 2654435761u + 11u;
    const int64_t stride = dim + extra;
    const int64_t n_rows = mode == 2 ? std::max<int64_t>(n / 3, 1) : n;

    std::vector<float> part((size_t)n_split * n * dim), t_hat((size_t)n * dim), rinv((size_t)n), colw((size_t)n);
    for (auto &v : part) v = rndv();
    for (int64_t c = 0; c < n; ++c) {           // unit-ish rows, weights over many binades (the table's range)
        float ss = 0.f;
        for (int k = 0; k < dim; ++k) ss += (t_hat[c * dim + k] = rndv()) * t_hat[c * dim + k];
        const float s = 1.f / sqrtf(ss + 1e-8f);
        for (int k = 0; k < dim; ++k) t_hat[c * dim + k] *= s;
        rinv[c] = 0.25f + (float)(rnd() % 1000) / 100.f;
        colw[c] = ldexpf(1.f + (float)(rnd() % 1024) / 1024.f, (int)(rnd() % 28) - 14);
    }
    std::vector<int64_t> ids((size_t)n);
    for (int64_t c = 0; c < n; ++c) ids[c] = mode == 2 ? (int64_t)(rnd() % (uint32_t)n_rows) : c;
    if (mode == 1)
        for (int64_t c = n - 1; c > 0; --c) std::swap(ids[c], ids[rnd() % (uint32_t)(c + 1)]);
    std::vector<float> sink((size_t)(n_rows - 1) * stride + dim);          // exact size: one float too far is an ASan error
    for (auto &v : sink) v = mode == 0 ? -0.0f : rndv();

    // restatement, column by column, lanes as the kernel holds them
    std::vector<double> want_acc(sink.size(), 0.0), want_abs(sink.size(), 0.0);
    std::vector<float> want = sink;
    for (int64_t c = 0; c < n; ++c) {
        float d[128], t[128], v[128];
        for (int k = 0; k < dim; ++k) {
            float a = 0.f;
            for (int s = 0; s < n_split; ++s) a = a + part[((size_t)s * n + c) * dim + k];
            d[k] = a * colw[c];
            t[k] = t_hat[c * dim + k];
        }
        float lanes[32];
        for (int l = 0; l < 32; ++l) {
            float ch = 0.f;
            for (int i = 0; i < 4; ++i) {
                const int k = l + 32 * i;
                ch = fmaf(k < dim ? t[k] : 0.f, k < dim ? d[k] : 0.f, ch);
            }
            lanes[l] = ch;
        }
        for (int o = 16; o > 0; o >>= 1) {
            float nx[32];
            for (int l = 0; l < 32; ++l) nx[l] = lanes[l] + lanes[l ^ o];
            memcpy(lanes, nx, sizeof(lanes));
        }
        const float proj = lanes[0];
        for (int k = 0; k < dim; ++k) v[k] = rinv[c] * fmaf(-t[k], proj, d[k]);
        const int64_t row = mode == 0 ? c : ids[c];
        for (int k = 0; k < dim; ++k) {
            want[row * stride + k] = want[row * stride + k] + v[k];
            want_acc[row * stride + k] += (double)v[k];
            want_abs[row * stride + k] += fabs((double)v[k]);
        }
    }

    const float *pp = part.data(), *tp = t_hat.data(), *rp = rinv.data(), *wp = colw.data();
    const int64_t *ip = mode == 0 ? nullptr : ids.data();
    float *sp = sink.data();
    const unsigned blocks = (unsigned)((n + ssl_inb::kWarpsPerBlock - 1) / ssl_inb::kWarpsPerBlock);
    std::vector<float> prior = sink;
    emu_launch(dim3(blocks), dim3(ssl_inb::kWarpsPerBlock * 32),
               [&]() { ssl_inb::nce_bwd_cols_kernel(pp, n_split, tp, rp, wp, ip, n, dim, sp, stride); });

    int64_t bad = 0;
    for (size_t i = 0; i < sink.size(); ++i) {
        if (mode < 2) {
            bad += memcmp(&sink[i], &want[i], 4) != 0;
        } else {
            const double ref = (double)prior[i] + want_acc[i];
            bad += fabs((double)sink[i] - ref) > 1e-6 * (fabs((double)prior[i]) + want_abs[i]);
        }
    }
    printf("n=%lld n_split=%d dim=%d stride=%lld mode=%d bad=%lld\n", (long long)n, n_split, dim, (long long)stride, mode, (long long)bad);
    return bad == 0 ? 0 : 1;
}
