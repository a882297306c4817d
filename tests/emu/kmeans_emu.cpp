// Host execution of sslrec_b200/csrc/kmeans_assign.cuh (the SAME source the library compiles for sm_90a): the R = 4 instantiation
// against the R = 1 one (bit for bit: assignments, per-CTA partial sums and counts, change counter) and against a plain restatement
// of one Lloyd assignment pass (aug_utils.py:150-155).  usage: kmeans_emu n dim K n_cta W seed
#include <stdio.h>
#include <stdlib.h>

#define SSL_HOST_EMU 1
#include "cuda_emu.h"
#include "kmeans_assign.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
static inline float rndf() { return (float)(rnd() & 0xffffff) / 16777216.0f; }

struct Out {
    std::vector<int64_t> assign;
    std::vector<float> part_sum, part_cnt;
    int changed = 0;
};

template <int R>
static Out run(const std::vector<float> &x, int64_t stride, int64_t n, int dim, int K, const std::vector<float> &cents, int n_cta, int W,
               const std::vector<int64_t> &assign0) {
    Out o;
    o.assign = assign0;
    o.part_sum.assign((size_t)n_cta * K * dim, -1.f);
    o.part_cnt.assign((size_t)n_cta * K, -1.f);
    std::vector<float> smem(ssl_kmeans::smem_floats(K, dim, W, R));      // exact size: one float too far is an ASan error
    emu_dyn_smem_ptr = smem.data();
    const int64_t rows_per_cta = (n + n_cta - 1) / n_cta, rows_per_warp = (rows_per_cta + W - 1) / W;
    const float *xp = x.data(), *cp = cents.data();
    int64_t *ap = o.assign.data();
    float *ps = o.part_sum.data(), *pc = o.part_cnt.data();
    int *ch = &o.changed;
    emu_launch(dim3((unsigned)n_cta), dim3((unsigned)W * 32), [&]() {
        ssl_kmeans::kmeans_assign_kernel<R>(xp, stride, n, dim, K, cp, ap, ps, pc, ch, rows_per_cta, rows_per_warp);
    });
    return o;
}

int main(int argc, char **argv) {
    if (argc < 7) return 2;
    const int64_t n = atoll(argv[1]);
    const int dim = atoi(argv[2]), K = atoi(argv[3]), n_cta = atoi(argv[4]), W = atoi(argv[5]);
    rng_state = (uint64_t)atoll(argv[6]) * 2654435761u + 99u;
    const int64_t stride = dim + (rnd() % 3);
    std::vector<float> x((size_t)((n - 1) * stride + dim)), cents((size_t)K * dim);
    for (auto &v : x) v = rndf();
    for (auto &v : cents) v = rndf();
    if (K > 2)                                                       // two identical centroids: exact distance ties -> lowest id
        for (int j = 0; j < dim; ++j) cents[(size_t)(K - 1) * dim + j] = cents[j];
    std::vector<int64_t> assign0((size_t)n);
    for (auto &a : assign0) a = (int64_t)(rnd() % K) - (rnd() % 4 == 0 ? 1 : 0);

    const Out a = run<1>(x, stride, n, dim, K, cents, n_cta, W, assign0);
    const Out b = run<4>(x, stride, n, dim, K, cents, n_cta, W, assign0);
    int64_t bad = 0;
    bad += a.assign != b.assign;
    bad += a.changed != b.changed;
    bad += memcmp(a.part_sum.data(), b.part_sum.data(), a.part_sum.size() * 4) != 0;
    bad += memcmp(a.part_cnt.data(), b.part_cnt.data(), a.part_cnt.size() * 4) != 0;

    // restatement: nearest centroid by the sequential fp32 chain, lowest id on ties; members counted and summed in double
    std::vector<double> sum((size_t)K * dim, 0.0), cnt((size_t)K, 0.0);
    int changed = 0;
    for (int64_t r = 0; r < n; ++r) {
        float best = INFINITY;
        int bk = 0;
        for (int k = 0; k < K; ++k) {
            float d2 = 0.f;
            for (int j = 0; j < dim; ++j) {
                const float t = x[r * stride + j] - cents[(size_t)k * dim + j];
                d2 = fmaf(t, t, d2);
            }
            if (d2 < best) {
                best = d2;
                bk = k;
            }
        }
        if (b.assign[r] != bk) ++bad;
        if (assign0[r] != bk) ++changed;
        cnt[bk] += 1.0;
        for (int j = 0; j < dim; ++j) sum[(size_t)bk * dim + j] += x[r * stride + j];
    }
    if (changed != b.changed) ++bad;
    double worst = 0.0;
    for (int k = 0; k < K; ++k) {
        double c = 0.0;
        for (int q = 0; q < n_cta; ++q) c += b.part_cnt[(size_t)q * K + k];
        if (c != cnt[k]) ++bad;
        for (int j = 0; j < dim; ++j) {
            double s = 0.0;
            for (int q = 0; q < n_cta; ++q) s += b.part_sum[((size_t)q * K + k) * dim + j];
            const double err = fabs(s - sum[(size_t)k * dim + j]);
            if (err > worst) worst = err;
            if (err > 1e-3 * (1.0 + fabs(sum[(size_t)k * dim + j])) * 1e-2) ++bad;
        }
    }
    printf("n=%lld dim=%d K=%d ctas=%d W=%d changed=%d worst_sum_err=%.3e bad=%lld\n", (long long)n, dim, K, n_cta, W, b.changed, worst,
           (long long)bad);
    return bad == 0 ? 0 : 1;
}
