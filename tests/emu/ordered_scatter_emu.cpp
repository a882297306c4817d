// Host execution of sslrec_b200/csrc/ordered_scatter.cuh (the SAME source the library compiles for sm_90a) against a sequential
// float32 restatement of its contract, bit for bit:  sink[r] = sink[r] + (((c_p1 + c_p2) + c_p3) + ...), p1 < p2 < ... the
// positions with ids[p] == r, negative ids skipped.
// usage: ordered_scatter_emu P dim stride_extra prior pattern seed grid warps
//   pattern 0 random ids with repeats | 1 all distinct | 2 one id P times | 3 ids 0 and N-1 only | 4 random, a quarter of them -1
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <numeric>

#define SSL_HOST_EMU 1
#include "cuda_emu.h"
#include "cuda_emu_warp.h"
#include "ordered_scatter.cuh"

static uint64_t rng_state;
static inline uint32_t rnd() {
    rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
    return (uint32_t)(rng_state >> 33);
}
// values over several binades and both signs, so that the order of the adds shows in the last bits
static inline float rndv() { return ((float)(rnd() & 0xffffff) / 16777216.0f - 0.5f) * (float)(1u << (rnd() % 12)); }

int main(int argc, char **argv) {
    if (argc < 9) return 2;
    const int64_t P = atoll(argv[1]);
    const int dim = atoi(argv[2]), extra = atoi(argv[3]), prior = atoi(argv[4]), pattern = atoi(argv[5]);
    rng_state = (uint64_t)atoll(argv[6]) * 2654435761u + 7u;
    const int grid = atoi(argv[7]), warps = atoi(argv[8]);
    const int64_t N = P + 3, stride = dim + extra;

    std::vector<int64_t> ids((size_t)std::max<int64_t>(P, 1));
    for (int64_t p = 0; p < P; ++p) {
        switch (pattern) {
            case 0: ids[p] = (int64_t)(rnd() % (uint32_t)(P / 8 + 1)); break;
            case 1: ids[p] = p; break;
            case 2: ids[p] = N / 2; break;
            case 3: ids[p] = (rnd() & 1) ? 0 : N - 1; break;
            default: ids[p] = (rnd() % 4 == 0) ? -1 : (int64_t)(rnd() % (uint32_t)(P / 4 + 1)); break;
        }
    }
    if (pattern == 1)
        for (int64_t p = P - 1; p > 0; --p) std::swap(ids[p], ids[rnd() % (uint32_t)(p + 1)]);
    std::vector<int64_t> order((size_t)std::max<int64_t>(P, 1));
    std::iota(order.begin(), order.begin() + P, 0);
    std::stable_sort(order.begin(), order.begin() + P, [&](int64_t a, int64_t b) { return ids[a] < ids[b]; });

    std::vector<float> stage((size_t)std::max<int64_t>(P, 1) * dim);
    for (auto &v : stage) v = rndv();
    std::vector<float> sink((size_t)(N - 1) * stride + dim);          // exact size: one float too far is an ASan error
    for (auto &v : sink) v = prior ? rndv() : 0.f;
    std::vector<float> want = sink;

    // restatement: per sink row, the running sum of its positions' rows in position order, then one add onto the prior value
    std::vector<float> acc((size_t)N * dim, 0.f);
    std::vector<char> seen((size_t)N, 0);
    for (int64_t p = 0; p < P; ++p) {
        const int64_t r = ids[p];
        if (r < 0) continue;
        for (int k = 0; k < dim; ++k) acc[(size_t)r * dim + k] = seen[r] ? acc[(size_t)r * dim + k] + stage[(size_t)p * dim + k] : stage[(size_t)p * dim + k];
        seen[r] = 1;
    }
    for (int64_t r = 0; r < N; ++r)
        if (seen[r])
            for (int k = 0; k < dim; ++k) want[(size_t)r * stride + k] = want[(size_t)r * stride + k] + acc[(size_t)r * dim + k];

    const float *sp = stage.data();
    const int64_t *ip = ids.data(), *op = order.data();
    float *kp = sink.data();
    emu_launch(dim3((unsigned)grid), dim3((unsigned)warps * 32), [&]() { ssl_scatter::ordered_scatter_kernel(sp, ip, op, P, dim, kp, stride); });

    int64_t bad = 0;
    for (size_t i = 0; i < sink.size(); ++i) bad += memcmp(&sink[i], &want[i], 4) != 0;
    printf("P=%lld dim=%d stride=%lld prior=%d pattern=%d grid=%d warps=%d bad=%lld\n", (long long)P, dim, (long long)stride, prior, pattern,
           grid, warps, (long long)bad);
    return bad == 0 ? 0 : 1;
}
