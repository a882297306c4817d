// Host execution of sslrec_b200/csrc/ssm.cuh (the SAME source the library compiles for sm_90a): both kernels on the tables
// and ids of an input file, the outputs written to an output file that tests/test_host_ssm_emulation.py compares with the
// sequential float32 restatement of tests/ssm_oracle.py.
// usage: ssm_emu in.bin out.bin
//   in:  int64 B, M, d, u_floats, i_floats, u_off, i_off, u_stride, i_stride; float32 tau, scale, gscale;
//        float32 u_block[u_floats], i_block[i_floats]; int64 ancs[B], poss[B], cands[B * M]
//        (user table = u_block + u_off, item table = i_block + i_off, rows at id * stride)
//   out: float32 loss_b[B], s[B, M+1], w[B, M+1], nrm[B, M+2]  (forward on the tables)
//        float32 su[B, d], si[B (M+1), d]  (backward on gathered rows, identity ids, -0.0 stages: one contribution per position)
//        float32 gu[u_floats], gi[i_floats]  (backward on the tables into zeroed sinks of the tables' layout)
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "cuda_emu.h"
struct float4 {
    float x, y, z, w;
};
static std::mutex emu_atomic_mutex;
static inline void atomicAdd(float4 *p, float4 v) {         // the stages get one add per element: order never matters there
    std::lock_guard<std::mutex> lk(emu_atomic_mutex);
    p->x += v.x, p->y += v.y, p->z += v.z, p->w += v.w;
}
#include "ssm.cuh"

// exactly n floats, 16-byte aligned: one float too far is an ASan error; freed at the end of main
static std::vector<void *> emu_buffers;
static float *fbuf(int64_t n, float fill) {
    void *p = nullptr;
    if (posix_memalign(&p, 16, (size_t)(n > 0 ? n : 1) * 4) != 0) abort();
    emu_buffers.push_back(p);
    float *f = static_cast<float *>(p);
    for (int64_t i = 0; i < n; ++i) f[i] = fill;
    return f;
}

template <class T>
static void rd(FILE *f, T *p, size_t n) {
    if (n && fread(p, sizeof(T), n, f) != n) {
        fprintf(stderr, "short input\n");
        exit(2);
    }
}

int main(int argc, char **argv) {
    if (argc < 3) return 2;
    FILE *in = fopen(argv[1], "rb");
    if (!in) return 2;
    int64_t h[9];
    rd(in, h, 9);
    const int64_t B = h[0], n_u = h[3], n_i = h[4], u_off = h[5], i_off = h[6], us = h[7], is = h[8];
    const int M = (int)h[1], d = (int)h[2];
    float sc[3];
    rd(in, sc, 3);
    const float tau = sc[0], scale = sc[1], gscale = sc[2];
    float *ub = fbuf(n_u, 0.f), *ib = fbuf(n_i, 0.f);
    rd(in, ub, (size_t)n_u);
    rd(in, ib, (size_t)n_i);
    std::vector<int64_t> ancs(B), poss(B), cands(B * M);
    rd(in, ancs.data(), (size_t)B);
    rd(in, poss.data(), (size_t)B);
    rd(in, cands.data(), (size_t)(B * M));
    fclose(in);
    const float *ut = ub + u_off, *it = ib + i_off;
    const int64_t Q = M + 1;
    float *loss = fbuf(B, -7.f), *s = fbuf(B * Q, -7.f), *w = fbuf(B * Q, -7.f), *nrm = fbuf(B * (Q + 1), -7.f);
    const int G = ssl_ssm::group_lanes(d);
    const int per_block = ssl_ssm::kWarpsPerBlock * (32 / G);
    const dim3 grid((unsigned)((B + per_block - 1) / per_block)), block(ssl_ssm::kWarpsPerBlock * 32);
    emu_launch(grid, block, [&]() {
        ssl_ssm::ssm_fwd_kernel(ut, us, it, is, ancs.data(), poss.data(), cands.data(), B, M, d, tau, loss, s, w, nrm);
    });
    // staged backward: gathered rows [ug], [I[poss]; I[cands]], identity ids
    float *ug = fbuf(B * d, 0.f), *ig = fbuf(B * Q * d, 0.f);
    std::vector<int64_t> ar(B), ci(B * M);
    for (int64_t b = 0; b < B; ++b) {
        ar[b] = b;
        memcpy(ug + b * d, ut + ancs[b] * us, 4 * (size_t)d);
        memcpy(ig + b * d, it + poss[b] * is, 4 * (size_t)d);
        for (int j = 0; j < M; ++j) {
            ci[b * M + j] = B + b * M + j;
            memcpy(ig + (B + b * M + j) * d, it + cands[b * M + j] * is, 4 * (size_t)d);
        }
    }
    float *su = fbuf(B * d, -0.f), *si = fbuf(B * Q * d, -0.f);
    emu_launch(grid, block, [&]() {
        ssl_ssm::ssm_bwd_kernel(ug, d, ig, d, ar.data(), ar.data(), ci.data(), B, M, d, tau, s, w, nrm, &gscale, scale, su, d, si, d);
    });
    // backward on the tables themselves
    float *gu = fbuf(n_u, 0.f), *gi = fbuf(n_i, 0.f);
    emu_launch(grid, block, [&]() {
        ssl_ssm::ssm_bwd_kernel(ut, us, it, is, ancs.data(), poss.data(), cands.data(), B, M, d, tau, s, w, nrm, &gscale, scale, gu + u_off,
                                us, gi + i_off, is);
    });
    FILE *out = fopen(argv[2], "wb");
    if (!out) return 2;
    fwrite(loss, 4, (size_t)B, out);
    fwrite(s, 4, (size_t)(B * Q), out);
    fwrite(w, 4, (size_t)(B * Q), out);
    fwrite(nrm, 4, (size_t)(B * (Q + 1)), out);
    fwrite(su, 4, (size_t)(B * d), out);
    fwrite(si, 4, (size_t)(B * Q * d), out);
    fwrite(gu, 4, (size_t)n_u, out);
    fwrite(gi, 4, (size_t)n_i, out);
    fclose(out);
    for (void *p : emu_buffers) free(p);
    return 0;
}
