// More warp-level primitives for tests/emu/cuda_emu.h (include it first): __shfl_sync, __shfl_up_sync and __ballot_sync as two waits on
// the warp's barrier around its exchange buffer, __popc / __ffs, the float <-> bit casts, and unsigned shared-memory atomics.  The
// kernels that use them call them from warp-uniform control flow, on whole warps.  Test infrastructure only.
#pragma once
#include "cuda_emu.h"

template <class T>
static inline T __shfl_sync(unsigned, T v, int src_lane) {
    static_assert(sizeof(T) == 4, "32-bit shuffles only");
    const int w = emu_linear_tid() >> 5, l = emu_linear_tid() & 31;
    memcpy(&emu_xchg[w][l], &v, 4);
    pthread_barrier_wait(&emu_warp_barrier[w]);
    T r;
    memcpy(&r, &emu_xchg[w][src_lane & 31], 4);
    pthread_barrier_wait(&emu_warp_barrier[w]);
    return r;
}
template <class T>
static inline T __shfl_up_sync(unsigned, T v, unsigned delta) {
    static_assert(sizeof(T) == 4, "32-bit shuffles only");
    const int w = emu_linear_tid() >> 5, l = emu_linear_tid() & 31;
    memcpy(&emu_xchg[w][l], &v, 4);
    pthread_barrier_wait(&emu_warp_barrier[w]);
    T r = v;
    if (l >= (int)delta) memcpy(&r, &emu_xchg[w][l - (int)delta], 4);
    pthread_barrier_wait(&emu_warp_barrier[w]);
    return r;
}
static inline unsigned __ballot_sync(unsigned, int pred) {
    const int w = emu_linear_tid() >> 5, l = emu_linear_tid() & 31;
    emu_xchg[w][l] = pred ? 1u : 0u;
    pthread_barrier_wait(&emu_warp_barrier[w]);
    unsigned r = 0;
    for (int q = 0; q < 32; ++q) r |= emu_xchg[w][q] << q;
    pthread_barrier_wait(&emu_warp_barrier[w]);
    return r;
}
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline unsigned __float_as_uint(float f) {
    unsigned u;
    memcpy(&u, &f, 4);
    return u;
}
static inline float __uint_as_float(unsigned u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}
static inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
