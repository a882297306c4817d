// ssl_softmax_gemm_f16x3: the InfoNCE contraction on the Hopper tensor cores (wgmma, f16 inputs, f32 accumulation) with
// fp32-grade accuracy through 3xFP16 error compensation with scaled residuals (f16x3.cuh: x = hi + 2^-12 lo).
//
//   S  = R C^T   = R_hi C_hi^T + 2^-12 (R_lo C_hi^T + R_hi C_lo^T)
//   E' = exp2(S - offset) * colscale * 2^14 / M ;  rowsum' += sum_c E'          (M: a power of two >= max |colscale|)
//   E' = exp2(S - (offset - 14))                       without colscale (M = 1): the bias folded into the offset
//   O' = E' C    = E'_hi C_hi + 2^-12 (E'_lo C_hi + E'_hi C_lo) ;    O = O' M 2^-14, rowsum = rowsum' M 2^-14
//
// Same contract as ssl_softmax_gemm_tf32x3 (nce_gemm_tc.cu) and ssl_softmax_gemm (nce_gemm.cu), at twice the tf32 MMA rate.
// The same structure as softmax_gemm_tc_kernel: persistent (min(units, #SMs) CTAs of 384 threads, unit u = R tile
// u / n_split against C chunk u % n_split, CTA b runs units b, b + gridDim.x, ...), one TMA producer thread, two consumer
// warpgroups of 64 rows with ping-pong MMA issue, and a ring that runs on across units.  What fp16 changes:
// * One copy of the C tile serves both GEMMs.  A ring stage is the row-major C_hi and C_lo tiles (64 rows x d fp16,
//   SWIZZLE_128B at d = 64, 64B at d = 32): GEMM1 reads them K-major (B = C^T), GEMM2 reads the same bytes MN-major
//   (imm-trans-b, B = C), which wgmma allows for 16-bit types only.  16 KB per tile at d = 64 instead of 64 KB.
// * The f32 accumulator fragment of an m64nNk16 GEMM has the layout of the f16 A fragment of the next k16 step in
//   natural column order, so E goes from GEMM1's accumulator to GEMM2's A registers without a lane exchange.
// * GEMM1's correction products go to their own accumulator SC, added as S = S_hi + 2^-12 SC in the exp phase.  Folding
//   them into one accumulator would need R_hi pre-scaled by 2^12, which overflows fp16 at the operand bound |x| = 16
//   (2^16 > 65504); the extra 32 registers fit (no spills).  GEMM2's corrections go to OC as in the tf32 kernel: the
//   tensor core does not round its fp32 accumulation to nearest, so the long hi*hi sum must not also carry them.
// * colscale (the backward role: g ln2 / rowsum, ~1e-9) lies below fp16's range.  Every CTA's consumers scan
//   colscale[0, n_c) in the prologue for M, a power of two >= its largest magnitude, and E' carries colscale / M with an
//   exponent bias of 2^14, so E' <= 2^14 and its hi part is a normal fp16 down to E' = 2^-14.  All of these scalings are
//   exact, need no host read-back (CUDA-graph capture), and every grid size finds the same M.
// * The exp phase runs while the other warpgroup's two GEMMs (768 tensor-core clocks at the data-sheet rate) run, and
//   it took longer than that (profiles/r09_nce_exp_phase.md).  So each launch takes an exp phase specialised for its role
//   (kExp* flags): the forward folds the 2^14 into the offset and, up to offset 13.5, drops the flush rule, which cannot
//   fire there (f16x3.cuh); the backward does not sum the row sums nobody reads, and computes O as it always has.
// Units write disjoint o_part / rowsum_part slices and the order of every sum is fixed: no atomics, bit-identical results
// from launch to launch and for every grid size.
#include <cuda_fp16.h>
#include <cmath>

#include "sm90.cuh"
#include "f16x3.cuh"

namespace {

constexpr int BM = 128, BN = 64;
constexpr int kNumThreads = 384;       // warpgroup 0: TMA producer; warpgroups 1, 2: consumers (64 rows each)

template <int D> struct Cfg {
    static constexpr uint32_t ROW_BYTES = D * 2;                // one fp16 row of the tile: 128 B at d = 64, 64 B at d = 32
    static constexpr uint32_t PART_BYTES = BN * ROW_BYTES;      // one precision part of a 64-row tile
    static constexpr uint32_t STAGE_BYTES = 2 * PART_BYTES;     // C_hi, C_lo
    static constexpr uint32_t GROUP = 8 * ROW_BYTES;            // 8-row core-matrix group = one swizzle repeat
    static constexpr uint64_t SWIZZLE = (D == 64) ? 1 : 2;      // descriptor layout type: 1 = 128B, 2 = 64B swizzle
    static constexpr int ST = (D == 32) ? 16 : 10;              // ring stages: 10 x 16 KB at d = 64, 16 x 8 KB at d = 32
    static constexpr size_t SMEM = 1024 + (size_t)ST * STAGE_BYTES + 2 * ST * sizeof(uint64_t);
};

#ifdef SSL_NCE_PHASES
// Instrumented build (tools/nce_phases.py only, never part of the library): each consumer warpgroup sums the clock64()
// cycles it spends in each phase of its tile loop; thread 0 of the warpgroup writes the sums to g_phases[CTA][cw][phase]
// at the end, read back once by ssl_nce_phases_read.
enum Phase { kPhFull, kPhBar1, kPhIssue1, kPhWait1, kPhExp, kPhBar2, kPhIssue2, kPhWait2, kPhOther, kPhTiles, kNumPhases };
constexpr int kPhaseCtas = 256;
__device__ unsigned long long g_phases[kPhaseCtas * 2 * kNumPhases];
#define SSL_PHASE(k)                                \
    do {                                            \
        const unsigned long long t_ = clock64();    \
        ph[k] += t_ - ph_t;                         \
        ph_t = t_;                                  \
    } while (0)
#else
#define SSL_PHASE(k) do { } while (0)
#endif

// ---- wgmma (sm_90a) ----
// Shared-memory matrix descriptors over a tile of 64 rows x D fp16, rows ROW_BYTES apart, swizzled by the TMA in repeats
// of 8 rows (GROUP bytes).
// K-major (GEMM1, B = C^T: K = the d features of a row): 8-row groups GROUP bytes apart; a k16 step inside the swizzle
// atom advances the start address by 32 bytes.  The leading offset is unused for swizzled K-major layouts.
template <int D>
__device__ __forceinline__ uint64_t desc_k(uint32_t addr) {
    using K = Cfg<D>;
    return (uint64_t)((addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(K::GROUP >> 4) << 32) | (K::SWIZZLE << 62);
}
// MN-major (GEMM2, B = C: K = the 64 rows, N = the d features, contiguous): N = d is one swizzle atom wide, so only the
// stride between 8-row K groups matters; it is GROUP bytes, given as both offsets.  A k16 step is 16 rows.
template <int D>
__device__ __forceinline__ uint64_t desc_mn(uint32_t addr) {
    using K = Cfg<D>;
    return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(K::GROUP >> 4) << 16) | ((uint64_t)(K::GROUP >> 4) << 32) | (K::SWIZZLE << 62);
}
// GEMM1: d[64 x 64] (+)= A[registers, one k16 block] * B[smem, K-major]^T
__device__ __forceinline__ void wgmma_k_n64(float (&d)[32], const uint32_t *a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
// GEMM2: d[64 x 64] += A[registers, one k16 block] * B[smem, MN-major]
__device__ __forceinline__ void wgmma_t_n64(float (&d)[32], const uint32_t *a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
// GEMM2: d[64 x 32] += A[registers, one k16 block] * B[smem, MN-major]
__device__ __forceinline__ void wgmma_t_n32(float (&d)[16], const uint32_t *a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <int D>
__device__ __forceinline__ void wgmma_t(float (&d)[D / 2], const uint32_t *a, uint64_t b) {
    if constexpr (D == 64) wgmma_t_n64(d, a, b);
    else wgmma_t_n32(d, a, b);
}

// What the exp phase computes, fixed per launch (launch_f16x3 picks it from the arguments), so that each role issues
// only the instructions it needs:
constexpr int kExpColscale = 1;   // colscale != nullptr (the backward): E' = exp2(S - offset) * colscale * 2^14 / M
                                  // without it (the forward) M = 1 and E' = exp2(S - (offset - 14)): the 2^14 is in the offset
constexpr int kExpRowsum = 2;     // the row sums are summed (rowsum_part != nullptr, or no colscale)
constexpr int kExpFlush = 4;      // E' can fall below 2^-14, so hi goes through the flush rule (colscale, or offset > 13.5)

// One 64-column tile: accumulators s / sc (s[4j + 2h + c] = S(row g + 8h, col 8j + 2t + c), g = lane / 4, t = lane % 4)
// -> E', the two row sums, and E' split into GEMM2's f16 A fragments.  The A fragment of k16 block kk holds
// a[4kk + 2i + h] = E'(row g + 8h, cols 16kk + 8i + 2t + {0, 1}), i.e. the accumulator pair of column group j = 2kk + i.
// With colscale, cscale = 2^14 / M scales it and offset is the caller's; without, offset is already offset - 14.
template <bool CHECK, int EXP>
__device__ __forceinline__ void exp_tile(const float (&s)[32], const float (&sc)[32], uint32_t (&ahi)[16], uint32_t (&alo)[16],
                                         float offset, const float *__restrict__ cs_ptr, float cscale, int64_t col0, int64_t n_c,
                                         float (&rowsum)[2]) {
    constexpr bool COLSCALE = EXP & kExpColscale, ROWSUM = EXP & kExpRowsum, FLUSH = EXP & kExpFlush;
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int64_t col = col0 + 8 * j + 2 * t;
        float cs0 = 1.f, cs1 = 1.f;
        if constexpr (COLSCALE) {
            if (!CHECK) {
                const float2 c2 = __ldg(reinterpret_cast<const float2 *>(cs_ptr + col));
                cs0 = c2.x * cscale; cs1 = c2.y * cscale;
            } else {
                cs0 = col < n_c ? __ldg(cs_ptr + col) * cscale : 0.f;
                cs1 = col + 1 < n_c ? __ldg(cs_ptr + col + 1) * cscale : 0.f;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float x0 = fmaf(sc[4 * j + 2 * h], ssl::kF16LoUnscale, s[4 * j + 2 * h]);
            const float x1 = fmaf(sc[4 * j + 2 * h + 1], ssl::kF16LoUnscale, s[4 * j + 2 * h + 1]);
            float e0 = ssl::ex2(x0 - offset), e1 = ssl::ex2(x1 - offset);
            if constexpr (COLSCALE) {
                e0 *= cs0;
                e1 *= cs1;
            }
            if (CHECK) {
                e0 = (col < n_c) ? e0 : 0.f;
                e1 = (col + 1 < n_c) ? e1 : 0.f;
            }
            if constexpr (ROWSUM) rowsum[h] += e0 + e1;
            const int q = 4 * (j >> 1) + 2 * (j & 1) + h;
            ssl::f16x3_split2<FLUSH>(e0, e1, ahi[q], alo[q]);
        }
    }
}

// LIVE selects a device-side bound (ssl_softmax_gemm_f16x3_live): 0 none (n_live unused), 1 only the first min(*n_live, n_r)
// rows of R are live, 2 only the first min(*n_live, n_c) rows of C.  n_r stays the row pitch of the outputs.  EXP: the
// kExp* flags of the exp phase; colscale is read if and only if kExpColscale is set.
template <int D, int LIVE, int EXP>
__global__ void __launch_bounds__(kNumThreads, 1)
softmax_gemm_f16x3_kernel(const __half *__restrict__ R_hi, const __half *__restrict__ R_lo,
                          const __grid_constant__ CUtensorMap map_c_hi, const __grid_constant__ CUtensorMap map_c_lo,
                          int64_t n_r, int64_t n_c_cap, const float *__restrict__ colscale, float offset, int n_split,
                          float *__restrict__ rowsum_part, float *__restrict__ o_part, const int64_t *__restrict__ n_live) {
    using K = Cfg<D>;
    // live extents: rows of R past n_r_live are neither read nor written; columns past n_c are masked like a ragged tail
    const int64_t n_r_live = (LIVE == 1) ? ssl::live_count(n_live, n_r) : n_r;
    const int64_t n_c = (LIVE == 2) ? ssl::live_count(n_live, n_c_cap) : n_c_cap;
    constexpr int ST = K::ST;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ float cs_max[8];
    uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(ring + ST * K::STAGE_BYTES);   // stage s: C hi, C lo (row-major tiles)
    uint64_t *empty = full + ST;

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const int64_t n_ct = (n_c + BN - 1) / BN;
    const int n_units = (int)((n_r_live + BM - 1) / BM) * n_split;     // unit u: R tile u / n_split, C chunk u % n_split

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c_hi));
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c_lo));
        for (int s = 0; s < ST; ++s) {
            ssl::mbar_init(&full[s], 1);
            ssl::mbar_init(&empty[s], 256);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
        if (threadIdx.x == 0) {
            // ===================== TMA producer: the hi and lo tiles of every C tile of every unit =====================
            int it = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
                const int sp = u % n_split;
                const int t0 = (int)(n_ct * sp / n_split), t1 = (int)(n_ct * (sp + 1) / n_split);
                for (int tile = t0; tile < t1; ++tile, ++it) {
                    const int s = it % ST;
                    ssl::mbar_wait(&empty[s], ((it / ST) & 1) ^ 1);
                    uint8_t *c_hi = ring + s * K::STAGE_BYTES;
                    ssl::mbar_expect_tx(&full[s], K::STAGE_BYTES);
                    ssl::tma_load_2d(c_hi, &map_c_hi, 0, tile * BN, &full[s]);
                    ssl::tma_load_2d(c_hi + K::PART_BYTES, &map_c_lo, 0, tile * BN, &full[s]);
                }
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
    // ===================== consumers: rows [64 * cw, +64) of each unit's R tile =====================
    const int cw = wg - 1, w = (threadIdx.x >> 5) & 3, g = lane >> 2, t = lane & 3;
    // ping-pong: named barrier 1 + cw is this warpgroup's turn to issue MMAs (see softmax_gemm_tc_kernel).
    const int bar_mine = 1 + cw, bar_other = 2 - cw;
    if (cw == 1) ssl::named_arrive(1);

    // M = 2^e >= max |colscale[c]|, c < n_c (frexp: m = f 2^e, f in [0.5, 1)); e is clamped so that 2^(14 - e) and
    // 2^(e - 14) stay normal floats.  Without colscale M = 1.
    int e_m = 0;
    if constexpr ((EXP & kExpColscale) != 0) {
        float m = 0.f;
        for (int64_t i = threadIdx.x - 128; i < n_c; i += 256) m = fmaxf(m, fabsf(__ldg(colscale + i)));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) cs_max[(threadIdx.x - 128) >> 5] = m;
        ssl::named_sync(3);
#pragma unroll
        for (int i = 0; i < 8; ++i) m = fmaxf(m, cs_max[i]);
        frexpf(m, &e_m);
        e_m = e_m < -100 ? -100 : (e_m > 100 ? 100 : e_m);
    }
    const float cscale = ldexpf(1.f, ssl::kF16Bias - e_m), back = ldexpf(1.f, e_m - ssl::kF16Bias);
    // without colscale, exp2(S - offset) * 2^14 = exp2(S - (offset - 14)): one subtraction per launch instead of one
    // multiplication per element
    const float offset_e = (EXP & kExpColscale) ? offset : offset - (float)ssl::kF16Bias;

    float o[D / 2], oc[D / 2], sacc[32], scor[32];
    uint32_t rhi[D / 4], rlo[D / 4], ahi[16], alo[16];
#pragma unroll
    for (int k = 0; k < 32; ++k) sacc[k] = scor[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) ahi[k] = alo[k] = 0u;
    const uint32_t *rh32 = reinterpret_cast<const uint32_t *>(R_hi), *rl32 = reinterpret_cast<const uint32_t *>(R_lo);
#ifdef SSL_NCE_PHASES
    unsigned long long ph[kNumPhases] = {}, ph_t = clock64();
#endif
    int it = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int rt = u / n_split, sp = u % n_split;
        const int t0 = (int)(n_ct * sp / n_split), t1 = (int)(n_ct * (sp + 1) / n_split);
        const int64_t row_a = (int64_t)rt * BM + 64 * cw + 16 * w + g;        // this thread's rows: row_a, row_a + 8
        // GEMM1's A operand, read once per unit straight into the f16 A fragment:
        // r[4kk + 2i + h] = R(row_a + 8h, cols 16kk + 8i + 2t + {0, 1}); rows past n_r are 0
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = row_a + 8 * h;
            const bool ok = row < n_r_live;
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int64_t at = (row * D + 16 * kk + 8 * i + 2 * t) >> 1;
                    rhi[4 * kk + 2 * i + h] = ok ? __ldg(rh32 + at) : 0u;
                    rlo[4 * kk + 2 * i + h] = ok ? __ldg(rl32 + at) : 0u;
                }
        }
#pragma unroll
        for (int k = 0; k < D / 2; ++k) o[k] = oc[k] = 0.f;
        float rowsum[2] = {0.f, 0.f};
        for (int tile = t0; tile < t1; ++tile, ++it) {
            const int s = it % ST;
            SSL_PHASE(kPhOther);
            ssl::mbar_wait(&full[s], (it / ST) & 1);
            SSL_PHASE(kPhFull);
            const uint32_t c_hi_a = ssl::smem_u32(ring + s * K::STAGE_BYTES), c_lo_a = c_hi_a + K::PART_BYTES;
            // ---- GEMM1: S = R C^T; the two correction products into SC first, then hi*hi into S ----
            ssl::named_sync(bar_mine);
            SSL_PHASE(kPhBar1);
            ssl::wg_fence();
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk) wgmma_k_n64(scor, rlo + 4 * kk, desc_k<D>(c_hi_a + 32 * kk), kk > 0 ? 1u : 0u);
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk) wgmma_k_n64(scor, rhi + 4 * kk, desc_k<D>(c_lo_a + 32 * kk), 1u);
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk) wgmma_k_n64(sacc, rhi + 4 * kk, desc_k<D>(c_hi_a + 32 * kk), kk > 0 ? 1u : 0u);
            ssl::wg_commit();
            ssl::named_arrive(bar_other);
            SSL_PHASE(kPhIssue1);
            ssl::wg_wait0();
            ssl::reg_fence(sacc);
            ssl::reg_fence(scor);
            ssl::reg_fence(rhi);
            ssl::reg_fence(rlo);
            SSL_PHASE(kPhWait1);
            // ---- E' = exp2(S - offset) * colscale * 2^14 / M, row sums, GEMM2's A fragments ----
            const int64_t col0 = (int64_t)tile * BN;
            if (col0 + BN <= n_c) exp_tile<false, EXP>(sacc, scor, ahi, alo, offset_e, colscale, cscale, col0, n_c, rowsum);
            else exp_tile<true, EXP>(sacc, scor, ahi, alo, offset_e, colscale, cscale, col0, n_c, rowsum);
            // ---- GEMM2: O' += E' C, the same tiles read MN-major (hi*hi into O, the two correction products into OC) ----
#ifdef SSL_NCE_PHASES
            ssl::reg_fence(ahi);
            ssl::reg_fence(alo);
#endif
            SSL_PHASE(kPhExp);
            ssl::named_sync(bar_mine);
            SSL_PHASE(kPhBar2);
            ssl::wg_fence();
#pragma unroll
            for (int kk = 0; kk < BN / 16; ++kk) wgmma_t<D>(oc, alo + 4 * kk, desc_mn<D>(c_hi_a + kk * 2 * K::GROUP));
#pragma unroll
            for (int kk = 0; kk < BN / 16; ++kk) wgmma_t<D>(oc, ahi + 4 * kk, desc_mn<D>(c_lo_a + kk * 2 * K::GROUP));
#pragma unroll
            for (int kk = 0; kk < BN / 16; ++kk) wgmma_t<D>(o, ahi + 4 * kk, desc_mn<D>(c_hi_a + kk * 2 * K::GROUP));
            ssl::wg_commit();
            ssl::named_arrive(bar_other);
            SSL_PHASE(kPhIssue2);
            // waiting here rather than under the next GEMM1 keeps ptxas from serialising the wgmmas
            ssl::wg_wait0();
            ssl::reg_fence(ahi);
            ssl::reg_fence(alo);
            ssl::reg_fence(o);
            ssl::reg_fence(oc);
            SSL_PHASE(kPhWait2);
#ifdef SSL_NCE_PHASES
            ++ph[kPhTiles];
#endif
            ssl::mbar_arrive(&empty[s]);                               // the tile is consumed by both GEMMs
        }

        // ---- unit epilogue: o[4j + 2h + c] = O'(row 16w + g + 8h, col 8j + 2t + c); O = (O + 2^-12 OC) M 2^-14 ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if constexpr ((EXP & kExpRowsum) != 0) {
                rowsum[h] += __shfl_xor_sync(0xffffffffu, rowsum[h], 1);
                rowsum[h] += __shfl_xor_sync(0xffffffffu, rowsum[h], 2);
            }
            const int64_t grow = row_a + 8 * h;
            if (grow >= n_r_live) continue;
            float *dst = o_part + ((size_t)sp * n_r + grow) * D;
#pragma unroll
            for (int j = 0; j < D / 8; ++j)
                *reinterpret_cast<float2 *>(dst + 8 * j + 2 * t) =
                    make_float2(fmaf(oc[4 * j + 2 * h], ssl::kF16LoUnscale, o[4 * j + 2 * h]) * back,
                                fmaf(oc[4 * j + 2 * h + 1], ssl::kF16LoUnscale, o[4 * j + 2 * h + 1]) * back);
            if ((EXP & kExpRowsum) != 0 && t == 0 && rowsum_part != nullptr) rowsum_part[(size_t)sp * n_r + grow] = rowsum[h] * back;
        }
    }
    if (cw == 0) ssl::named_sync(1);                                  // consumer 1's last hand-over
#ifdef SSL_NCE_PHASES
    SSL_PHASE(kPhOther);
    if ((threadIdx.x & 127) == 0 && blockIdx.x < kPhaseCtas)
        for (int k = 0; k < kNumPhases; ++k) g_phases[(blockIdx.x * 2 + cw) * kNumPhases + k] = ph[k];
#endif
}

template <int D, int LIVE, int EXP>
int launch_f16x3_exp(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi, const uint16_t *C_lo, int64_t n_c,
                     const float *colscale, float offset, int n_split, float *rowsum_part, float *o_part, const int64_t *n_live,
                     cudaStream_t st) {
    // [n_c, D] fp16, row-major -> boxes of D x 64 rows (one row = 128 B with SWIZZLE_128B at D = 64, 64 B with SWIZZLE_64B
    // at D = 32)
    constexpr CUtensorMapSwizzle SW = D == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    CUtensorMap mc_hi, mc_lo;
    int rc;
    if ((rc = ssl::make_map_2d(&mc_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, C_hi, n_c, D, D * 2, D, BN, SW)) != SSL_OK) return rc;
    if ((rc = ssl::make_map_2d(&mc_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, C_lo, n_c, D, D * 2, D, BN, SW)) != SSL_OK) return rc;
    const size_t smem = Cfg<D>::SMEM;
    int n_sm = 0;
    if ((rc = ssl::configure_once<softmax_gemm_f16x3_kernel<D, LIVE, EXP>>(smem, &n_sm)) != SSL_OK) return rc;
    const int64_t grid = ssl::persistent_grid(((n_r + BM - 1) / BM) * n_split, n_sm);
    softmax_gemm_f16x3_kernel<D, LIVE, EXP><<<(unsigned)grid, kNumThreads, smem, st>>>(
        reinterpret_cast<const __half *>(R_hi), reinterpret_cast<const __half *>(R_lo), mc_hi, mc_lo, n_r, n_c, colscale, offset,
        n_split, rowsum_part, o_part, n_live);
    SSL_LAUNCH_CHECK("softmax_gemm_f16x3_kernel");
    return SSL_OK;
}

// the exp phase of the launch's role: the backward (colscale, row sums unread), the forward (no colscale; E' >= 2^-13
// up to offset 13.5, so no flush), or both (colscale and row sums: every flag)
template <int D, int LIVE>
int launch_f16x3(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi, const uint16_t *C_lo, int64_t n_c,
                 const float *colscale, float offset, int n_split, float *rowsum_part, float *o_part, const int64_t *n_live,
                 cudaStream_t st) {
#define SSL_F16X3_LAUNCH(EXP) \
    launch_f16x3_exp<D, LIVE, EXP>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st)
    if (colscale != nullptr)
        return rowsum_part != nullptr ? SSL_F16X3_LAUNCH(kExpColscale | kExpRowsum | kExpFlush) : SSL_F16X3_LAUNCH(kExpColscale | kExpFlush);
    return offset <= ssl::kF16NoFlushOffset ? SSL_F16X3_LAUNCH(kExpRowsum) : SSL_F16X3_LAUNCH(kExpRowsum | kExpFlush);
#undef SSL_F16X3_LAUNCH
}

int check_f16x3_args(const uint16_t *R_hi, const uint16_t *R_lo, const uint16_t *C_hi, const uint16_t *C_lo, int64_t n_c, int32_t dim,
                     const float *colscale, float offset, int32_t n_split, const float *o_part, const char *name) {
    SSL_CHECK_ARG(R_hi && R_lo && C_hi && C_lo && o_part, "%s: null argument", name);
    SSL_CHECK_ARG(dim == 32 || dim == 64, "%s: dim %d not supported (32 or 64; other sizes use ssl_softmax_gemm)", name, dim);
    SSL_CHECK_ARG((n_split >= 1 && n_split <= (n_c + BN - 1) / BN) || n_c == 0, "%s: n_split %d exceeds the number of C tiles", name, n_split);
    SSL_CHECK_ARG(offset >= 0.f && offset <= ssl::kF16MaxOffset, "%s: offset %g outside [0, %g] (larger offsets use ssl_softmax_gemm_tf32x3)",
                  name, (double)offset, (double)ssl::kF16MaxOffset);
    SSL_CHECK_ARG(((reinterpret_cast<uintptr_t>(R_hi) | reinterpret_cast<uintptr_t>(R_lo) | reinterpret_cast<uintptr_t>(C_hi) |
                    reinterpret_cast<uintptr_t>(C_lo) | reinterpret_cast<uintptr_t>(o_part)) & 15) == 0,
                  "%s: operands must be 16-byte aligned", name);
    SSL_CHECK_ARG((reinterpret_cast<uintptr_t>(colscale) & 7) == 0, "%s: colscale must be 8-byte aligned", name);
    return SSL_OK;
}

}  // namespace

#ifdef SSL_NCE_PHASES
// copies the per-warpgroup phase sums of the last launch (kPhaseCtas x 2 x kNumPhases) to host memory and clears them
extern "C" int ssl_nce_phases_read(unsigned long long *host, int n) {
    SSL_CHECK_ARG(n == kPhaseCtas * 2 * kNumPhases, "ssl_nce_phases_read: n must be %d", kPhaseCtas * 2 * kNumPhases);
    SSL_CUDA(cudaMemcpyFromSymbol(host, g_phases, sizeof(g_phases)));
    static const unsigned long long zero[kPhaseCtas * 2 * kNumPhases] = {};
    SSL_CUDA(cudaMemcpyToSymbol(g_phases, zero, sizeof(g_phases)));
    return SSL_OK;
}
#endif

extern "C" int ssl_softmax_gemm_f16x3(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi, const uint16_t *C_lo,
                                      int64_t n_c, int32_t dim, const float *colscale, float offset, int32_t n_split, float *rowsum_part,
                                      float *o_part, void *stream) {
    const int rc = check_f16x3_args(R_hi, R_lo, C_hi, C_lo, n_c, dim, colscale, offset, n_split, o_part, "ssl_softmax_gemm_f16x3");
    if (rc != SSL_OK) return rc;
    if (n_r == 0 || n_c == 0) return SSL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dim == 32) return launch_f16x3<32, 0>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, nullptr, st);
    return launch_f16x3<64, 0>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, nullptr, st);
}

extern "C" int ssl_softmax_gemm_f16x3_live(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi,
                                           const uint16_t *C_lo, int64_t n_c, int32_t dim, const float *colscale, float offset,
                                           int32_t n_split, float *rowsum_part, float *o_part, const int64_t *n_live, int32_t live_role,
                                           void *stream) {
    const int rc = check_f16x3_args(R_hi, R_lo, C_hi, C_lo, n_c, dim, colscale, offset, n_split, o_part, "ssl_softmax_gemm_f16x3_live");
    if (rc != SSL_OK) return rc;
    SSL_CHECK_ARG(n_live != nullptr, "ssl_softmax_gemm_f16x3_live: null n_live");
    SSL_CHECK_ARG(live_role == SSL_LIVE_ROWS || live_role == SSL_LIVE_COLS, "ssl_softmax_gemm_f16x3_live: bad live_role %d", live_role);
    if (n_r == 0 || n_c == 0) return SSL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (live_role == SSL_LIVE_ROWS) {
        if (dim == 32) return launch_f16x3<32, 1>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
        return launch_f16x3<64, 1>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
    }
    if (dim == 32) return launch_f16x3<32, 2>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
    return launch_f16x3<64, 2>(R_hi, R_lo, n_r, C_hi, C_lo, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
}
