// ssl_softmax_gemm_tf32x3: the InfoNCE contraction on the Hopper tensor cores (wgmma, tf32) with
// fp32-grade accuracy through 3xTF32 error compensation.
//
//   S  = R C^T   = R_hi C_hi^T + R_lo C_hi^T + R_hi C_lo^T          (x = x_hi + x_lo, x_hi = tf32(x))
//   E  = exp2(S - offset) * colscale ;  rowsum += sum_c E
//   O += E C     = E_hi C_hi   + E_lo C_hi   + E_hi C_lo
//
// Same contract as ssl_softmax_gemm (nce_gemm.cu): one launch is the forward of an InfoNCE term or,
// with the operand roles swapped, its backward.  Both parts are rounded to nearest (cvt.rna.tf32), so the
// dropped lo*lo products and the rounding of the lo parts are O(2^-22) relative and unbiased -- the fp32
// rounding level of the FFMA kernel.
//
// Structure (persistent: min(units, #SMs) CTAs of 384 threads = 3 warpgroups; a unit is one 128-row R tile against
// one of the n_split chunks of C, and CTA b runs units b, b + gridDim.x, ... in that static order):
//   warpgroup 0, one thread : TMA producer.  2-D tensor maps (SWIZZLE_128B, 32-float boxes) over the row-major
//                     hi / lo C arrays: per 64-row C tile one ring stage holding the row-major C tile (GEMM1's B
//                     operand) and the tile of the TRANSPOSED copy [d, n] (GEMM2's B operand).  wgmma reads tf32
//                     operands from shared memory K-major only, which is why both copies are streamed.  The ring
//                     runs on across units, so the next unit's first tiles load under the current unit's last ones.
//   warpgroups 1, 2 : consumers, 64 rows of the unit's R tile each.  At the start of a unit each thread loads its
//                     R_hi / R_lo rows from global memory straight into the tf32 A fragment, so shared memory holds
//                     only the C ring.  Per C tile: GEMM1 (m64 n64 k8, A = R from registers) -> S in registers;
//                     E = exp2(S - offset) with the row sums in registers, split into tf32 hi / lo in place: the
//                     accumulator fragment of S serves as GEMM2's A fragment as it is, because the transposed copy
//                     holds its columns in the matching order (see exp_tile);
//                     GEMM2 (m64 nD k8, A = E from registers, B = C^T tile) accumulates O, written out per unit.
//                     Two named barriers hand the MMA issue back and forth (ping-pong), so one warpgroup's exp
//                     phase runs under the other's MMAs.
//   Units write disjoint o_part / rowsum_part slices and the order of every sum is fixed, so the output does not
//   depend on the grid size or on timing.
//   The two correction products of GEMM2 go to their own accumulator: the tensor core does not round its fp32
//   accumulations to nearest, so the long hi*hi sum must not also carry them.
#include <cstdlib>

#include "sm90.cuh"

namespace {

constexpr int BM = 128, BN = 64;
constexpr int kNumThreads = 384;       // warpgroup 0: TMA producer; warpgroups 1, 2: consumers (64 rows each)

template <int D> struct Cfg {
    static constexpr int KCH = D / 32;                  // 128-byte K chunks per operand row (GEMM1: K = d)
    static constexpr int JCH = BN / 32;                 // 128-byte K chunks of the transposed tile (GEMM2: K = 64 rows)
    static constexpr uint32_t C_CHUNK = BN * 128, T_CHUNK = D * 128;
    static constexpr uint32_t C_BYTES = KCH * C_CHUNK, T_BYTES = JCH * T_CHUNK;   // one precision part
    static constexpr uint32_t STAGE_BYTES = 2 * C_BYTES + 2 * T_BYTES;
    static constexpr int ST = (D == 32) ? 6 : 3;        // ring stages: 3 x 64 KB at d = 64, 6 x 32 KB at d = 32
    static constexpr size_t SMEM = 1024 + (size_t)ST * STAGE_BYTES + 2 * ST * sizeof(uint64_t);
};

// ---- wgmma (sm_90a) ----
// shared-memory matrix descriptor: K-major, SWIZZLE_128B (layout type 1), 8-row core-matrix groups 1024 bytes apart.
// A K step of 8 tf32 inside the 128-byte swizzle atom advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t wg_desc(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// d[64 x 64] (+)= A[registers, one k8 block] * B[smem]^T
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t *a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
// d[64 x 64] += A[registers, one k8 block] * B[smem]^T
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t *a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
// d[64 x 32] += A[registers, one k8 block] * B[smem]^T
__device__ __forceinline__ void wgmma_rs_n32(float (&d)[16], const uint32_t *a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <int D>
__device__ __forceinline__ void wgmma_rs(float (&d)[D / 2], const uint32_t *a, uint64_t b) {
    if constexpr (D == 64) wgmma_rs_n64(d, a, b);
    else wgmma_rs_n32(d, a, b);
}

// One 64-column tile of S (accumulator fragment: s[4j + 2h + c] = S(row g + 8h, col 8j + 2t + c), g = lane / 4,
// t = lane % 4) -> E, the two row sums, and E as GEMM2's A fragment in tf32 hi / lo: a[4j + 2c + h] = E(g + 8h, 8j + 2t + c).
// The A fragment's k index 8j + t + 4c thus stands for column 8j + 2t + c; ssl_rows_normalize writes the transposed copy
// (GEMM2's B operand) in that column order, so no lane exchange is needed.
template <bool CHECK>
__device__ __forceinline__ void exp_tile(const float (&s)[32], uint32_t (&ahi)[32], uint32_t (&alo)[32], float offset,
                                         const float *__restrict__ cs_ptr, int64_t col0, int64_t n_c, float (&rowsum)[2]) {
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int64_t col = col0 + 8 * j + 2 * t;
        float cs0 = 1.f, cs1 = 1.f;
        if (cs_ptr != nullptr) {
            if (!CHECK) {
                const float2 c2 = __ldg(reinterpret_cast<const float2 *>(cs_ptr + col));
                cs0 = c2.x; cs1 = c2.y;
            } else {
                cs0 = col < n_c ? __ldg(cs_ptr + col) : 0.f;
                cs1 = col + 1 < n_c ? __ldg(cs_ptr + col + 1) : 0.f;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float e0 = ssl::ex2(s[4 * j + 2 * h] - offset) * cs0;
            float e1 = ssl::ex2(s[4 * j + 2 * h + 1] - offset) * cs1;
            if (CHECK) {
                e0 = (col < n_c) ? e0 : 0.f;
                e1 = (col + 1 < n_c) ? e1 : 0.f;
            }
            rowsum[h] += e0 + e1;
            float hi, lo;
            ssl::tf32_split(e0, hi, lo);
            ahi[4 * j + h] = __float_as_uint(hi);
            alo[4 * j + h] = __float_as_uint(lo);
            ssl::tf32_split(e1, hi, lo);
            ahi[4 * j + 2 + h] = __float_as_uint(hi);
            alo[4 * j + 2 + h] = __float_as_uint(lo);
        }
    }
}

// LIVE selects a device-side bound (ssl_softmax_gemm_tf32x3_live): 0 none (n_live unused), 1 only the first min(*n_live, n_r)
// rows of R are live, 2 only the first min(*n_live, n_c) rows of C.  n_r stays the row pitch of the outputs.
template <int D, int LIVE>
__global__ void __launch_bounds__(kNumThreads, 1)
softmax_gemm_tc_kernel(const float *__restrict__ R_hi, const float *__restrict__ R_lo,
                       const __grid_constant__ CUtensorMap map_c_hi, const __grid_constant__ CUtensorMap map_c_lo,
                       const __grid_constant__ CUtensorMap map_ct_hi, const __grid_constant__ CUtensorMap map_ct_lo,
                       int64_t n_r, int64_t n_c_cap, const float *__restrict__ colscale, float offset, int n_split,
                       float *__restrict__ rowsum_part, float *__restrict__ o_part, const int64_t *__restrict__ n_live) {
    using K = Cfg<D>;
    // live extents: rows of R past n_r_live are neither read nor written; columns past n_c are masked like a ragged tail
    const int64_t n_r_live = (LIVE == 1) ? ssl::live_count(n_live, n_r) : n_r;
    const int64_t n_c = (LIVE == 2) ? ssl::live_count(n_live, n_c_cap) : n_c_cap;
    constexpr int ST = K::ST, KCH = K::KCH, JCH = K::JCH;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(ring + ST * K::STAGE_BYTES);   // stage s: C hi, C lo (row-major tile), C^T hi, C^T lo
    uint64_t *empty = full + ST;

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const int64_t n_ct = (n_c + BN - 1) / BN;
    const int n_units = (int)((n_r_live + BM - 1) / BM) * n_split;     // unit u: R tile u / n_split, C chunk u % n_split

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c_hi));
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c_lo));
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ct_hi));
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ct_lo));
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
            // ===================== TMA producer: per C tile of every unit its row-major and transposed copies =====================
            // the ring runs on across units, so the next unit's first tiles load under the current unit's last ones
            int it = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
                const int sp = u % n_split;
                const int t0 = (int)(n_ct * sp / n_split), t1 = (int)(n_ct * (sp + 1) / n_split);
                for (int tile = t0; tile < t1; ++tile, ++it) {
                    const int s = it % ST;
                    ssl::mbar_wait(&empty[s], ((it / ST) & 1) ^ 1);
                    uint8_t *c_hi = ring + s * K::STAGE_BYTES, *c_lo = c_hi + K::C_BYTES;
                    uint8_t *ct_hi = c_lo + K::C_BYTES, *ct_lo = ct_hi + K::T_BYTES;
                    ssl::mbar_expect_tx(&full[s], K::STAGE_BYTES);
                    for (int c = 0; c < KCH; ++c) {
                        ssl::tma_load_2d(c_hi + c * K::C_CHUNK, &map_c_hi, c * 32, tile * BN, &full[s]);
                        ssl::tma_load_2d(c_lo + c * K::C_CHUNK, &map_c_lo, c * 32, tile * BN, &full[s]);
                    }
                    for (int c = 0; c < JCH; ++c) {
                        ssl::tma_load_2d(ct_hi + c * K::T_CHUNK, &map_ct_hi, tile * BN + c * 32, 0, &full[s]);
                        ssl::tma_load_2d(ct_lo + c * K::T_CHUNK, &map_ct_lo, tile * BN + c * 32, 0, &full[s]);
                    }
                }
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
    // ===================== consumers: rows [64 * cw, +64) of each unit's R tile =====================
    const int cw = wg - 1, w = (threadIdx.x >> 5) & 3, g = lane >> 2, t = lane & 3;
    // ping-pong: named barrier 1 + cw is this warpgroup's turn to issue MMAs.  Each warpgroup issues a GEMM, passes the turn
    // and only then waits for it, so one warpgroup's exp phase runs under the other's MMAs.  Consumer 0 goes first.
    const int bar_mine = 1 + cw, bar_other = 2 - cw;
    if (cw == 1) ssl::named_arrive(1);
    float o[D / 2], oc[D / 2], sacc[32];
    uint32_t rhi[D / 2], rlo[D / 2], ahi[32], alo[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) {
        sacc[k] = 0.f;
        ahi[k] = alo[k] = 0u;
    }
    int it = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int rt = u / n_split, sp = u % n_split;
        const int t0 = (int)(n_ct * sp / n_split), t1 = (int)(n_ct * (sp + 1) / n_split);
        const int64_t row_a = (int64_t)rt * BM + 64 * cw + 16 * w + g;        // this thread's rows: row_a, row_a + 8
        // GEMM1's A operand, read once per unit straight into the tf32 A fragment (same layout as GEMM2's, see exp_tile):
        // r[4kk + 2c + h] = R(row_a + 8h, 8kk + t + 4c); rows past n_r are 0
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = row_a + 8 * h;
            const bool ok = row < n_r_live;
#pragma unroll
            for (int kk = 0; kk < D / 8; ++kk)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int64_t at = row * D + 8 * kk + t + 4 * c;
                    rhi[4 * kk + 2 * c + h] = ok ? __float_as_uint(__ldg(R_hi + at)) : 0u;
                    rlo[4 * kk + 2 * c + h] = ok ? __float_as_uint(__ldg(R_lo + at)) : 0u;
                }
        }
#pragma unroll
        for (int k = 0; k < D / 2; ++k) o[k] = oc[k] = 0.f;
        float rowsum[2] = {0.f, 0.f};
        for (int tile = t0; tile < t1; ++tile, ++it) {
            const int s = it % ST;
            ssl::mbar_wait(&full[s], (it / ST) & 1);
            const uint32_t c_hi_a = ssl::smem_u32(ring + s * K::STAGE_BYTES), c_lo_a = c_hi_a + K::C_BYTES;
            const uint32_t t_hi_a = c_lo_a + K::C_BYTES, t_lo_a = t_hi_a + K::T_BYTES;
            // ---- GEMM1: S = R C^T, three tf32 products, the small ones first ----
            ssl::named_sync(bar_mine);
            ssl::wg_fence();
#pragma unroll
            for (int part = 0; part < 3; ++part) {
                const uint32_t *ra = (part == 0) ? rlo : rhi;
                const uint32_t cb = (part == 1) ? c_lo_a : c_hi_a;
#pragma unroll
                for (int kk = 0; kk < D / 8; ++kk)
                    wgmma_rs_n64(sacc, ra + 4 * kk, wg_desc(cb + (kk >> 2) * K::C_CHUNK + (kk & 3) * 32), (part > 0 || kk > 0) ? 1u : 0u);
            }
            ssl::wg_commit();
            ssl::named_arrive(bar_other);
            ssl::wg_wait0();
            ssl::reg_fence(sacc);
            ssl::reg_fence(rhi);
            ssl::reg_fence(rlo);
            // ---- E = exp2(S - offset) * colscale, row sums, GEMM2's A fragment ----
            const int64_t col0 = (int64_t)tile * BN;
            if (col0 + BN <= n_c) exp_tile<false>(sacc, ahi, alo, offset, colscale, col0, n_c, rowsum);
            else exp_tile<true>(sacc, ahi, alo, offset, colscale, col0, n_c, rowsum);
            // ---- GEMM2: O += E C (hi*hi into O, the two correction products into OC) ----
            ssl::named_sync(bar_mine);
            ssl::wg_fence();
#pragma unroll
            for (int part = 0; part < 3; ++part) {
                const uint32_t *ea = (part == 0) ? alo : ahi;
                const uint32_t tb = (part == 1) ? t_lo_a : t_hi_a;
#pragma unroll
                for (int kk = 0; kk < BN / 8; ++kk) {
                    const uint64_t bd = wg_desc(tb + (kk >> 2) * K::T_CHUNK + (kk & 3) * 32);
                    if (part == 2) wgmma_rs<D>(o, ea + 4 * kk, bd);
                    else wgmma_rs<D>(oc, ea + 4 * kk, bd);
                }
            }
            ssl::wg_commit();
            ssl::named_arrive(bar_other);
            // waiting here rather than under the next GEMM1 keeps ptxas from serialising the wgmmas
            ssl::wg_wait0();
            ssl::reg_fence(ahi);
            ssl::reg_fence(alo);
            ssl::reg_fence(o);
            ssl::reg_fence(oc);
            ssl::mbar_arrive(&empty[s]);                               // both copies of the tile are consumed
        }

        // ---- unit epilogue: o[4j + 2h + c] = O(row 16w + g + 8h, col 8j + 2t + c) ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            rowsum[h] += __shfl_xor_sync(0xffffffffu, rowsum[h], 1);
            rowsum[h] += __shfl_xor_sync(0xffffffffu, rowsum[h], 2);
            const int64_t grow = row_a + 8 * h;
            if (grow >= n_r_live) continue;
            float *dst = o_part + ((size_t)sp * n_r + grow) * D;
#pragma unroll
            for (int j = 0; j < D / 8; ++j)
                *reinterpret_cast<float2 *>(dst + 8 * j + 2 * t) =
                    make_float2(o[4 * j + 2 * h] + oc[4 * j + 2 * h], o[4 * j + 2 * h + 1] + oc[4 * j + 2 * h + 1]);
            if (t == 0 && rowsum_part != nullptr) rowsum_part[(size_t)sp * n_r + grow] = rowsum[h];
        }
    }
    if (cw == 0) ssl::named_sync(1);                                  // consumer 1's last hand-over
}

template <int D, int LIVE>
int launch_tc(const float *R_hi, const float *R_lo, int64_t n_r, const float *C_hi, const float *C_lo, const float *CT_hi,
              const float *CT_lo, int64_t ct_pitch, int64_t n_c, const float *colscale, float offset, int n_split,
              float *rowsum_part, float *o_part, const int64_t *n_live, cudaStream_t st) {
    // fp32 boxes of 32 floats (128 B, SWIZZLE_128B) x 64 rows of C, x D rows of C^T [D, ct_pitch]
    constexpr CUtensorMapDataType F32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    constexpr CUtensorMapSwizzle SW = CU_TENSOR_MAP_SWIZZLE_128B;
    CUtensorMap mc_hi, mc_lo, mt_hi, mt_lo;
    int rc;
    if ((rc = ssl::make_map_2d(&mc_hi, F32, C_hi, n_c, D, D * 4, 32, BN, SW)) != SSL_OK) return rc;
    if ((rc = ssl::make_map_2d(&mc_lo, F32, C_lo, n_c, D, D * 4, 32, BN, SW)) != SSL_OK) return rc;
    // the transposed copy's columns are permuted within groups of 8 (see exp_tile): its last group is read whole
    const int64_t n_c8 = (n_c + 7) / 8 * 8;
    if ((rc = ssl::make_map_2d(&mt_hi, F32, CT_hi, D, n_c8, ct_pitch * 4, 32, D, SW)) != SSL_OK) return rc;
    if ((rc = ssl::make_map_2d(&mt_lo, F32, CT_lo, D, n_c8, ct_pitch * 4, 32, D, SW)) != SSL_OK) return rc;
    const size_t smem = Cfg<D>::SMEM;
    int n_sm = 0;
    if ((rc = ssl::configure_once<softmax_gemm_tc_kernel<D, LIVE>>(smem, &n_sm)) != SSL_OK) return rc;
    // units (R tile, C chunk), sized for the capacity when the live count is on the device (the units past it are skipped,
    // the live ones stay spread round-robin)
    const int64_t grid = ssl::persistent_grid(((n_r + BM - 1) / BM) * n_split, n_sm);
    softmax_gemm_tc_kernel<D, LIVE><<<(unsigned)grid, kNumThreads, smem, st>>>(R_hi, R_lo, mc_hi, mc_lo, mt_hi, mt_lo, n_r, n_c, colscale,
                                                                               offset, n_split, rowsum_part, o_part, n_live);
    SSL_LAUNCH_CHECK("softmax_gemm_tc_kernel");
    return SSL_OK;
}

}  // namespace

namespace {
int check_tc_args(const float *R_hi, const float *R_lo, const float *C_hi, const float *C_lo, const float *CT_hi, const float *CT_lo,
                  int64_t ct_pitch, int64_t n_c, int32_t dim, const float *colscale, int32_t n_split, const float *o_part,
                  const char *name) {
    SSL_CHECK_ARG(R_hi && R_lo && C_hi && C_lo && CT_hi && CT_lo && o_part, "%s: null argument", name);
    SSL_CHECK_ARG(ct_pitch >= (n_c + 7) / 8 * 8 && ct_pitch % 4 == 0, "%s: ct_pitch must be >= ceil8(n_c) and a multiple of 4", name);
    SSL_CHECK_ARG(dim == 32 || dim == 64, "%s: dim %d not supported (32 or 64; other sizes use ssl_softmax_gemm)", name, dim);
    SSL_CHECK_ARG((n_split >= 1 && n_split <= (n_c + BN - 1) / BN) || n_c == 0, "%s: n_split %d exceeds the number of C tiles", name, n_split);
    SSL_CHECK_ARG(((reinterpret_cast<uintptr_t>(R_hi) | reinterpret_cast<uintptr_t>(R_lo) | reinterpret_cast<uintptr_t>(C_hi) |
                    reinterpret_cast<uintptr_t>(C_lo) | reinterpret_cast<uintptr_t>(CT_hi) | reinterpret_cast<uintptr_t>(CT_lo) |
                    reinterpret_cast<uintptr_t>(o_part)) & 15) == 0,
                  "%s: operands must be 16-byte aligned", name);
    SSL_CHECK_ARG((reinterpret_cast<uintptr_t>(colscale) & 7) == 0, "%s: colscale must be 8-byte aligned", name);
    return SSL_OK;
}
}  // namespace

extern "C" int ssl_softmax_gemm_tf32x3(const float *R_hi, const float *R_lo, int64_t n_r, const float *C_hi, const float *C_lo,
                                       const float *CT_hi, const float *CT_lo, int64_t ct_pitch, int64_t n_c, int32_t dim,
                                       const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                                       void *stream) {
    const int rc = check_tc_args(R_hi, R_lo, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, dim, colscale, n_split, o_part, "ssl_softmax_gemm_tf32x3");
    if (rc != SSL_OK) return rc;
    if (n_r == 0 || n_c == 0) return SSL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dim == 32) return launch_tc<32, 0>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, nullptr, st);
    return launch_tc<64, 0>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, nullptr, st);
}

extern "C" int ssl_softmax_gemm_tf32x3_live(const float *R_hi, const float *R_lo, int64_t n_r, const float *C_hi, const float *C_lo,
                                            const float *CT_hi, const float *CT_lo, int64_t ct_pitch, int64_t n_c, int32_t dim,
                                            const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                                            const int64_t *n_live, int32_t live_role, void *stream) {
    const int rc = check_tc_args(R_hi, R_lo, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, dim, colscale, n_split, o_part, "ssl_softmax_gemm_tf32x3_live");
    if (rc != SSL_OK) return rc;
    SSL_CHECK_ARG(n_live != nullptr, "ssl_softmax_gemm_tf32x3_live: null n_live");
    SSL_CHECK_ARG(live_role == SSL_LIVE_ROWS || live_role == SSL_LIVE_COLS, "ssl_softmax_gemm_tf32x3_live: bad live_role %d", live_role);
    if (n_r == 0 || n_c == 0) return SSL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (live_role == SSL_LIVE_ROWS) {
        if (dim == 32) return launch_tc<32, 1>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
        return launch_tc<64, 1>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
    }
    if (dim == 32) return launch_tc<32, 2>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
    return launch_tc<64, 2>(R_hi, R_lo, n_r, C_hi, C_lo, CT_hi, CT_lo, ct_pitch, n_c, colscale, offset, n_split, rowsum_part, o_part, n_live, st);
}
