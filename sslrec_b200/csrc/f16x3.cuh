// 3xFP16 operand split for the tensor-core InfoNCE contraction (ssl_softmax_gemm_f16x3) and its operand writer
// (ssl_rows_normalize_f16x3):
//
//   hi = fp16(x)                    (0 when |x| < 2^-14, the smallest normal fp16)
//   lo = fp16((x - hi) * 2^k),  k = kF16LoShift = 12          x = hi + 2^-k lo + O(2^-22 |x|)
//
// FP16 has the 11-bit significand of TF32, so the three products hi*hi + 2^-k (lo*hi + hi*lo) recover fp32-grade
// accuracy as 3xTF32 does, provided the residual x - hi, up to 2^-11 |x|, is lifted into fp16's narrow exponent range
// (Ootomo & Yokota, IJHPCA 2022).  The bounds, for the operands and offsets the C ABI accepts:
//
// * Operands R, C: rows normalised to norm <= 1 and scaled by |alpha| <= 16 (kF16MaxAlpha), so |x| <= 16: hi is finite,
//   and |x - hi| <= 2^-8 (half an fp16 ulp in [8, 16)), so |lo| <= 2^4.
// * E = exp2(S - offset) * colscale[c] * 2^b / M with b = kF16Bias = 14, M a power of two >= max |colscale| and
//   S <= offset (|R_r| |C_c| <= offset), so |E| <= 2^14 (1 + a few ulp) < 2^15.  Half an fp16 ulp below 2^15 is 2^3, and
//   lo = (E - hi) 2^k must stay below 65504: 2^(3 + k) < 65504 gives k <= 12.  One k has to serve both factors of each
//   correction product (lo_R * hi_C and hi_R * lo_C share an accumulator, as do lo_E * hi_C and hi_E * lo_C), so k = 12
//   for R, C and E alike.  (R alone would allow k <= 22.)
// * Without colscale (the forward role, M = 1) the kernel folds the bias into the offset: E = exp2(S - (offset - 14)).
//   offset - 14 is rounded once per launch, exactly for offset in [7, 16] (Sterbenz) and by at most 2^-21 below, and the
//   subtraction once per element; S <= offset still bounds the argument by 14 + those roundings, so E <= 2^14 (1 + a
//   few ulp) as above.  Only the argument's rounding moves (at |S - offset + 14| instead of |S - offset|, both <= 32).
// * The lower end: S - offset >= -2 offset >= -32, so E >= 2^-18 * colscale[c] / M.  Values below 2^-14 have hi = 0 and
//   lo = fp16(x 2^12) carries them whole: a normal fp16 down to |x| = 2^-26 (2^-11 relative, so < 2^-25 absolute), an
//   fp16 subnormal below that (at most 2^-25 * 2^-12 = 2^-37 absolute).
// * Without colscale, E >= 2^(14 - 2 offset) >= 2^-13 for offset <= kF16NoFlushOffset = 13.5 (half a binade above the
//   flush threshold covers the roundings of S and of the argument).  There the flush rule can never fire, and the forward
//   splits with f16x3_split2<false>, which leaves it out.  Above 13.5 (tau < 0.107) the forward keeps it.
// * Reconstruction: |x - hi - 2^-k lo| <= 2^-11 |x - hi| <= 2^-22 |x| for |x| >= 2^-14 -- the grade of the 3xTF32 split
//   (tf32_split in common.cuh) -- and < 2^-25 absolute below.  Against the scales involved that is below fp32 rounding:
//   an operand entry < 2^-14 moves S = R . C by < 2^-25 |C_c| (S itself is rounded at 2^-24 |S|), and an E' < 2^-14 moves O'
//   by < 2^-25 |C_c| where E' reaches 2^14.
// * hi is never an fp16 subnormal (the flush rule), so whether the tensor core flushes subnormal inputs does not decide
//   the hi products; the only subnormals are lo parts of |x| < 2^-26, so a flush of them moves x by < 2^-26.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace ssl {

constexpr int kF16LoShift = 12;
constexpr float kF16LoScale = 4096.f;                 // 2^kF16LoShift
constexpr float kF16LoUnscale = 1.f / 4096.f;         // 2^-kF16LoShift
constexpr float kF16MinNormal = 6.103515625e-05f;     // 2^-14
constexpr int kF16Bias = 14;                          // E's exponent bias b
constexpr float kF16MaxAlpha = 16.f;                  // bound on |alpha| of the operand writer (operand entries <= 16)
constexpr float kF16MaxOffset = 16.f;                 // bound on the contraction's offset (covers tau >= 0.0902)
constexpr float kF16NoFlushOffset = 13.5f;            // without colscale, E' >= 2^(14 - 2 offset) >= 2^-13 up to here

__device__ __forceinline__ float f16x3_hi_input(float x) { return fabsf(x) < kF16MinNormal ? 0.f : x; }

// two values -> packed f16x2 hi / lo parts, x0 in the low half (the lower k index of a wgmma A fragment register).
// FLUSH = false leaves the flush rule out, for values known to be 0 or of magnitude >= 2^-14 (hi is then never an fp16
// subnormal either way): the forward's E' at offsets <= kF16NoFlushOffset.
template <bool FLUSH = true>
__device__ __forceinline__ void f16x3_split2(float x0, float x1, uint32_t &hi, uint32_t &lo) {
    const __half2 h = FLUSH ? __floats2half2_rn(f16x3_hi_input(x0), f16x3_hi_input(x1)) : __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn((x0 - hf.x) * kF16LoScale, (x1 - hf.y) * kF16LoScale);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}

__device__ __forceinline__ void f16x3_split1(float x, __half &hi, __half &lo) {
    hi = __float2half_rn(f16x3_hi_input(x));
    lo = __float2half_rn((x - __half2float(hi)) * kF16LoScale);
}

}  // namespace ssl
