"""The 3xFP16 operand split of the tensor-core InfoNCE contraction (csrc/f16x3.cuh), restated in numpy:

    hi = fp16(x)  (0 when |x| < 2^-14),   lo = fp16((x - hi) 2^12)

checked over every fp32 exponent the kernel can meet (operands |x| <= 16, E' <= 2^14 and its rounding, down to fp32
subnormals): the reconstruction bound (2^-22 relative from 2^-14 on, 2^-25 absolute below), no overflow at the bound,
and the flush rule.  test_gpu_nce_f16x3.py checks the
device split against ``f16x3_split`` bit for bit."""
import numpy as np

K = 12                                   # kF16LoShift
MIN_NORMAL = np.float32(2.0 ** -14)


def f16x3_split(x, k=K):
    """fp32 array -> (hi, lo) float16 arrays, with numpy's round-to-nearest-even conversions (those of __float2half_rn)."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over='ignore'):
        hi = np.where(np.abs(x) < MIN_NORMAL, np.float32(0), x).astype(np.float16)
        lo = ((x - hi.astype(np.float32)) * np.float32(2.0 ** k)).astype(np.float16)   # x - hi and the scaling are exact in fp32
    return hi, lo


def _values(e_lo, e_hi, per_exp=4096, seed=0):
    """Per binade [2^e, 2^(e+1)) for e in [e_lo, e_hi]: its ends, mantissas next to fp16 rounding ties, and random
    mantissas; both signs."""
    rng = np.random.default_rng(seed)
    out = []
    for e in range(e_lo, e_hi + 1):
        m = np.concatenate([rng.integers(0, 1 << 23, per_exp), [0, (1 << 23) - 1, 1 << 12, (1 << 12) - 1, (1 << 12) + 1, 3 << 12]])
        if e < -126:                     # fp32 subnormals: the mantissa is the whole value
            bits = (m >> (-126 - e)).astype(np.uint32)
        else:
            bits = ((e + 127) << 23 | m).astype(np.uint32)
        v = bits.view(np.float32)
        out += [v, -v]
    return np.concatenate(out)


def _check(x):
    hi, lo = f16x3_split(x)
    assert np.isfinite(hi).all() and np.isfinite(lo).all(), 'overflow'
    x64 = x.astype(np.float64)
    rec = hi.astype(np.float64) + lo.astype(np.float64) * 2.0 ** -K
    err = np.abs(x64 - rec)
    # from 2^-14 on: 2^-22 relative (the 3xTF32 grade); below, lo alone carries x: 2^-11 relative (< 2^-25 absolute)
    # while lo is a normal fp16, 2^-37 absolute once it is subnormal
    ax = np.abs(x64)
    bound = np.where(ax >= 2.0 ** -14, 2.0 ** -22 * ax, np.where(ax >= 2.0 ** -26, 2.0 ** -11 * ax, 2.0 ** -37))
    assert (err <= bound).all(), f'reconstruction: max err / bound {(err / bound).max():.3f} at x = {x[np.argmax(err / bound)]!r}'
    h = np.abs(hi.astype(np.float32))
    assert ((h == 0) | (h >= MIN_NORMAL)).all(), 'hi must never be an fp16 subnormal'
    assert (hi[np.abs(x) < MIN_NORMAL] == 0).all(), 'entries below 2^-14 must go to lo whole'
    return err, bound


def test_split_operands_every_exponent():
    """Normalised rows scaled by |alpha| <= 16: every binade from fp32 subnormals to 16 itself."""
    x = np.concatenate([_values(-149, 3), np.float32([16.0, -16.0, 0.0, -0.0])])
    _check(x)


def test_split_exp_values_every_exponent():
    """E' = exp2(S - offset) colscale 2^14 / M <= 2^14 (1 + a few ulp): every binade up to [2^14, 2^15)."""
    _check(_values(-149, 14, seed=1))


def test_flush_rule_puts_small_entries_in_lo_whole():
    x = np.float32([2.0 ** -14, np.nextafter(np.float32(2.0 ** -14), np.float32(0)), 2.0 ** -20, 2.0 ** -26, 1e-30, 0.0])
    hi, lo = f16x3_split(x)
    assert hi[0] == np.float16(2.0 ** -14) and lo[0] == 0
    assert (hi[1:] == 0).all()
    np.testing.assert_array_equal(lo[2:4].astype(np.float64), x[2:4].astype(np.float64) * 2.0 ** K)   # normal fp16, exact
    # without the rule, hi would be an fp16 subnormal for these
    assert (np.abs(x[2:4].astype(np.float16).astype(np.float32)) < MIN_NORMAL).all()


def test_shift_12_is_the_largest_without_overflow():
    """k = 12 keeps lo finite for every value below 2^15; k = 13 overflows there (half an fp16 ulp at 2^14 is 2^3)."""
    x = _values(14, 14, seed=2)
    assert np.isfinite(f16x3_split(x, 12)[1]).all()
    assert not np.isfinite(f16x3_split(x, 13)[1]).all()
