"""The exp phase of the 3xFP16 InfoNCE contraction (exp_tile in csrc/nce_gemm_f16x3.cu), restated in float32 numpy for
each role the launch picks:

  forward  (no colscale)  E' = ex2(x - (offset - 14))                      flush rule only above offset 13.5
  backward (colscale)     E' = ex2(x - offset) * (colscale * 2^14 / M)     flush rule always

then split into hi = fp16(E') (0 below 2^-14 where the flush rule applies) and lo = fp16((E' - hi) 2^12).  The tensor
core is modelled at its least favourable: it flushes fp16 subnormal inputs to zero.  Every E' must be reconstructed
within 2^-18 relative (the argument's fp32 rounding, ex2's and the split's) plus 2^-25 absolute, and the row sums and
O = E' C within the bounds test_gpu_nce_f16x3.py holds the kernel to against float64.  The restatement with the 2^14
dropped from the fold, or without the flush rule in the backward, fails those bounds."""
import numpy as np
import pytest

from test_host_f16x3_split import K, MIN_NORMAL

BIAS = 14                    # kF16Bias
NO_FLUSH_OFFSET = 13.5       # kF16NoFlushOffset
F32 = np.float32


def _ex2(y):
    """ex2.approx.ftz.f32, modelled as the correctly rounded exp2."""
    return np.exp2(y.astype(np.float64)).astype(F32)


def exp_phase(x, off, cs=None, fold_bias=BIAS, flush=None):
    """fp32 S values x [rows, cols] -> (E', hi, lo, back) as the kernel computes them; back = M 2^-14 undoes the scaling
    of E'.  ``flush`` None picks the kernel's rule; ``fold_bias`` is the exponent the forward folds into its offset."""
    x = np.asarray(x, dtype=F32)
    if cs is None:
        e = _ex2(x - (F32(off) - F32(fold_bias)))
        e_m = 0
        flush = off > NO_FLUSH_OFFSET if flush is None else flush
    else:
        _, e_m = np.frexp(np.abs(cs).max())
        e_m = int(np.clip(e_m, -100, 100))
        cs0 = (cs.astype(F32) * F32(2.0 ** (BIAS - e_m))).astype(F32)      # exact: a power of two
        e = (_ex2(x - F32(off)) * cs0[None, :]).astype(F32)
        flush = True if flush is None else flush
    hi_in = np.where(np.abs(e) < MIN_NORMAL, F32(0), e) if flush else e
    hi = hi_in.astype(np.float16)
    lo = ((e - hi.astype(F32)) * F32(2.0 ** K)).astype(np.float16)
    return e, hi, lo, 2.0 ** (e_m - BIAS)


def _tensor_core(h):
    """fp16 inputs as a tensor core that flushes subnormals sees them."""
    h = h.astype(np.float64)
    return np.where(np.abs(h) < 2.0 ** -14, 0.0, h)


def _case(off, backward, n_r=256, n_c=512, d=64, seed=0):
    """S = R C^T of rows scaled to the contraction's bound (|S| <= off, or S <= 0 at off = 0) with the extremes S = +-off
    included, and the backward's colscale (magnitude 1e-9, max / min ratio 2^12)."""
    rng = np.random.default_rng(seed)
    r, c = rng.standard_normal((n_r, d)), rng.standard_normal((n_c, d))
    if off == 0.0:
        r, c, alpha = -np.abs(r), np.abs(c), 1.0
    else:
        alpha = off
    r = (alpha * r / np.linalg.norm(r, axis=1, keepdims=True)).astype(F32)
    c = (c / np.linalg.norm(c, axis=1, keepdims=True)).astype(F32)
    if off > 0.0:
        r[0], r[1] = alpha * c[0], -alpha * c[0]                           # S = +off and S = -off at column 0
    x = (r.astype(np.float64) @ c.T.astype(np.float64)).astype(F32)
    cs = (1e-9 * np.exp2(-12.0 * rng.random(n_c))).astype(F32) if backward else None
    return x, c, cs


def _errors(off, backward, **kw):
    """Largest violation ratios of the per-element bound and of the row-sum and O bounds (<= 1 passes)."""
    x, c, cs = _case(off, backward)
    e, hi, lo, back = exp_phase(x, off, cs, **kw)
    rec = (_tensor_core(hi) + _tensor_core(lo) * 2.0 ** -K) * back
    ref = np.exp2(x.astype(np.float64) - off) * (1.0 if cs is None else cs.astype(np.float64)[None, :])
    elem = np.abs(rec - ref) / (2.0 ** -18 * np.abs(ref) + 2.0 ** -25 * back)
    rs, rs_ref = e.astype(np.float64).sum(1) * back, ref.sum(1)
    o, o_ref = rec @ c.astype(np.float64), ref @ c.astype(np.float64)
    rs_err = np.abs(rs - rs_ref) / (2e-4 * np.abs(rs_ref) + 1e-5 * np.abs(rs_ref).max())
    o_err = np.abs(o - o_ref) / (2e-4 * np.abs(o_ref) + 1e-5 * np.abs(o_ref).max())
    return elem.max(), rs_err.max(), o_err.max(), (np.abs(e) < MIN_NORMAL).sum()


@pytest.mark.parametrize('backward', [False, True])
@pytest.mark.parametrize('off', [0.0, 7.2, 13.5, 16.0])
def test_exp_phase_meets_the_bounds(off, backward):
    elem, rs, o, _ = _errors(off, backward)
    assert elem <= 1.0 and rs <= 1.0 and o <= 1.0, (elem, rs, o)


@pytest.mark.parametrize('off', [0.0, 7.2, 13.5])
def test_forward_without_flush_stays_normal(off):
    """Up to offset 13.5 the forward's E' >= 2^(14 - 2 offset) >= 2^-13: the flush rule could never fire."""
    x, _, _ = _case(off, False)
    e, hi, _, _ = exp_phase(x, off)
    assert e.min() >= 2.0 ** -13
    assert (np.abs(hi.astype(F32)) >= MIN_NORMAL).all()


def test_fold_without_the_bias_fails():
    """Folding only the offset (E' = ex2(x - offset)) leaves O' 2^14 times too small after the back-scaling."""
    elem, rs, o, _ = _errors(7.2, False, fold_bias=0)
    assert elem > 1.0 and o > 1.0


def test_backward_without_flush_fails():
    """Without the flush rule the backward's E' below 2^-14 give subnormal hi parts, which a flushing tensor core drops."""
    elem, _, _, n_small = _errors(16.0, True, flush=False)
    assert n_small > 0 and elem > 1.0


def test_forward_above_the_no_flush_offset_needs_the_flush():
    """At offset 16, E' reaches down to 2^-18: the forward there keeps the flush rule (the kernel picks it above 13.5)."""
    elem, _, _, n_small = _errors(16.0, False, flush=False)
    assert n_small > 0 and elem > 1.0
