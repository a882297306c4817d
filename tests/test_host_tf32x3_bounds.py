"""The error bound of the 3xTF32 InfoNCE contraction (csrc/nce_gemm_tc.cu), derived from the kernel's arithmetic, and a
numpy restatement of that arithmetic in float32 / tf32 that meets it while slightly wrong restatements miss it.
test_gpu_nce_tf32x3.py checks the device against the same bound (``bound_coefs``).

One unit computes, for row i of R and the columns j of one C chunk (log2 units: R carries log2(e) / temp),

    S_ij = R_lo.C_hi + R_hi.C_lo + R_hi.C_hi    E_ij = ex2(S_ij - off) cs_j    rowsum_i = sum_j E_ij    O_i = sum_j E_ij C_j

Let u = 2^-23 (one fp32 ulp relative), P_ij = sum_k |a_ik c_jk| and Pw_ij = sum_k w_k |a_ik c_jk| with w_k = d/8 - floor(k/8).

GEMM1, the split.  x = hi + lo + r with hi = rna_tf32(x), lo = rna_tf32(x - hi).  For x in [2^e, 2^(e+1)): |x - hi| <= 2^(e-11),
x - hi is exact and lies on the fp32 grid 2^(e-23), so rounding it to 11 bits leaves |r| <= 2^(e-23) <= u|x|; |lo| <= 2^-11 |x|.
The dropped lo.lo product is <= 2^-22 |a||c| = 2u |a||c|.  a c - (lo_a hi_c + hi_a lo_c + hi_a hi_c) = lo_a lo_c + r_a c + (hi_a + lo_a) r_c,
so the split costs <= (2 + 1 + 1 + 2^-11) u P_ij.  Every tf32 x tf32 product is exact in fp32 (11 x 11 bits).

GEMM1, the accumulator.  The tensor core's fp32 accumulator truncates.  Model: one m64nNk8 step forms acc + its 8 products and
truncates the result once, an error < ulp(result) <= u |result|.  The two correction parts run first (2 d/8 steps, |acc| <=
2^-10 (1 + 2^-10) P), then the d/8 steps of hi.hi, where after step s |acc| <= 2^-10 P + sum_{k < 8s} |a_k c_k| (1 + 2^-10):
summed, <= u ((1 + 2^-10) Pw + (3d/8) 2^-9 P).  So |S~ - S| <= u (c_P P + c_w Pw) with c_P = 4 + 2^-11 + (3d/8) 2^-9, c_w = 1 + 2^-10
(Pw <= (d/8) P gives the plain form c1 = c_P + d/8).

E.  S~ - off rounds to nearest: u/2 |S - off|.  An error x in the exponent is a relative error ln2 |x| of E.  ex2.approx.ftz: 2 ulp,
<= 2u relative; the colscale product rounds to nearest: u/2.  Results below 2^-126 flush to 0: an absolute 2^-126 per column.
    eps_E(i) = ln2 u max_j (c_P P_ij + c_w Pw_ij + |S_ij - off| / 2) + 2u + [u/2 with colscale]

rowsum.  Each thread sums its 2 columns per 8-column group, then adds the pair to its running fp32 sum (both rounded to nearest),
over the chunk's columns; two shuffles add the 4 threads' sums.  A term passes through <= cols/8 + 3 roundings:
    |rowsum~_i - rowsum_i| <= (1 + 2^-8) (eps_E(i) + (cols/8 + 3) u/2) rowsum_i + cols 2^-126

O.  E and C^T are split again (4u of W_ik = sum_j E_ij |c_jk|); hi.hi has its own truncating accumulator, cols/8 steps of <= u W;
the two correction parts share one, 2 cols/8 steps of <= 2^-10 u W; o + oc rounds to nearest:
    |O~_ik - O_ik| <= (1 + 2^-8) (eps_E(i) + 4u + (cols/8)(1 + 2^-9) u + u/2) W_ik + cols 2^-126 max_j |c_jk|

cols is the longest C chunk of the split, ceil(ceil(n_c / 64) / n_split) * 64.  The factor 1 + 2^-8 covers the second-order
terms.  For the sum over the split's partials (done in float64 by the tests) the per-chunk bounds add up to these."""
import math

import numpy as np
import pytest

U = 2.0 ** -23
LN2 = math.log(2.0)
FLUSH = 2.0 ** -126
LOG2E = 1.4426950408889634


def bound_coefs(d, cols, colscale):
    """(c_P, c_w, base_rs, base_o, slack): eps_E = ln2 u max_j(c_P P + c_w Pw + |S - off| / 2) + 2u [+ u/2];
    rowsum bound = slack (eps_E + base_rs) rowsum + cols 2^-126; O bound = slack (eps_E + base_o) W + cols 2^-126 max|c|,
    where the base terms already hold the exponent-independent parts of eps_E."""
    c_p = 4 + 2.0 ** -11 + (3 * d / 8) * 2.0 ** -9
    c_w = 1 + 2.0 ** -10
    e0 = 2 * U + (U / 2 if colscale else 0.0)
    base_rs = e0 + (cols / 8 + 3) * U / 2
    base_o = e0 + 4 * U + (cols / 8) * (1 + 2.0 ** -9) * U + U / 2
    return c_p, c_w, base_rs, base_o, 1 + 2.0 ** -8


def chunk_cols(n_c, n_split):
    n_ct = -(-n_c // 64)
    return -(-n_ct // n_split) * 64


def step_weights(d):
    """w_k = number of hi.hi accumulator steps at or after the one that adds column k of the operands."""
    return (d // 8 - np.arange(d) // 8).astype(np.float64)


def reference(A, T, cs, off, n_split):
    """float64: rowsum, O and their bounds for rows A [n_r, d] against T [n_c, d] (fp32 values, as the kernel reads them)."""
    A, T = A.astype(np.float64), T.astype(np.float64)
    d = A.shape[1]
    S = A @ T.T
    E = np.exp2(S - off) * (1.0 if cs is None else cs.astype(np.float64))
    P = np.abs(A) @ np.abs(T).T
    Pw = (np.abs(A) * step_weights(d)) @ np.abs(T).T
    c_p, c_w, base_rs, base_o, slack = bound_coefs(d, chunk_cols(T.shape[0], n_split), cs is not None)
    g1 = (c_p * P + c_w * Pw + 0.5 * np.abs(S - off)).max(1) if T.shape[0] else np.zeros(A.shape[0])
    eps = LN2 * U * g1
    rs, O, W = E.sum(1), E @ T, E @ np.abs(T)
    cols = T.shape[0]
    b_rs = slack * (eps + base_rs) * rs + cols * FLUSH
    b_o = slack * (eps + base_o)[:, None] * W + cols * FLUSH * (np.abs(T).max() if cols else 0.0)
    return rs, O, b_rs, b_o


# ---- the kernel's arithmetic in numpy --------------------------------------------------------------------------------------

def tf32(x, rz=False):
    """cvt.rna.tf32.f32 (round to nearest, ties away) or, ``rz``, cvt.rz: keep 10 explicit mantissa bits."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    if not rz:
        b = b + np.uint32(0x1000)
    return (b & np.uint32(0xFFFFE000)).view(np.float32)


def split(x, rz=False):
    hi = tf32(x, rz)
    return hi, tf32(np.float32(x) - hi, rz)


def trunc32(x):
    """float64 -> float32 rounded toward zero."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def emulate(A, T, cs, off, n_split, drop_r_lo=False, rz=False, drop_e_lo=False, no_mask=False):
    """The kernel's value path for fp32 R = A [n_r, d], C = T [n_c, d] (zero rows up to ceil64(n_c), as the writer pads them),
    colscale ``cs`` (None, or ceil64(n_c) entries): per split partials (rowsum [n_split, n_r], O [n_split, n_r, d])."""
    n_r, d = A.shape
    n_c = T.shape[0]
    n_ct = -(-n_c // 64)
    Tp = np.zeros((n_ct * 64, d), np.float32)
    Tp[:n_c] = T
    ahi, alo = split(A, rz)
    chi, clo = split(Tp, rz)
    off32 = np.float32(off)
    rs_part = np.zeros((n_split, n_r), np.float32)
    o_part = np.zeros((n_split, n_r, d), np.float32)
    for sp in range(n_split):
        t0, t1 = n_ct * sp // n_split, n_ct * (sp + 1) // n_split
        rs_thr = np.zeros((n_r, 4), np.float32)                  # the 4 threads of a row
        o, oc = np.zeros((n_r, d), np.float32), np.zeros((n_r, d), np.float32)
        for tile in range(t0, t1):
            cols = slice(tile * 64, tile * 64 + 64)
            acc = np.zeros((n_r, 64), np.float32)
            parts = ([] if drop_r_lo else [(alo, chi)]) + [(ahi, clo), (ahi, chi)]       # the small products first
            for ra, cb in parts:
                for kk in range(d // 8):
                    k = slice(8 * kk, 8 * kk + 8)
                    acc = trunc32(acc.astype(np.float64) + ra[:, k].astype(np.float64) @ cb[cols, k].astype(np.float64).T)
            x = (acc - off32).astype(np.float32)
            with np.errstate(over='ignore', under='ignore'):
                e = np.exp2(x.astype(np.float64)).astype(np.float32)
            e[np.abs(e) < FLUSH] = 0                                # ex2.approx.ftz
            col = tile * 64 + np.arange(64)
            if cs is not None:
                c = cs[cols].astype(np.float32)
                if tile * 64 + 64 > n_c:
                    c = np.where(col < n_c, c, np.float32(0))
                e = (e * c).astype(np.float32)
            if tile * 64 + 64 > n_c and not no_mask:
                e = np.where(col < n_c, e, np.float32(0)).astype(np.float32)
            for j in range(8):                                    # thread t: columns 8j + 2t, 8j + 2t + 1
                pair = e[:, 8 * j + 0:8 * j + 8:2] + e[:, 8 * j + 1:8 * j + 8:2]
                rs_thr = (rs_thr + pair).astype(np.float32)
            ehi, elo = split(e, rz)
            thi, tlo = chi[cols], clo[cols]
            gemm2 = [(ehi, tlo)] if drop_e_lo else [(elo, thi), (ehi, tlo)]
            for ea, tb in gemm2:
                for kk in range(8):
                    k = slice(8 * kk, 8 * kk + 8)
                    oc = trunc32(oc.astype(np.float64) + ea[:, k].astype(np.float64) @ tb[k].astype(np.float64))
            for kk in range(8):
                k = slice(8 * kk, 8 * kk + 8)
                o = trunc32(o.astype(np.float64) + ehi[:, k].astype(np.float64) @ thi[k].astype(np.float64))
        s01 = (rs_thr[:, 0] + rs_thr[:, 1]).astype(np.float32)     # xor 1, then xor 2
        s23 = (rs_thr[:, 2] + rs_thr[:, 3]).astype(np.float32)
        rs_part[sp] = (s01 + s23).astype(np.float32)
        o_part[sp] = (o + oc).astype(np.float32)
    return rs_part, o_part


# ---- operands of the GPU file's cases, at reduced sizes ---------------------------------------------------------------------

def _unit(rng, n, d, alpha):
    x = rng.standard_normal((n, d))
    return (x / np.linalg.norm(x, axis=1, keepdims=True) * alpha).astype(np.float32)


def raw_rows(rng, n_a, n_t, d, temp, max_logit):
    """LightGCL's raw operands: anchors a log2(e) / temp and table rows t, scaled so that max |a . t| / temp = max_logit."""
    a, t = rng.standard_normal((n_a, d)), rng.standard_normal((n_t, d))
    t *= max_logit * temp / np.abs(a @ t.T).max()
    return (a.astype(np.float32) * np.float32(LOG2E / temp)).astype(np.float32), t.astype(np.float32)


def cancelling_rows(rng, n_a, d, p):
    """Raw rows where sum_k |a_k t_k| = p (log2 units) while S = a . t nearly cancels: one table row t, half of it the first
    anchor and half its negative, and anchors that are small perturbations of the first (|S| up to ~ p / 20)."""
    h = rng.standard_normal(d // 2)
    a0 = np.concatenate([h, h]) * math.sqrt(p / (2 * (h * h).sum()))
    a = a0 + rng.standard_normal((n_a, d)) * 0.05 * math.sqrt(p / d)
    a[0] = a0
    t = np.concatenate([a0[:d // 2] * (1 + 1e-4), -a0[d // 2:]])[None]
    return a.astype(np.float32), t.astype(np.float32)


def _colscale(rng, n, kind):
    n64 = -(-n // 64) * 64
    if kind is None:
        return None
    if kind == 'uniform':
        c = rng.uniform(0.5, 1.5, n64)
    elif kind == 'zeros':                                         # _DenseLseFn: zero past the anchors
        c = 1e-9 * np.exp2(-12 * rng.random(n64))
        c[rng.random(n64) < 0.2] = 0.0
    else:                                                         # the backward role: g ln2 / rowsum, max / min up to 2^12
        c = kind * np.exp2(-12 * rng.random(n64))
    return c.astype(np.float32)


def _hard_mantissas(n_r, n_c, d, off):
    """Rows whose last 8 entries have the mantissa 1.0000000000 1111111111111 (tf32 rounding can only go wrong there),
    all of one sign, with the rows of R parallel to rows of C so that one column dominates each row sum and S_ij = off."""
    m = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    T = np.zeros((n_c, d), np.float32)
    T[:, d - 8:] = m * np.float32(2.0 ** -2)
    T[:, :d - 8] = np.float32(1e-3)
    A = np.zeros((n_r, d), np.float32)
    A[:, d - 8:] = m * np.float32(2.0 ** 3)
    S = float((A[0].astype(np.float64) * T[0]).sum())
    return A, T, np.float32(S if off is None else off)


def cases():
    """(name, A, T, colscale, off, n_split) at the GPU file's shapes and regimes, at sizes the CPU runs in seconds."""
    rng = np.random.default_rng(7)
    out = []
    for d in (32, 64):
        for tau in (0.0899, 0.05, 0.02):                          # unit rows, the InfoNCE role
            off = LOG2E / tau
            out.append((f'unit tau={tau} d={d}', _unit(rng, 65, d, off), _unit(rng, 130, d, 1.0), None, off, 2))
        off = 16.5
        out.append((f'unit off=16.5 bwd d={d}', _unit(rng, 63, d, 1.0), _unit(rng, 129, d, off), _colscale(rng, 129, 1e-9), off, 3))
        out.append((f'unit uniform cs d={d}', _unit(rng, 64, d, off), _unit(rng, 200, d, 1.0), _colscale(rng, 200, 'uniform'), off, 1))
        # raw rows at offset 0, logits up to ~ +-60 natural units: a log2(e) / temp, t as they come
        A, t = raw_rows(rng, 127, 9, d, 0.2, 60.0)
        out.append((f'raw null cs ragged d={d}', A, t, None, 0.0, 1))
        out.append((f'raw bwd zeros d={d}', t, A, _colscale(rng, 127, 'zeros'), 0.0, 2))
        out.append((f'raw cs 1e-12 d={d}', A, t, _colscale(rng, 9, 1e-12), 0.0, 1))
        ac, tc = cancelling_rows(rng, 7, d, 1000.0)
        out.append((f'raw cancel d={d}', ac, tc, None, 0.0, 1))
        A, T, off = _hard_mantissas(8, 7, d, None)
        out.append((f'hard mantissas d={d}', A, T, None, off, 1))
    return out


def _ratios(name, A, T, cs, off, n_split, **wrong):
    rs_p, o_p = emulate(A, T, cs, off, n_split, **wrong)
    ref_rs, ref_o, b_rs, b_o = reference(A, T, None if cs is None else cs[:T.shape[0]], float(np.float32(off)), n_split)
    rs, o = rs_p.astype(np.float64).sum(0), o_p.astype(np.float64).sum(0)
    with np.errstate(invalid='ignore', divide='ignore'):
        r1 = np.nan_to_num(np.abs(rs - ref_rs) / b_rs, nan=np.inf)
        r2 = np.nan_to_num(np.abs(o - ref_o) / b_o, nan=np.inf, posinf=np.inf)
    r2 = np.where(np.abs(o - ref_o) == 0, 0.0, r2)
    return max(r1.max(initial=0.0), r2.max(initial=0.0))


CASES = cases()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_restatement_meets_the_bound(case):
    name, A, T, cs, off, n_split = case
    assert np.isfinite(A).all() and np.isfinite(T).all()
    r = _ratios(*case)
    print(f'{name}: max err / bound {r:.3f}')
    assert r <= 1.0, f'{name}: err / bound {r:.3f}'


@pytest.mark.parametrize('wrong', ['drop_r_lo', 'rz', 'drop_e_lo', 'no_mask'])
def test_wrong_restatements_miss_the_bound(wrong):
    worst = max(_ratios(*c, **{wrong: True}) for c in CASES)
    print(f'{wrong}: max err / bound {worst:.3f}')
    assert worst > 1.0, f'{wrong} meets the bound ({worst:.3f})'


def test_bound_has_the_plain_shape():
    """Pw <= (d/8) P, so the bound is at most (ln2 c1 max_j P_ij + c2 cols u) rowsum_i with c1 = c_P + d/8, c2 = 1/16 (rowsum)
    and 1/8 (O), plus terms independent of the operands."""
    for d in (32, 64):
        w = step_weights(d)
        assert w.max() == d / 8 and w.min() == 1
        c_p, c_w, base_rs, base_o, _ = bound_coefs(d, 4096, True)
        assert c_p + c_w * d / 8 < 4.3 + d / 8
        assert abs(base_rs - (4096 / 16) * U) < 8 * U and abs(base_o - (4096 / 8) * U) < 12 * U


def test_tf32_rounding_modes():
    x = np.float32([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 2.0 ** -10 - 2.0 ** -23, 3.0])
    np.testing.assert_array_equal(tf32(x), np.float32([1 + 2.0 ** -10, 1 + 2.0 ** -9, -(1 + 2.0 ** -10), 1 + 2.0 ** -10, 3.0]))
    np.testing.assert_array_equal(tf32(x, rz=True), np.float32([1, 1 + 2.0 ** -10, -1, 1, 3.0]))
    rng = np.random.default_rng(1)
    v = (rng.standard_normal(100000) * np.exp2(rng.integers(-60, 60, 100000))).astype(np.float32)
    hi, lo = split(v)
    res = np.abs(v.astype(np.float64) - hi - lo)
    assert (res <= U * np.abs(v.astype(np.float64))).all() and (np.abs(lo) <= 2.0 ** -11 * np.abs(v)).all()
