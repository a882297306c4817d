"""The 3xTF32 tensor-core InfoNCE contraction (ssl_softmax_gemm_tf32x3[_live]) through the C ABI against float64, within the
bound derived in test_host_tf32x3_bounds.py, on the paths only this kernel serves: raw rows at offset 0 (LightGCL, both roles),
offsets above 16 (tau < 0.0902), the device-bounded variants, ragged and one-tile shapes, every kind of n_split; then the
engine's routes onto it (dense_logsumexp_mean, cal_infonce_loss at small tau, the device-bounded spec-node term) with the
entry point that ran asserted.

Every partial output starts as NaN with a guard tail behind it: what must be written has to be finite and within the bound,
what must not be written (dead rows, the guard) has to stay NaN."""
import math

import pytest
import torch

from test_host_tf32x3_bounds import LOG2E, U, FLUSH, LN2, bound_coefs, chunk_cols, step_weights

pytestmark = pytest.mark.gpu

F32 = dict(device='cuda', dtype=torch.float32)
F64 = dict(device='cuda', dtype=torch.float64)
LIVE_ROWS, LIVE_COLS = 1, 2
SSL_E_ARG = -1
GUARD = 37
NUM_SM = 132


def _s():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from sslrec_b200._lib import lib, check
    return lib, check


def _report(group, ratio):
    print(f'ERR/BOUND {group} {ratio:.4g}')


class Op:
    """One operand as ssl_rows_normalize writes it for the 3xTF32 kernel: ``hat`` [npad, d] and the hi / lo row-major and
    transposed copies (pitch npad)."""

    def __init__(self, x, alpha, mode=0, npad=None):
        lib, check = _lib()
        n, d = x.shape
        self.n, self.d = n, d
        self.npad = npad = (max(64, (n + 63) // 64 * 64) if npad is None else npad)
        nan = lambda *s: torch.full(s, float('nan'), **F32)
        self.hat, self.hi, self.lo = nan(npad, d), nan(npad, d), nan(npad, d)
        self.thi, self.tlo = nan(d, npad), nan(d, npad)
        rinv = None if mode == 3 else torch.empty(max(n, 1), **F32)
        check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, mode, alpha, self.hat.data_ptr(), None,
                                     None if rinv is None else rinv.data_ptr(), self.hi.data_ptr(), self.lo.data_ptr(),
                                     self.thi.data_ptr(), self.tlo.data_ptr(), npad, _s()), 'ssl_rows_normalize')

    @property
    def rows(self):
        return self.hat[:self.n]


def _bufs(n_split, n_r, d, with_rowsum=True):
    """NaN-filled partial outputs with a guard tail: (rowsum view or None, O view, rowsum buffer, O buffer)."""
    rsb = torch.full((n_split * n_r + GUARD,), float('nan'), **F32) if with_rowsum else None
    ob = torch.full((n_split * n_r * d + GUARD,), float('nan'), **F32)
    rs = None if rsb is None else rsb[:n_split * n_r].view(n_split, n_r)
    return rs, ob[:n_split * n_r * d].view(n_split, n_r, d), rsb, ob


def _launch(R, n_r, C, n_c, cs, off, n_split, with_rowsum=True, live=None, role=LIVE_ROWS, expect_ok=True):
    lib, check = _lib()
    d = R.d
    rs, o, rsb, ob = _bufs(n_split, n_r, d, with_rowsum)
    args = (R.hi.data_ptr(), R.lo.data_ptr(), n_r, C.hi.data_ptr(), C.lo.data_ptr(), C.thi.data_ptr(), C.tlo.data_ptr(), C.npad, n_c, d,
            None if cs is None else cs.data_ptr(), off, n_split, None if rsb is None else rsb.data_ptr(), ob.data_ptr())
    if live is None:
        rc = lib.ssl_softmax_gemm_tf32x3(*args, _s())
    else:
        rc = lib.ssl_softmax_gemm_tf32x3_live(*args, live.data_ptr(), role, _s())
    torch.cuda.synchronize()
    if expect_ok:
        check(rc, 'ssl_softmax_gemm_tf32x3' + ('' if live is None else '_live'))
    assert torch.isnan(ob[n_split * n_r * d:]).all(), 'O guard tail written'
    if rsb is not None:
        assert torch.isnan(rsb[n_split * n_r:]).all(), 'rowsum guard tail written'
    return rs, o, rc


def reference(A, T, cs, off, n_split, extra_p=0.0, rows=2048):
    """float64 on the device: rowsum, O, W = E |T| and the bounds of test_host_tf32x3_bounds, for A [n_r, d] against T [n_c, d];
    ``off`` is the fp32 offset the kernel receives.  ``extra_p``: a further per-product error of the operands, in units of u P."""
    A, T = A.double(), T.double()
    n_r, d = A.shape
    n_c = T.shape[0]
    c_p, c_w, base_rs, base_o, slack = bound_coefs(d, chunk_cols(n_c, n_split), cs is not None)
    c_p += extra_p
    w = torch.tensor(step_weights(d), **F64)
    aT = T.abs()
    out = [torch.zeros(n_r, **F64), torch.zeros(n_r, d, **F64), torch.zeros(n_r, d, **F64), torch.zeros(n_r, **F64)]
    csd = None if cs is None else cs.double()
    for r in range(0, n_r, rows):
        a = A[r:r + rows]
        S = a @ T.T
        E = torch.exp2(S - off)
        if csd is not None:
            E = E * csd
        g1 = c_p * (a.abs() @ aT.T) + c_w * ((a.abs() * w) @ aT.T) + 0.5 * (S - off).abs()
        out[0][r:r + rows], out[1][r:r + rows], out[2][r:r + rows] = E.sum(1), E @ T, E @ aT
        out[3][r:r + rows] = LN2 * U * g1.max(1).values if n_c else 0.0
    rs, O, W, eps = out
    tmax = aT.max().item() if n_c else 0.0
    b_rs = slack * (eps + base_rs) * rs + n_c * FLUSH
    b_o = slack * (eps + base_o)[:, None] * W + n_c * FLUSH * tmax
    return dict(rs=rs, O=O, W=W, b_rs=b_rs, b_o=b_o, eps_rs=b_rs / rs)


def _within(rs, o, ref, what):
    """Partials summed in float64 against the reference; -> max err / bound."""
    worst = 0.0
    for got, want, bound, name in ((rs, ref['rs'], ref['b_rs'], 'rowsum'), (o, ref['O'], ref['b_o'], 'O')):
        if got is None:
            continue
        assert torch.isfinite(got).all(), f'{what}: {name} has non-finite or unwritten entries'
        err = (got.double().sum(0) - want).abs()
        r = (err / bound).max().item() if err.numel() else 0.0
        assert r <= 1.0, f'{what}: {name} err / bound {r:.3f} (max err {err.max().item():.3e})'
        worst = max(worst, r)
    return worst


def _colscale(n_pad, kind, g):
    if kind is None:
        return None
    if kind == 'uniform':
        c = torch.rand(n_pad, generator=g, dtype=torch.float64) + 0.5
    else:                       # the backward role: g ln2 / (B rowsum), max / min up to 2^12; 'zeros': a fifth of them 0
        mag = 1e-9 if kind == 'zeros' else kind
        c = mag * torch.exp2(-12.0 * torch.rand(n_pad, generator=g, dtype=torch.float64))
        if kind == 'zeros':
            c[torch.rand(n_pad, generator=g) < 0.2] = 0.0
    return c.float().cuda()


def _raw(B, n, d, temp, max_logit, g):
    """LightGCL's raw rows: a [B, d], t [n, d] with max |a . t| / temp = max_logit."""
    a, t = torch.randn(B, d, generator=g, dtype=torch.float64), torch.randn(n, d, generator=g, dtype=torch.float64)
    t *= max_logit * temp / (a @ t.T).abs().max()
    return a.float().cuda(), t.float().cuda()


# ---- 1. the kernel in both roles --------------------------------------------------------------------------------------

TAU_OFFS = [16.5, LOG2E / 0.05, LOG2E / 0.02, LOG2E / 0.0899]
# (n_r, n_c, d, n_split, offset, colscale, backward): backward = R is the table and C the anchors scaled by the offset
ROLE_CASES = [
    # the 12 cases of the former persistent-kernel file, now at offsets this kernel serves (InfoNCE role at tau < 0.0902)
    (83761, 4096, 64, 1, TAU_OFFS[1], 1e-9, True),      # the amazon backward role: 655 units, 5 rounds of 132 CTAs
    (83761, 4096, 64, 3, TAU_OFFS[1], None, False),
    (300, 1000, 64, 1, TAU_OFFS[0], None, False),
    (300, 1000, 64, 16, TAU_OFFS[2], 1e-12, True),       # n_split at its maximum (one C tile per unit)
    (300, 1000, 32, 1, TAU_OFFS[3], 'uniform', False),
    (300, 1000, 32, 16, TAU_OFFS[1], None, False),
    (4096, 9000, 64, 5, TAU_OFFS[2], None, False),
    (1000, 777, 32, 13, TAU_OFFS[0], 1e-9, True),
    (200, 778, 64, 1, TAU_OFFS[3], 'uniform', False),    # n_c % 8 = 2 and 3: the last column group is partly past n_c
    (300, 1003, 32, 2, TAU_OFFS[1], None, False),
    # ragged edges of both tile sizes, n_c % 8 and % 64 at every edge value
    (1, 1, 32, 1, TAU_OFFS[1], None, False),
    (63, 7, 64, 1, TAU_OFFS[2], 1e-9, True),
    (64, 8, 32, 1, TAU_OFFS[0], None, False),
    (65, 9, 64, 1, TAU_OFFS[3], 'zeros', True),
    (127, 63, 32, 1, TAU_OFFS[1], 'uniform', False),
    (128, 64, 64, 1, TAU_OFFS[2], None, False),
    (129, 65, 32, 2, TAU_OFFS[0], 1e-12, True),
    (4097, 83761, 64, 7, TAU_OFFS[1], None, False),      # the forward role at the amazon table; 7 does not divide 1309 tiles
    (4097, 83761, 32, 1309, TAU_OFFS[3], None, False),   # n_split at its maximum: 33 x 1309 units
    (83761, 4096, 32, 'choose', TAU_OFFS[2], 1e-12, True),
    (4096, 83761, 64, 'choose', TAU_OFFS[0], None, False),
]


def _split(n_split, n_r, n_c):
    if n_split != 'choose':
        return n_split
    from sslrec_b200 import engine
    return engine.choose_split((n_r + 127) // 128, (n_c + 63) // 64, slots=NUM_SM, prefer_few=True)


@pytest.mark.parametrize('n_r,n_c,d,n_split,off,cs_kind,backward', ROLE_CASES)
def test_unit_rows_match_float64(n_r, n_c, d, n_split, off, cs_kind, backward):
    g = torch.Generator().manual_seed(n_r + 3 * n_c + d)
    off = float(torch.tensor(off, dtype=torch.float32))
    n_split = _split(n_split, n_r, n_c)
    # forward: R = anchors scaled by the offset, C = unit table rows; backward: R = unit table rows, C = scaled anchors
    R = Op(torch.randn(n_r, d, generator=g).cuda(), 1.0 if backward else off)
    C = Op(torch.randn(n_c, d, generator=g).cuda(), off if backward else 1.0)
    cs = _colscale(C.npad, cs_kind, g)
    rs, o, _ = _launch(R, n_r, C, n_c, cs, off, n_split)
    ref = reference(R.rows, C.rows, None if cs is None else cs[:n_c], off, n_split)
    _report('kernel-roles', _within(rs, o, ref, f'{n_r}x{n_c} d={d} split={n_split}'))


# raw rows at offset 0 (LightGCL): (B, n, d, n_split, max_logit, colscale of the backward role)
RAW_CASES = [(1000, 777, 32, 1, 60.0, None), (4097, 83761, 64, 4, 60.0, None), (129, 9, 64, 1, 60.0, None),
             (65, 7, 32, 1, 40.0, None), (300, 1003, 64, 2, 60.0, 'zeros'), (2000, 5000, 32, 'choose', 60.0, 'zeros'),
             (127, 63, 64, 1, 60.0, 1e-12)]


@pytest.mark.parametrize('B,n,d,n_split,max_logit,cs_kind', RAW_CASES)
def test_raw_rows_match_float64(B, n, d, n_split, max_logit, cs_kind):
    """Both roles of _DenseLseFn: forward R = a log2(e) / temp, C = t; backward R = t, C = the scaled anchors with colscale."""
    g = torch.Generator().manual_seed(B + n + d)
    temp = 0.2
    a, t = _raw(B, n, d, temp, max_logit, g)
    A, T = Op(a, LOG2E / temp, 3), Op(t, 1.0, 3)
    ns = _split(n_split, B, n)
    rs, o, _ = _launch(A, B, T, n, None, 0.0, ns)
    _report('raw-rows', _within(rs, o, reference(A.rows, T.rows, None, 0.0, ns), f'raw fwd {B}x{n}'))
    cs = _colscale(A.npad, cs_kind or 1e-9, g)
    ns = _split(n_split, n, B)
    rs, o, _ = _launch(T, n, A, B, cs, 0.0, ns, with_rowsum=False)
    _report('raw-rows', _within(None, o, reference(T.rows, A.rows, cs[:B], 0.0, ns), f'raw bwd {n}x{B}'))


@pytest.mark.parametrize('d', [32, 64])
def test_raw_rows_large_products_that_cancel(d):
    """sum_k |a_k t_k| ~ 1000 (log2 units) while a . t stays within a few units: the regime where the bound is tight."""
    from test_host_tf32x3_bounds import cancelling_rows
    import numpy as np
    a, t = cancelling_rows(np.random.default_rng(d), 200, d, 1000.0)
    A, T = Op(torch.from_numpy(a).cuda(), 1.0, 3), Op(torch.from_numpy(np.repeat(t, 70, 0)).cuda(), 1.0, 3)
    rs, o, _ = _launch(A, 200, T, 70, None, 0.0, 1)
    _report('raw-rows', _within(rs, o, reference(A.rows, T.rows, None, 0.0, 1), 'cancel'))


@pytest.mark.parametrize('d', [32, 64])
def test_null_colscale_on_ragged_columns(d):
    """No colscale, raw rows at offset 0: the padding rows of C are zero, so an unmasked column would add exactly 1."""
    g = torch.Generator().manual_seed(d)
    for n_c in (1, 7, 9, 63, 65, 777):
        a, t = _raw(130, n_c, d, 0.2, 5.0, g)
        A, T = Op(a, LOG2E / 0.2, 3), Op(t, 1.0, 3)
        rs, o, _ = _launch(A, 130, T, n_c, None, 0.0, 1)
        _report('raw-rows', _within(rs, o, reference(A.rows, T.rows, None, 0.0, 1), f'null cs n_c={n_c}'))


@pytest.mark.parametrize('d', [32, 64])
def test_writer_zeroes_the_padding_of_raw_operands(d):
    """The kernel multiplies the transposed copy's columns [n_c, ceil8(n_c)) by a masked E = 0, so they must be finite: the
    writer zeroes every padding row and column, for raw rows (norm mode 3) as _DenseLseFn builds them too."""
    g = torch.Generator().manual_seed(d)
    for n in (1, 7, 65, 130):
        a, _ = _raw(n, 3, d, 0.2, 60.0, g)
        for alpha in (LOG2E / 0.2, 1.0):
            op = Op(a, alpha, 3, npad=max(64, (n + 63) // 64 * 64))
            # the transposed copy holds row c at column (c & ~7) | (c & 7) >> 1 | (c & 1) << 2 (the kernel's fragment order)
            c = torch.arange(n, op.npad, device='cuda')
            q = (c & ~7) | ((c & 7) >> 1) | ((c & 1) << 2)
            for x in (op.hat[n:], op.hi[n:], op.lo[n:], op.thi[:, q], op.tlo[:, q]):
                assert (x == 0).all()
            assert torch.isfinite(op.thi).all() and torch.isfinite(op.tlo).all()
            assert torch.equal(op.hat[:n], (a * torch.tensor(alpha, dtype=torch.float32)).float())


# ---- 2. the device-bounded variants ---------------------------------------------------------------------------------------

@pytest.mark.parametrize('d', [32, 64])
def test_live_rows_match_float64(d):
    g = torch.Generator().manual_seed(10 + d)
    off = float(torch.tensor(LOG2E / 0.05, dtype=torch.float32))
    cap, n_c, ns = 1000, 3000, 4
    A = Op(torch.randn(cap, d, generator=g).cuda(), off)
    T = Op(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    ref = reference(A.rows, T.rows, None, off, ns)
    worst = 0.0
    for live_n in (0, 1, 63, 64, 65, cap - 1, cap, -3, cap + 5):
        n = min(max(live_n, 0), cap)
        live = torch.tensor([live_n], dtype=torch.int64, device='cuda')
        rs, o, _ = _launch(A, cap, T, n_c, None, off, ns, live=live, role=LIVE_ROWS)
        assert torch.isnan(rs[:, n:]).all() and torch.isnan(o[:, n:]).all(), f'live {live_n}: dead rows written'
        sub = {k: v[:n] for k, v in ref.items()}
        worst = max(worst, _within(rs[:, :n], o[:, :n], sub, f'live rows {live_n}'))
    _report('live', worst)


@pytest.mark.parametrize('d', [32, 64])
@pytest.mark.parametrize('with_cs', [True, False])
def test_live_cols_match_float64(d, with_cs):
    """The backward role: only the first live rows of C (the anchors) count; colscale past them is NaN and never read.  The
    TMA maps span the capacity, so the live count alone masks.  Splits with no live tile write zero partials."""
    g = torch.Generator().manual_seed(20 + d + with_cs)
    off = float(torch.tensor(LOG2E / 0.02, dtype=torch.float32))
    cap, n_r = 1000, 700
    ns = (cap + 63) // 64                                   # 16: the maximum, so small live counts leave empty splits
    T = Op(torch.randn(n_r, d, generator=g).cuda(), 1.0)
    A = Op(torch.randn(cap, d, generator=g).cuda(), off)
    cs_full = _colscale(A.npad, 1e-9, g) if with_cs else None
    worst = 0.0
    for live_n in (0, 1, 63, 64, 65, cap - 1, cap, -3, cap + 5):
        n = min(max(live_n, 0), cap)
        live = torch.tensor([live_n], dtype=torch.int64, device='cuda')
        cs = None
        if with_cs:
            cs = cs_full.clone()
            cs[n:] = float('nan')
        rs, o, _ = _launch(T, n_r, A, cap, cs, off, ns, live=live, role=LIVE_COLS)
        n_ct = (n + 63) // 64
        for sp in range(ns):
            if n_ct * sp // ns == n_ct * (sp + 1) // ns:
                assert (rs[sp] == 0).all() and (o[sp] == 0).all(), f'live {live_n}: empty split {sp} not zero'
        if n == 0:
            assert (rs == 0).all() and (o == 0).all()
            continue
        ref = reference(T.rows, A.rows[:n], None if cs is None else cs_full[:n], off, ns)
        worst = max(worst, _within(rs, o, ref, f'live cols {live_n}'))
    _report('live', worst)


# ---- 3. relaunch, rejected arguments, empty launches ------------------------------------------------------------------

@pytest.mark.parametrize('n_r,n_c,d,n_split', [(83761, 4096, 64, 1), (4096, 9000, 32, 4), (300, 1003, 64, 2)])
def test_relaunch_is_bit_identical(n_r, n_c, d, n_split):
    g = torch.Generator().manual_seed(11)
    off = LOG2E / 0.05
    R = Op(torch.randn(n_r, d, generator=g).cuda(), off)
    C = Op(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    cs = _colscale(C.npad, 'uniform', g)
    rs1, o1, _ = _launch(R, n_r, C, n_c, cs, off, n_split)
    rs2, o2, _ = _launch(R, n_r, C, n_c, cs, off, n_split)
    assert torch.isfinite(o1).all() and torch.equal(rs1, rs2) and torch.equal(o1, o2)


def test_rejected_arguments_write_nothing():
    lib, _ = _lib()
    d, n = 64, 256
    g = torch.Generator().manual_seed(5)
    R, C = Op(torch.randn(n, d, generator=g).cuda(), 7.0), Op(torch.randn(n, d, generator=g).cuda(), 1.0)
    rs, o, rsb, ob = _bufs(1, n, d)
    live = torch.tensor([n], dtype=torch.int64, device='cuda')
    cs_buf = torch.zeros(C.npad + 4, **F32)
    base = dict(rh=R.hi.data_ptr(), rl=R.lo.data_ptr(), ch=C.hi.data_ptr(), cl=C.lo.data_ptr(), th=C.thi.data_ptr(), tl=C.tlo.data_ptr(),
                pitch=C.npad, nc=n, d=d, cs=None, ns=1, o=ob.data_ptr())
    bad = [dict(rh=None), dict(rl=None), dict(ch=None), dict(cl=None), dict(th=None), dict(tl=None), dict(o=None),
           dict(pitch=248, nc=250), dict(pitch=258), dict(d=48), dict(ns=0), dict(ns=5), dict(rh=R.hi.data_ptr() + 4),
           dict(tl=C.tlo.data_ptr() + 4), dict(o=ob.data_ptr() + 4), dict(cs=cs_buf.data_ptr() + 4)]
    for b in bad:
        a = {**base, **b}
        args = (a['rh'], a['rl'], n, a['ch'], a['cl'], a['th'], a['tl'], a['pitch'], a['nc'], a['d'], a['cs'], 7.0, a['ns'],
                rsb.data_ptr(), a['o'])
        assert lib.ssl_softmax_gemm_tf32x3(*args, _s()) == SSL_E_ARG, b
        assert lib.ssl_softmax_gemm_tf32x3_live(*args, live.data_ptr(), LIVE_ROWS, _s()) == SSL_E_ARG, b
    args = (base['rh'], base['rl'], n, base['ch'], base['cl'], base['th'], base['tl'], base['pitch'], n, d, None, 7.0, 1,
            rsb.data_ptr(), ob.data_ptr())
    assert lib.ssl_softmax_gemm_tf32x3_live(*args, None, LIVE_ROWS, _s()) == SSL_E_ARG
    for role in (0, 3):
        assert lib.ssl_softmax_gemm_tf32x3_live(*args, live.data_ptr(), role, _s()) == SSL_E_ARG
    # empty launches succeed and write nothing
    for n_r, n_c in ((0, n), (n, 0), (0, 0)):
        a = (base['rh'], base['rl'], n_r, base['ch'], base['cl'], base['th'], base['tl'], base['pitch'], n_c, d, None, 7.0, 1,
             rsb.data_ptr(), ob.data_ptr())
        assert lib.ssl_softmax_gemm_tf32x3(*a, _s()) == 0
        for role in (LIVE_ROWS, LIVE_COLS):
            assert lib.ssl_softmax_gemm_tf32x3_live(*a, live.data_ptr(), role, _s()) == 0
    torch.cuda.synchronize()
    assert torch.isnan(rsb).all() and torch.isnan(ob).all()


# ---- 4. the engine's routes onto this kernel ------------------------------------------------------------------------------

def _record(monkeypatch):
    from test_gpu_model_paths import _record as rec
    return rec(monkeypatch)


def _lse_bounds(a, t, temp, g_out):
    """float64 value, gradients and derived bounds of mean_b log(sum_j exp(a_b . t_j / temp) + eps) as _DenseLseFn computes it:
    the forward contraction's bounds (plus the rounding of a log2(e) / temp, u/2 per product), the finalize (obar = O / rowsum,
    log) and the backward contraction with colscale g ln2 / (B rowsum), whose rowsum carries the forward's error."""
    B, d = a.shape
    alpha = float(torch.tensor(LOG2E / temp, dtype=torch.float32))
    A = (a * torch.tensor(alpha, dtype=torch.float32, device=a.device)).double()
    f = reference(A, t, None, 0.0, 1, extra_p=0.5)
    rs = f['rs']
    e_rs = f['b_rs'] / rs
    loss_b = f['b_rs'] / (rs + 1e-8) + 4 * U * torch.log(rs + 1e-8).abs()
    b_loss = loss_b.mean().item() + 2 * U * abs(torch.log(rs + 1e-8).mean().item())
    scale = g_out / (B * temp)
    ga = f['O'] / rs[:, None] * scale
    b_ga = (f['b_o'] / rs[:, None] + f['O'].abs() * e_rs[:, None] / rs[:, None]) * abs(scale) + 4 * U * ga.abs()
    cs = g_out * LN2 / (B * rs)
    bk = reference(t, A, cs, 0.0, 1, extra_p=0.5)
    gt = bk['O']
    b_gt = bk['b_o'] + bk['W'] * (e_rs.max().item() + 3 * U)
    return b_loss, ga, b_ga, gt, b_gt


LSE_CASES = [(32, 129, 1000, 60.0), (64, 1000, 4097, 60.0), (64, 63, 65, 40.0), (32, 1, 7, 60.0)]


@pytest.mark.parametrize('d,B,n,max_logit', LSE_CASES)
def test_dense_logsumexp_mean_matches_float64(d, B, n, max_logit, monkeypatch):
    from sslrec_b200 import engine
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', True)
    g = torch.Generator().manual_seed(B + n)
    temp, g_out = 0.2, 1.7
    a, t = _raw(B, n, d, temp, max_logit, g)
    rec = _record(monkeypatch)
    ins = [x.clone().requires_grad_(True) for x in (a, t)]
    out = engine.dense_logsumexp_mean(ins[0], ins[1], temp, 1e-8)
    (out * g_out).backward()
    torch.cuda.synchronize()
    assert rec.calls == ['ssl_softmax_gemm_tf32x3'] * 2, rec.calls
    a64, t64 = a.double().requires_grad_(True), t.double().requires_grad_(True)
    want = torch.log(torch.exp(a64 @ t64.T / temp).sum(1) + 1e-8).mean()
    (want * g_out).backward()
    b_loss, _, b_ga, _, b_gt = _lse_bounds(a, t, temp, g_out)
    worst = abs(out.item() - want.item()) / b_loss
    assert worst <= 1.0, (out.item(), want.item(), b_loss)
    for got, ref, bound, name in ((ins[0].grad, a64.grad, b_ga, 'anchors'), (ins[1].grad, t64.grad, b_gt, 'table')):
        r = ((got.double() - ref).abs() / bound).max().item()
        assert r <= 1.0, f'grad {name}: err / bound {r:.3f}'
        worst = max(worst, r)
    _report('engine-routes', worst)


def test_dense_logsumexp_mean_gathered_anchors(monkeypatch):
    """Anchors a gathered, non-leaf slice of a larger tensor and the table a slice of it, as LightGCL passes them; B and n ragged."""
    from sslrec_b200 import engine
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', True)
    g = torch.Generator().manual_seed(3)
    d, n, B, temp = 64, 777, 300, 0.2
    base = torch.randn(n + 50, d, generator=g, dtype=torch.float64)
    idx = torch.randint(0, n, (B,), generator=g)
    s = 60.0 * temp / (base[:n][idx] @ base[:n].T).abs().max().item()
    big = (base * math.sqrt(s)).float().cuda().requires_grad_(True)
    rec = _record(monkeypatch)
    out = engine.dense_logsumexp_mean(big[:n][idx.cuda()], big[:n], temp)
    out.backward()
    torch.cuda.synchronize()
    assert rec.calls == ['ssl_softmax_gemm_tf32x3'] * 2, rec.calls
    b64 = big.detach().double().requires_grad_(True)
    want = torch.log(torch.exp(b64[:n][idx.cuda()] @ b64[:n].T / temp).sum(1) + 1e-8).mean()
    want.backward()
    b_loss, _, b_ga, _, b_gt = _lse_bounds(big.detach()[:n][idx.cuda()], big.detach()[:n], temp, 1.0)
    bound = torch.zeros_like(b64)
    bound[:n] += b_gt
    bound.index_add_(0, idx.cuda(), b_ga)
    bound += 8 * U * b64.grad.abs()                           # the fp32 sums of the gathered rows' gradients
    r = max(abs(out.item() - want.item()) / b_loss, ((big.grad.double() - b64.grad).abs() / bound).max().item())
    assert r <= 1.0, r
    _report('engine-routes', r)


@pytest.mark.parametrize('d', [32, 64])
def test_dense_logsumexp_mean_past_the_exp_range(d, monkeypatch):
    """One logit of 150 (exp overflows fp32 at 88.7), all others 0: the float32 reference formula gives loss inf, a NaN
    gradient on that anchor row and on that table row (inf / inf) and finite ones elsewhere.  The engine returns the same:
    the overflow stays in its row and column, every other gradient row matches float64."""
    from sslrec_b200 import engine
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', True)
    g = torch.Generator().manual_seed(d)
    B, n, temp = 130, 70, 0.2
    e = torch.zeros(d, dtype=torch.float64)
    e[0] = 1.0
    a = torch.randn(B, d, generator=g, dtype=torch.float64) * 0.3
    t = torch.randn(n, d, generator=g, dtype=torch.float64) * 0.3
    a[:, 0] = 0.0
    t[:, 0] = 0.0
    a[5], t[9] = e * math.sqrt(150 * temp), e * math.sqrt(150 * temp)      # a_5 . t_9 / temp = 150; a_5, t_9 orthogonal to the rest
    a[5, 1:], t[9, 1:] = 0.0, 0.0
    a, t = a.float().cuda(), t.float().cuda()
    ins = [x.clone().requires_grad_(True) for x in (a, t)]
    out = engine.dense_logsumexp_mean(ins[0], ins[1], temp, 1e-8)
    out.backward()
    r32 = [x.clone().requires_grad_(True) for x in (a, t)]
    w32 = torch.log(torch.exp(r32[0] @ r32[1].T / temp).sum(1) + 1e-8).mean()
    w32.backward()
    assert math.isinf(out.item()) and out.item() > 0 and math.isinf(w32.item())
    for got, ref, row in ((ins[0].grad, r32[0].grad, 5), (ins[1].grad, r32[1].grad, 9)):
        assert torch.equal(torch.isnan(got).any(1), torch.isnan(ref).any(1))
        bad = torch.isnan(got).any(1).nonzero().flatten().tolist()
        assert bad == [row], bad
    # every other row against float64, within the bounds of the 129 anchors without the overflow (mean over 130)
    keep_a, keep_t = torch.ones(B, dtype=torch.bool, device='cuda'), torch.ones(n, dtype=torch.bool, device='cuda')
    keep_a[5], keep_t[9] = False, False
    a64, t64 = a.double().requires_grad_(True), t.double().requires_grad_(True)
    want = torch.log(torch.exp(a64 @ t64.T / temp).sum(1) + 1e-8).mean()
    want.backward()
    _, _, b_ga, _, b_gt = _lse_bounds(a[keep_a], t, temp, (B - 1) / B)
    r = max(((ins[0].grad[keep_a].double() - a64.grad[keep_a]).abs() / b_ga).max().item(),
            ((ins[1].grad[keep_t].double() - t64.grad[keep_t]).abs() / b_gt[keep_t]).max().item())
    assert r <= 1.0, r
    _report('engine-routes', r)


def _infonce_tol(want, grads):
    import ssl_test_helpers as H
    return H.LOSS_RTOL * max(1.0, abs(want)), [H.GRAD_RTOL * x.abs().max().item() for x in grads]


@pytest.mark.parametrize('d', [32, 64])
@pytest.mark.parametrize('tau', [0.02, 0.05, 0.0899])
def test_cal_infonce_loss_matches_float64(d, tau, monkeypatch):
    """cal_infonce_loss on dense rows with repeated anchors and a 1000-row table (not a multiple of 64)."""
    from oracle import cf_oracle as O
    from sslrec_b200 import engine, loss_utils
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', True)
    g = torch.Generator().manual_seed(int(tau * 1e4) + d)
    n, B = 1000, 300
    x1, x2 = torch.randn(n, d, generator=g), torch.randn(n, d, generator=g)
    # views that agree only weakly: where the positive takes nearly all of the softmax, the loss and gradient are small
    # differences of O(1 / tau) terms that no float32 evaluation resolves (see ssl_test_helpers._path_matrix)
    x2 = 0.3 * x1 + x2
    idx = torch.randint(0, 200, (B,), generator=g)               # repeated anchors
    ins = [x.cuda().requires_grad_(True) for x in (x1, x2)]
    rec = _record(monkeypatch)
    out = loss_utils.cal_infonce_loss(ins[0][idx.cuda()], ins[1][idx.cuda()], ins[1], tau)
    out.backward()
    torch.cuda.synchronize()
    assert rec.calls == ['ssl_softmax_gemm_tf32x3'] * 2, rec.calls
    r64 = [x.double().requires_grad_(True) for x in (x1, x2)]
    want = O.infonce_loss_sum(r64[0][idx], r64[1][idx], r64[1], tau)
    want.backward()
    tl, tg = _infonce_tol(want.item(), [r.grad for r in r64])
    worst = abs(out.item() - want.item()) / tl
    for got, ref, tol in zip(ins, r64, tg):
        worst = max(worst, (got.grad.cpu().double() - ref.grad).abs().max().item() / tol)
    assert worst <= 1.0, worst
    _report('engine-routes', worst)


@pytest.mark.parametrize('d', [32, 64])
def test_spec_nodes_dev_matches_float64_and_the_unique_path(d, monkeypatch):
    """HCCF's spec-node term at tau = 0.05 with the node list de-duplicated on the device: the _live route, against float64
    and against the torch.unique path (the plain launch)."""
    from oracle import cf_oracle as O
    from sslrec_b200 import engine
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', True)
    g = torch.Generator().manual_seed(50 + d)
    n, tau = 1300, 0.05
    e1, e2 = torch.randn(n, d, generator=g), torch.randn(n, d, generator=g)
    e2 = 0.3 * e1 + e2                                           # weakly agreeing views, as in the test above
    ids = torch.randint(0, 700, (900,), generator=g)
    res = []
    for dev_path in (True, False):
        ins = [x.cuda().requires_grad_(True) for x in (e1, e2)]
        rec = _record(monkeypatch)
        if dev_path:
            out = engine.dense_infonce_spec_nodes_mean_dev(ins[0], ins[1], ids.cuda(), tau)
        else:
            out = engine.dense_infonce_spec_nodes_mean(ins[0], ins[1], torch.unique(ids).cuda(), tau)
        out.backward()
        torch.cuda.synchronize()
        want_calls = ['ssl_softmax_gemm_tf32x3_live'] * 2 if dev_path else ['ssl_softmax_gemm_tf32x3'] * 2
        assert rec.calls == want_calls, rec.calls
        monkeypatch.setattr(engine, 'lib', rec._lib)
        res.append((out.item(), ins[0].grad.cpu().double(), ins[1].grad.cpu().double()))
    r64 = [x.double().requires_grad_(True) for x in (e1, e2)]
    want = O.infonce_spec_nodes_mean(r64[0], r64[1], torch.unique(ids), tau)
    want.backward()
    tl, tg = _infonce_tol(want.item(), [r.grad for r in r64])
    worst = 0.0
    for loss, g1, g2 in res:
        worst = max(worst, abs(loss - want.item()) / tl, (g1 - r64[0].grad).abs().max().item() / tg[0],
                    (g2 - r64[1].grad).abs().max().item() / tg[1])
    assert worst <= 1.0, worst
    # the two paths differ only in summation order: the live launch runs at the list's capacity
    assert abs(res[0][0] - res[1][0]) <= 1e-5 * max(1.0, abs(res[1][0]))
    _report('engine-routes', worst)
