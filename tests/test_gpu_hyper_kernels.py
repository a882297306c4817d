"""HCCF's hyper-graph kernels (csrc/hyper.cu) through the C ABI against float64, at every instantiation and load path:

a. ssl_rowgemm: n_out across the four column-per-thread buckets (CPT 1, 2, 4, 8) and their edges; k1 / k2 multiples of 4
   and not; every M1 / M2 orientation; in2 absent and present; the pre_ref derivative multiply at slopes 0, 0.2 and 1;
   scale, slope and accumulate; contiguous, row-strided and one-float-offset operands (the 16-byte and the scalar staging
   branch); a strided output with NaN padding and a NaN row past the end; n_rows around one tile and past the 264-CTA
   grid.  Each output is checked bit for bit against the sequential fp32 FMA chain the kernel computes, and against
   float64 within a bound derived from sum |terms|.
b. ssl_colgemm: all 16 <N1, N2> instantiations with k a multiple of 4 and not; mode 0 with and without out_act, mode 1;
   pre_ref on in2; scale; n_rows from one row to 1000 tiles (multi-tile CTAs, empty trailing CTAs); NaN-filled partials
   with a NaN guard tail; two launches bit-identical.  A second run on non-negative inputs, where the bound is relative
   and a lost 64-row tile exceeds it.
c. ssl_hyper_dropout / ssl_hyper_dropout_dev: the in-kernel mask bit for bit against oracle/philox.hyper_keep; mode 1 equals
   mode 2 fed that mask, forward and accumulating; the device seed equals the host seed; keep = 1 keeps everything.
d. rejected arguments leave NaN-sentinel outputs untouched; n_rows = 0 with null row pointers is accepted.

The worst err / bound of each group is printed when the module finishes (visible with pytest -s)."""
import zlib

import numpy as np
import pytest
import torch

from oracle import philox as P

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                       # unit roundoff of fp32
NAN = float('nan')
F32 = dict(device='cuda', dtype=torch.float32)
TILE, ROW_GRID, COL_GRID = 64, 2 * 132, 3 * 132      # rows per tile; rowgemm's and colgemm's grid caps (132 SMs)

_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
    yield
    if _WORST:
        print('\nworst err/bound: ' + ', '.join(f'{k} {v:.3e}' for k, v in sorted(_WORST.items())))


def _L():
    from sslrec_b200._lib import lib, check
    return lib, check


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _nan(*shape):
    return torch.full(shape, NAN, **F32)


def _f32(x):
    """The float32 value a Python float becomes at the C ABI."""
    return float(np.float32(x))


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _within(group, got, ref, bound, what):
    """|got - ref| <= bound elementwise (NaN fails); records the worst err / bound of the group."""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (f'{what}: {int(bad.sum())} / {bad.numel()} off, max err {err.max().item():.3e}, '
                           f'max err/bound {(err / bound).max().item():.3e}')
    if err.numel():
        _WORST[group] = max(_WORST.get(group, 0.0), (err / bound.clamp_min(1e-300)).max().item())


def _rejected(rc, what):
    from sslrec_b200._lib import lib
    assert rc != 0, f'{what} was accepted'
    assert lib.ssl_last_error(), what


def _in_layout(data, layout):
    """A [n, k] operand in one of three layouts: 'contig' (row stride k), 'strided' (row stride k + 8) or 'offset' (one float
    past a 16-byte boundary, row stride k + 5: the scalar staging branch whatever k is).  The columns around it hold NaN,
    so a read past the operand poisons the result."""
    if layout == 'contig':
        return data.contiguous()
    n, k = data.shape
    base = _nan(n, k + (8 if layout == 'strided' else 5))
    off = 0 if layout == 'strided' else 1
    v = base[:, off:off + k]
    v.copy_(data)
    return v


def _leaky(x, slope):
    return torch.where(x > 0, x, x * slope)


def _act_grad(pre_ref, slope):
    """act'(.) from the saved output as the kernels load it: 1 where pre_ref > 0, else slope (float32)."""
    return torch.where(pre_ref > 0, torch.ones_like(pre_ref), torch.full_like(pre_ref, slope))


# =====================================================================================================================
# a. ssl_rowgemm
# =====================================================================================================================

def _rowgemm_chain(xs, ms, scale, slope, prev):
    """The kernel's arithmetic restated: acc = fmaf(x_k, m_k, acc) for k = 0 .. K-1 over in1's columns, then in2's; then
    leaky(acc * scale) and, accumulating, prev + that -- each step rounded to fp32.  x_k m_k is exact in float64, so a
    step is the fp32 rounding of the float64 sum: at most a rare double-rounding difference from a true fma."""
    s = torch.zeros(xs[0].shape[0], ms[0].shape[1], dtype=torch.float64, device='cuda')
    for x, m in zip(xs, ms):
        x, m = x.double(), m.double()
        for k in range(x.shape[1]):
            s = (x[:, k:k + 1] * m[k] + s).float().double()
    v = _leaky(s.float() * scale, slope)
    return v if prev is None else prev + v


def _rowgemm_case(n, n_out, k1, k2, t1, t2, pre_slope, scale, slope, accumulate, layout, what):
    """One ssl_rowgemm call: k2 = 0 means no in2; pre_slope None means no pre_ref.  Operands and out in `layout`."""
    lib, check = _L()
    g = _gen('rowgemm', n, n_out, k1, k2, t1, t2, pre_slope, layout)
    scale, slope = _f32(scale), _f32(slope)
    in1 = _in_layout(torch.randn(n, k1, generator=g, **F32), layout)
    in2 = _in_layout(torch.randn(n, k2, generator=g, **F32), layout) if k2 else None
    pre = _in_layout(torch.randn(n, k1, generator=g, **F32), layout) if pre_slope is not None else None
    pre_slope = _f32(pre_slope if pre_slope is not None else 1.0)
    M1 = torch.randn(k1, n_out, generator=g, **F32) * 0.3                 # the logical [k, n_out] matrices
    M2 = torch.randn(k2, n_out, generator=g, **F32) * 0.3 if k2 else None
    m1 = M1.T.contiguous() if t1 else M1
    m2 = None if M2 is None else (M2.T.contiguous() if t2 else M2)
    pad, off = {'contig': (0, 0), 'strided': (4, 0), 'offset': (5, 1)}[layout]
    base = _nan(n + 1, n_out + pad)                                       # one NaN row past the end, NaN padding columns
    out = base[:n, off:off + n_out]
    prev = None
    if accumulate:
        out.copy_(torch.randn(n, n_out, generator=g, **F32))
        prev = out.clone()
    check(lib.ssl_rowgemm(in1.data_ptr(), in1.stride(0), k1, m1.data_ptr(), t1, _p(in2), 0 if in2 is None else in2.stride(0), k2,
                          _p(m2), t2, _p(pre), 0 if pre is None else pre.stride(0), pre_slope, out.data_ptr(), out.stride(0), n_out,
                          scale, slope, int(accumulate), n, _s()), 'ssl_rowgemm')
    torch.cuda.synchronize()
    untouched = torch.ones_like(base, dtype=torch.bool)
    untouched[:n, off:off + n_out] = False
    assert base[untouched].isnan().all(), f'{what}: written outside out[:n_rows, :n_out]'
    x1 = in1 if pre is None else in1 * _act_grad(pre, pre_slope)         # the fp32 product the kernel stages
    xs, ms = [x1] + ([in2] if k2 else []), [M1] + ([M2] if k2 else [])
    chain = _rowgemm_chain(xs, ms, scale, slope, prev)
    bit_equal = (out == chain).double().mean().item()
    assert bit_equal >= 0.9999, f'{what}: {bit_equal:.6f} of the outputs equal the fp32 FMA chain'
    # float64: every step of the chain is off by at most u |partial sum| <= u sum |terms|; the staged product, * scale, leaky
    # (Lipschitz 1 for 0 <= slope <= 1) and + prev add one rounding each
    x1d = in1.double() * (1.0 if pre is None else _act_grad(pre, pre_slope).double())
    exact = x1d @ M1.double() + (in2.double() @ M2.double() if k2 else 0.0)
    absum = x1d.abs() @ M1.double().abs() + (in2.double().abs() @ M2.double().abs() if k2 else 0.0)
    ref = _leaky(scale * exact, slope) + (0.0 if prev is None else prev.double())
    bound = (k1 + k2 + 6) * U * (abs(scale) * absum + (0.0 if prev is None else prev.double().abs())) + 1e-300
    _within('a rowgemm', out, ref, bound, what)


NOUTS = [4, 13, 16, 17, 32, 33, 37, 64, 65, 100, 128]
KS = [(4, 0), (13, 0), (32, 37), (37, 64), (64, 13), (127, 128), (128, 128)]      # (k1, k2); k2 = 0: no in2
PRE_SLOPES = [None, 0.0, 0.2, 1.0]
LAYOUTS = ('contig', 'strided', 'offset')
ROWS = (1, 63, 64, 65)


@pytest.mark.parametrize('n_out', NOUTS)
def test_rowgemm_matches_fp32_chain_and_float64(n_out):
    """For every (k1, k2) and layout, the other arguments rotate so that each meets each: the four M orientations, pre_ref
    (every (k1, k2) pair keeps one pre slope across the three layouts, so (32, 37) and (128, 128) run the scalar branch with
    slope 0.2), scale 1 / 1.3 / -0.8, output slope 1 / 0.5 / 0.2, accumulate, n_rows 1 / 63 / 64 / 65.
    k1 = k2 = 128 at n_out = 128 takes the largest dynamic shared memory (196 864 B)."""
    for i, (k1, k2) in enumerate(KS):
        for j, layout in enumerate(LAYOUTS):
            c = i + j
            args = dict(n=ROWS[(c + n_out) % 4], n_out=n_out, k1=k1, k2=k2, t1=c % 2, t2=(c // 2) % 2, pre_slope=PRE_SLOPES[i % 4],
                        scale=(1.0, 1.3, -0.8)[c % 3], slope=(1.0, 0.5, 0.2)[(i + 2 * j) % 3], accumulate=(j + n_out) % 2,
                        layout=layout)
            _rowgemm_case(**args, what=' '.join(f'{k}={v}' for k, v in args.items()))


@pytest.mark.parametrize('n_out,k1,k2,layout,pre_slope', [(128, 128, 128, 'strided', 0.2), (17, 37, 0, 'contig', 0.0),
                                                         (65, 64, 13, 'offset', 0.2), (33, 64, 64, 'contig', None)])
def test_rowgemm_past_the_grid(n_out, k1, k2, layout, pre_slope):
    """2 x 264 x 64 + 37 rows: every CTA strides over two or three tiles, the last one partial."""
    n = 2 * ROW_GRID * TILE + 37
    args = dict(n=n, n_out=n_out, k1=k1, k2=k2, t1=1, t2=0, pre_slope=pre_slope, scale=1.3, slope=0.5, accumulate=n_out % 2,
                layout=layout)
    _rowgemm_case(**args, what=' '.join(f'{k}={v}' for k, v in args.items()))


# =====================================================================================================================
# b. ssl_colgemm
# =====================================================================================================================

KN = {1: (16, 13), 2: (32, 30), 4: (64, 37), 8: (128, 127)}     # round_n(k) = N: one k a multiple of 4, one not
CROWS = (1, 64, 65, COL_GRID * TILE, (COL_GRID + 1) * TILE, 1000 * TILE + 17)
GUARD = 64


def _colgemm_run(a, b, pre, k1, k2, slope, scale, mode, ref, want_act):
    """One ssl_colgemm call into NaN-filled partials / out / out_act, each followed by a NaN guard; returns out, out_act."""
    lib, check = _L()
    n = a.shape[0]
    n_part = int(lib.ssl_colgemm_parts(n))
    assert n_part == max(1, min(-(-n // TILE), COL_GRID))
    part, out = _nan(n_part * k1 * k2 + GUARD), _nan(k1 * k2 + GUARD)
    act = _nan(k1 * k2 + GUARD) if want_act else None
    check(lib.ssl_colgemm(a.data_ptr(), a.stride(0), k1, b.data_ptr(), b.stride(0), k2, _p(pre), 0 if pre is None else pre.stride(0),
                          slope, n, part.data_ptr(), scale, mode, _p(ref), out.data_ptr(), _p(act), _s()), 'ssl_colgemm')
    torch.cuda.synchronize()
    assert part[:n_part * k1 * k2].isfinite().all(), 'a partial was not written'
    for buf, name in ((part, 'part'), (out, 'out'), (act, 'out_act')):
        if buf is not None:
            assert buf[-GUARD:].isnan().all(), f'{name} written past its end'
    return out[:k1 * k2].view(k1, k2), None if act is None else act[:k1 * k2].view(k1, k2)


def _colgemm_check(a, b, pre, k1, k2, slope, scale, mode, ref, want_act, group, what):
    """ssl_colgemm against float64, and a second launch bit for bit.  Bound, first order: a partial is a sequential fp32 sum
    over at most R = per * 64 rows, the finalize adds at most n_part partials in sequence (8 lanes, then the lane sums),
    and the staged pre_ref product, * scale, the mode-1 factor and leaky round once each:
        |out - exact| <= (R + n_part + 6) u |scale| sum_r |a_r| |b'_r|."""
    n = a.shape[0]
    slope, scale = _f32(slope), _f32(scale)
    out, act = _colgemm_run(a, b, pre, k1, k2, slope, scale, mode, ref, want_act)
    out2, act2 = _colgemm_run(a, b, pre, k1, k2, slope, scale, mode, ref, want_act)
    assert torch.equal(out, out2) and (act is None or torch.equal(act, act2)), f'{what}: two launches differ'
    bd = b.double() * (1.0 if pre is None else _act_grad(pre, slope).double())
    exact = scale * (a.double().T @ bd)
    absum = abs(scale) * (a.double().abs().T @ bd.abs())
    if mode == 1:
        f = _act_grad(ref, slope).double()
        exact, absum = exact * f, absum * f
    n_tiles = -(-n // TILE)
    n_part = max(1, min(n_tiles, COL_GRID))
    rows_per_cta = min(n, -(-n_tiles // n_part) * TILE)
    bound = (rows_per_cta + n_part + 6) * U * absum + 1e-300
    _within(group, out, exact, bound, what)
    if act is not None:
        _within(group, act, _leaky(exact, slope), bound, what + ' out_act')


@pytest.mark.parametrize('n2', [1, 2, 4, 8])
@pytest.mark.parametrize('n1', [1, 2, 4, 8])
def test_colgemm_every_instantiation_matches_float64(n1, n2):
    """<N1, N2> = <round_n(k1), round_n(k2)>.  n_rows 396 x 64 fills the 396-CTA grid one tile each; 397 x 64 gives per = 2,
    so CTAs 199-395 are empty and write zero partials; 1000 x 64 + 17 gives per = 3 and a partial last tile.  Modes rotate
    (0, 0 with out_act, 1 with ref), layouts rotate (contiguous, row-strided, one float off: the scalar branch), pre_ref is
    on every other case.  Then the same shapes with non-negative inputs: there sum |a b| = the result, the bound is
    relative, (R + n_part + 6) u <= 3.6e-5, and a lost 64-row tile (about 1 / 1000 of an output at the most rows) exceeds
    it."""
    for v in (0, 1):
        k1, k2 = KN[n1][v], KN[n2][v]
        g = _gen('colgemm', n1, n2, v)
        n_max = CROWS[-1]
        A = torch.randn(n_max, k1, generator=g, **F32)
        B = torch.randn(n_max, k2, generator=g, **F32)
        PRE = torch.randn(n_max, k2, generator=g, **F32)
        REF = torch.randn(k1, k2, generator=g, **F32)
        for j, n in enumerate(CROWS):
            layout = LAYOUTS[(j + v) % 3]
            mode, want_act = ((0, False), (0, True), (1, False))[j % 3]
            with_pre = (j + v) % 2 == 0
            slope, scale = (0.2, 0.5)[j % 2], (1.3, 1.0, -0.7)[(j + v) % 3]
            what = f'k1={k1} k2={k2} n_rows={n} layout={layout} mode={mode} out_act={want_act} pre_ref={with_pre} slope={slope} scale={scale}'
            a, b = _in_layout(A[:n], layout), _in_layout(B[:n], layout)
            pre = _in_layout(PRE[:n], layout) if with_pre else None
            _colgemm_check(a, b, pre, k1, k2, slope, scale, mode, REF if mode == 1 else None, want_act, 'b colgemm', what)
            a, b = _in_layout(A[:n].abs(), layout), _in_layout(B[:n].abs(), layout)
            _colgemm_check(a, b, pre, k1, k2, slope, 1.0, 0, None, True, 'b colgemm (non-negative, relative)', what + ' non-negative')


# =====================================================================================================================
# c. ssl_hyper_dropout / ssl_hyper_dropout_dev
# =====================================================================================================================

def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('n,h,keep,stream', [(1, 4, 0.5, 0), (37, 12, 0.3, 5), (1000, 128, 0.5, 3), (4099, 64, 0.7, 2)])
def test_hyper_dropout_matches_the_philox_oracle(n, h, keep, stream):
    """Element (r, 4q + t) is kept when word t of philox(r, q, stream, "HYPR"; seed) gives U + keep >= 1 in float32; the kept
    values are x * 1 * (1 / keep) in float32, the dropped ones x * 0 * (1 / keep) (signed zeros included)."""
    lib, check = _L()
    s = _s()
    seed = 0x1234567890ABCDEF ^ (n * 7919 + stream)                      # both 32-bit halves of the key matter
    keep = _f32(keep)
    g = _gen('dropout', n, h)
    x = torch.randn(n, h, generator=g, **F32)
    mask_np = P.hyper_keep(seed, stream, n, h, keep)
    mask = torch.from_numpy(mask_np.astype(np.float32)).cuda()
    inv = float(np.float32(1.0) / np.float32(keep))
    want = x * mask * inv
    seed_dev = torch.tensor([seed], dtype=torch.int64, device='cuda')
    prev = torch.randn(n, h, generator=g, **F32)

    def run(kind, accumulate):
        out = prev.clone() if accumulate else _nan(n, h)
        if kind == 'host':
            rc = lib.ssl_hyper_dropout(x.data_ptr(), out.data_ptr(), n, h, keep, 1, None, seed, stream, accumulate, s)
        elif kind == 'mask':
            rc = lib.ssl_hyper_dropout(x.data_ptr(), out.data_ptr(), n, h, keep, 2, mask.data_ptr(), 0, 0, accumulate, s)
        else:
            rc = lib.ssl_hyper_dropout_dev(x.data_ptr(), out.data_ptr(), n, h, keep, 1, None, seed_dev.data_ptr(), stream, accumulate, s)
        check(rc, f'ssl_hyper_dropout ({kind})')
        torch.cuda.synchronize()
        return out

    for accumulate in (0, 1):
        expect = want if not accumulate else prev + want
        for kind in ('host', 'mask', 'dev'):
            got = run(kind, accumulate)
            if kind == 'host' and not accumulate:
                assert torch.equal((got != 0).cpu(), torch.from_numpy(mask_np)), 'in-kernel mask differs from oracle/philox.hyper_keep'
            assert torch.equal(_bits(got), _bits(expect)), f'{kind} accumulate={accumulate}: differs from x * mask / keep'
    if n * h >= 4000:
        assert abs(mask_np.mean() - keep) < 0.05, mask_np.mean()
    out = _nan(n, h)
    check(lib.ssl_hyper_dropout(x.data_ptr(), out.data_ptr(), n, h, 1.0, 1, None, seed, stream, 0, s), 'ssl_hyper_dropout keep=1')
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(x)), 'keep = 1 dropped or scaled something'


# =====================================================================================================================
# d. argument checks and empty sides
# =====================================================================================================================

def test_hyper_kernels_reject_bad_arguments():
    lib, _ = _L()
    s = _s()
    n, k = 70, 16
    x = torch.randn(n, 128, **F32)
    m = torch.randn(128 * 128, **F32)
    out = _nan(n, 128)
    part, cout, act = _nan(COL_GRID * 128 * 128), _nan(128 * 128), _nan(128 * 128)
    # ssl_rowgemm: (k1, in2 given, k2, n_out, n_rows, m2 given, in1 given)
    for k1, with_in2, k2, n_out, rows, with_m2, with_in1, what in (
            (3, False, 0, 16, n, False, True, 'k1 = 3'), (129, False, 0, 16, n, False, True, 'k1 = 129'),
            (k, True, 3, 16, n, True, True, 'k2 = 3'), (k, True, 129, 16, n, True, True, 'k2 = 129'),
            (k, False, 0, 3, n, False, True, 'n_out = 3'), (k, False, 0, 129, n, False, True, 'n_out = 129'),
            (k, True, k, 16, n, False, True, 'in2 without m2'), (k, False, 0, 16, n, False, False, 'null in1 with rows'),
            (k, False, 0, 16, -1, False, True, 'n_rows = -1')):
        _rejected(lib.ssl_rowgemm(x.data_ptr() if with_in1 else None, 128, k1, m.data_ptr(), 0, x.data_ptr() if with_in2 else None, 128, k2,
                                  m.data_ptr() if with_m2 else None, 0, None, 0, 1.0, out.data_ptr(), 128, n_out, 1.0, 1.0, 0, rows, s),
                  'ssl_rowgemm ' + what)
    _rejected(lib.ssl_rowgemm(x.data_ptr(), 128, k, m.data_ptr(), 0, None, 0, 0, None, 0, None, 0, 1.0, None, 128, 16, 1.0, 1.0, 0, n, s),
              'ssl_rowgemm null out with rows')
    # ssl_colgemm
    for k1, k2, mode, with_ref, rows, what in ((3, k, 0, False, n, 'k1 = 3'), (129, k, 0, False, n, 'k1 = 129'), (k, 3, 0, False, n, 'k2 = 3'),
                                               (k, 129, 0, False, n, 'k2 = 129'), (k, k, 1, False, n, 'mode 1 without ref'),
                                               (k, k, 2, True, n, 'mode 2'), (k, k, 0, False, -1, 'n_rows = -1')):
        _rejected(lib.ssl_colgemm(x.data_ptr(), 128, k1, x.data_ptr(), 128, k2, None, 0, 0.5, rows, part.data_ptr(), 1.0, mode,
                                  m.data_ptr() if with_ref else None, cout.data_ptr(), act.data_ptr(), s), 'ssl_colgemm ' + what)
    _rejected(lib.ssl_colgemm(None, 128, k, x.data_ptr(), 128, k, None, 0, 0.5, n, part.data_ptr(), 1.0, 0, None, cout.data_ptr(), None, s),
              'ssl_colgemm null in1 with rows')
    # ssl_hyper_dropout / _dev
    for h, keep, mode, with_mask, rows, what in ((6, 0.5, 1, False, n, 'h = 6'), (0, 0.5, 1, False, n, 'h = 0'), (k, 0.0, 1, False, n, 'keep = 0'),
                                                 (k, -0.5, 1, False, n, 'keep < 0'), (k, 1.5, 1, False, n, 'keep > 1'),
                                                 (k, 0.5, 2, False, n, 'mode 2 without mask'), (k, 0.5, 0, True, n, 'mode 0'),
                                                 (k, 0.5, 1, False, -1, 'n = -1')):
        _rejected(lib.ssl_hyper_dropout(x.data_ptr(), out.data_ptr(), rows, h, keep, mode, x.data_ptr() if with_mask else None, 1, 0, 0, s),
                  'ssl_hyper_dropout ' + what)
    _rejected(lib.ssl_hyper_dropout_dev(x.data_ptr(), out.data_ptr(), n, k, 0.5, 1, None, None, 0, 0, s), 'ssl_hyper_dropout_dev without seed_ptr')
    torch.cuda.synchronize()
    for buf, name in ((out, 'out'), (part, 'part'), (cout, 'colgemm out'), (act, 'out_act')):
        assert buf.isnan().all(), f'a rejected call wrote {name}'


def test_hyper_kernels_accept_an_empty_side_with_null_pointers():
    """An empty side (HGNNLayer's second side, any n = 0 slice: data_ptr() == 0): rowgemm and the dropout write nothing,
    colgemm writes out = 0 and out_act = leaky(0) = 0."""
    lib, check = _L()
    s = _s()
    k1, k2 = 40, 32
    m = torch.randn(128 * 128, **F32)
    check(lib.ssl_rowgemm(None, 0, k1, m.data_ptr(), 0, None, 0, k2, m.data_ptr(), 1, None, 0, 0.5, None, 0, k2, 1.0, 0.5, 0, 0, s),
          'ssl_rowgemm n_rows = 0')
    assert int(lib.ssl_colgemm_parts(0)) == 1
    ref = torch.randn(k1, k2, **F32)
    for mode, scale in ((0, 1.3), (1, -0.7)):
        part, out, act = _nan(k1 * k2 + GUARD), _nan(k1 * k2 + GUARD), _nan(k1 * k2 + GUARD)
        check(lib.ssl_colgemm(None, 0, k1, None, 0, k2, None, 0, 0.5, 0, part.data_ptr(), scale, mode, ref.data_ptr() if mode else None,
                              out.data_ptr(), act.data_ptr(), s), 'ssl_colgemm n_rows = 0')
        torch.cuda.synchronize()
        assert torch.equal(out[:k1 * k2], torch.zeros(k1 * k2, **F32)) and torch.equal(act[:k1 * k2], torch.zeros(k1 * k2, **F32)), mode
        assert out[k1 * k2:].isnan().all() and act[k1 * k2:].isnan().all() and part[k1 * k2:].isnan().all()
    seed_dev = torch.tensor([5], dtype=torch.int64, device='cuda')
    for mode in (1, 2):
        check(lib.ssl_hyper_dropout(None, None, 0, 128, 0.5, mode, None, 5, 0, 0, s), f'ssl_hyper_dropout n = 0 mode {mode}')
    check(lib.ssl_hyper_dropout_dev(None, None, 0, 128, 0.5, 1, None, seed_dev.data_ptr(), 0, 1, s), 'ssl_hyper_dropout_dev n = 0')
    torch.cuda.synchronize()
