"""The loss-side kernels of the training step through the C ABI against float64 restatements computed on the device:

a. ssl_rows_normalize: every norm_mode, gathers with duplicates, strided rows, all-zero rows; the K-major tile copy,
   the tf32 hi / lo split and the permuted transposed hi / lo copy checked bit for bit, zeroed padding rows.
b. ssl_softmax_gemm (the FP32-FMA contraction) at all three instantiations, ragged dims and shapes, every n_split
   from 1 to its maximum, colscale on / off, rowsum_part NULL, garbage in C's padding rows.
c. the InfoNCE, DirectAU and BPR epilogues: colliding atomics, NULL outputs, accumulate, strides > dim, B = 1,
   BPR margins around softplus's threshold.
d. ssl_sum / ssl_sumsq / ssl_axpy: n & 3 tails, n = 0, the full reduction grid.
e. Adam: host and on-device bias corrections, peer stores, three steps against float64.
f. uniformity at small batches, including near-antipodal rows.

Every output buffer starts as a NaN sentinel (and slack past the end of an input holds NaN), so an element a kernel
fails to write, or reads past its end, fails the test.  The worst err / scale of each group is printed when the
module finishes (visible with pytest -s)."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

import ssl_test_helpers as H
from oracle import cf_oracle as O

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
U = 2.0 ** -24                       # unit roundoff of fp32
NAN = float('nan')
F32 = dict(device='cuda', dtype=torch.float32)
F32_1E8 = float(np.float32(1e-8))    # the float constants the kernels use
F32_1E12 = float(np.float32(1e-12))

_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
    yield
    if _WORST:
        print('\nworst err/scale: ' + ', '.join(f'{k} {v:.3e}' for k, v in sorted(_WORST.items())))


def _L():
    from sslrec_b200._lib import lib, check
    return lib, check


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _nan(*shape):
    return torch.full(shape, NAN, **F32)


def _ceil64(n):
    return (n + 63) // 64 * 64


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _close(group, got, ref, scale, k, what):
    """|got - ref| <= k * scale elementwise (scale >= 0, broadcastable); NaN fails.  Records max |got - ref| / scale."""
    got, ref = got.double(), ref.double()
    scale = torch.as_tensor(scale, dtype=torch.float64, device=ref.device).expand_as(ref)
    err = (got - ref).abs()
    bad = ~(err <= k * scale)
    assert not bad.any(), (f'{what}: {int(bad.sum())} / {bad.numel()} off, max err {err.max().item():.3e}, '
                           f'max err/scale {(err / scale).max().item():.3e} > {k:.3e}')
    if err.numel():
        r = (err / scale.clamp_min(1e-300)).max().item()
        _WORST[group] = max(_WORST.get(group, 0.0), r)


def _rejected(rc, what):
    from sslrec_b200._lib import lib
    assert rc != 0, f'{what} was accepted'
    assert lib.ssl_last_error(), what


def _unit(x):
    return x / x.norm(dim=1, keepdim=True)


# =====================================================================================================================
# a. ssl_rows_normalize
# =====================================================================================================================

def _tf32_rna(a):
    """cvt.rna.tf32.f32 for finite x: round the 13 dropped mantissa bits to nearest, ties away from zero."""
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _thi_columns(npad):
    """Column of the transposed tf32 copy that row c lands in: 0 2 4 6 1 3 5 7 within every group of 8."""
    c = torch.arange(npad, device='cuda')
    return (c & ~7) | ((c & 7) >> 1) | ((c & 1) << 2)


def _kmajor_rows():
    """Row of its 64-row tile that slot q of the K-major tile copy holds: slot 4*(c%16) + c/16 holds row c."""
    q = torch.arange(64, device='cuda')
    return (q >> 2) + 16 * (q & 3)


def _normalize_ref(rows, mode, alpha):
    rows = rows.double()
    if mode == 1:
        rows = rows + F32_1E8
    ss = (rows * rows).sum(1)
    if mode == 0:
        ri = 1.0 / torch.sqrt(F32_1E8 + ss)
    elif mode == 3:
        ri = torch.ones_like(ss)
    else:
        ri = 1.0 / torch.sqrt(ss).clamp_min(F32_1E12)
    return rows * ri[:, None] * alpha, ri


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('n', [1, 63, 64, 65, 1000])
@pytest.mark.parametrize('dim', [4, 20, 36, 64, 100, 128])
def test_rows_normalize_copies(dim, n, mode):
    lib, check = _L()
    g = _gen('norm', dim, n, mode)
    m = n + 5
    base = (torch.randn(m, 3, dim, generator=g) * 0.7).cuda()          # rows are the middle view of an interleaved table
    zero_rows = sorted({0, n // 2})
    base[zero_rows, 1] = 0.0
    x = base[:, 1]
    idx = torch.randint(0, m, (n,), generator=g)
    idx[::7] = zero_rows[-1]
    if n > 1:
        idx[-1] = idx[0]
    idx = idx.cuda()
    npad = _ceil64(n)
    t_pitch = npad + 4
    cols = _thi_columns(npad)
    kq = _kmajor_rows()
    for alpha in (1.0, LOG2E / 0.2):
        for gidx in (None, idx):
            out, out_t, rinv = _nan(npad, dim), _nan(npad // 64, dim, 64), _nan(n)
            hi, lo, thi, tlo = _nan(npad, dim), _nan(npad, dim), _nan(dim, t_pitch), _nan(dim, t_pitch)
            check(lib.ssl_rows_normalize(x.data_ptr(), 3 * dim, _p(gidx), n, dim, mode, alpha, out.data_ptr(), out_t.data_ptr(),
                                         rinv.data_ptr(), hi.data_ptr(), lo.data_ptr(), thi.data_ptr(), tlo.data_ptr(), t_pitch, _s()),
                  'ssl_rows_normalize')
            torch.cuda.synchronize()
            rows = x[:n] if gidx is None else x[gidx]
            ref, ref_ri = _normalize_ref(rows, mode, alpha)
            what = f'alpha={alpha:.3f} gather={gidx is not None}'
            row_scale = 2.0 ** -23 * ref.abs().amax(1, keepdim=True) + 1e-300      # one ulp of the row's largest entry
            _close('a rows_normalize (ulp)', out[:n], ref, row_scale, 4.0, 'out ' + what)
            _close('a rows_normalize (ulp)', rinv, ref_ri, 2.0 ** -23 * ref_ri, 4.0, 'rinv ' + what)
            assert torch.equal(out[n:], torch.zeros(npad - n, dim, **F32)), 'padding rows of out are not zero'
            assert torch.equal(out_t, out.view(npad // 64, 64, dim)[:, kq, :].transpose(1, 2)), 'K-major tile copy'
            hi_ref = _tf32_rna(out.cpu().numpy())
            lo_ref = _tf32_rna(out.cpu().numpy() - hi_ref)
            assert np.array_equal(hi.cpu().numpy().view(np.uint32), hi_ref.view(np.uint32)), 'tf32 hi'
            assert np.array_equal(lo.cpu().numpy().view(np.uint32), lo_ref.view(np.uint32)), 'tf32 lo'
            for got, src, name in ((thi, hi, 'thi'), (tlo, lo, 'tlo')):
                want = torch.empty(dim, npad, **F32)
                want[:, cols] = src.T
                assert torch.equal(got[:, :npad], want), f'transposed {name} copy'
                assert got[:, npad:].isnan().all(), f'{name} wrote past ceil64(n)'


def test_rows_normalize_rejects_bad_layouts():
    lib, _ = _L()
    n, d = 70, 8
    npad = _ceil64(n)
    x = torch.randn(n, 8, **F32)
    out, hi, lo, thi, tlo = _nan(npad, d), _nan(npad, d), _nan(npad, d), _nan(d, npad + 8), _nan(d, npad + 8)
    s = _s()
    _rejected(lib.ssl_rows_normalize(x.data_ptr(), 8, None, n, 6, 0, 1.0, out.data_ptr(), None, None, None, None, None, None, 0, s),
              'dim 6')
    _rejected(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), None, None, None, None,
                                     thi.data_ptr(), tlo.data_ptr(), npad - 4, s), 't_pitch < ceil64(n)')
    _rejected(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), None, None, None, None,
                                     thi.data_ptr(), tlo.data_ptr(), npad + 2, s), 't_pitch not a multiple of 4')
    _rejected(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), None, None, hi.data_ptr(), None,
                                     None, None, 0, s), 'hi without lo')
    _rejected(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), None, None, None, None,
                                     thi.data_ptr(), None, npad, s), 'thi without tlo')
    torch.cuda.synchronize()
    assert out.isnan().all() and hi.isnan().all() and thi.isnan().all(), 'a rejected call wrote its outputs'


# =====================================================================================================================
# b. ssl_softmax_gemm, the FP32-FMA contraction
# =====================================================================================================================

def _operand(x, alpha, garbage_from=None):
    """F.normalize-like rows (norm_mode 0) scaled by alpha, and their K-major tile copy; rows >= garbage_from of both
    copies are overwritten with 1e3 (the kernel must mask them by index, not rely on their zeros)."""
    lib, check = _L()
    n, d = x.shape
    npad = _ceil64(n)
    out, out_t = _nan(npad, d), _nan(npad // 64, d, 64)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, out.data_ptr(), out_t.data_ptr(), None, None, None,
                                 None, None, 0, _s()), 'ssl_rows_normalize')
    if garbage_from is not None:
        out[garbage_from:] = 1e3
        row = 64 * torch.arange(npad // 64, device='cuda')[:, None] + _kmajor_rows()[None, :]
        out_t.masked_fill_((row >= garbage_from)[:, None, :], 1e3)
    return out, out_t


def _gemm(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum):
    lib, check = _L()
    rs = _nan(n_split, n_r) if with_rowsum else None
    o = _nan(n_split, n_r, d)
    check(lib.ssl_softmax_gemm(R.data_ptr(), n_r, C[0].data_ptr(), C[1].data_ptr(), n_c, d, _p(cs), off, n_split, _p(rs),
                               o.data_ptr(), _s()), 'ssl_softmax_gemm')
    torch.cuda.synchronize()
    return rs, o


def _gemm_ref(A, T, cs, off):
    """rowsum_i = sum_j exp2(a_i . t_j - off) cs_j and O_i = sum_j exp2(...) cs_j t_j in float64, in row chunks."""
    A, T = A.double(), T.double()
    rs, o = torch.empty(A.shape[0], dtype=torch.float64, device='cuda'), torch.empty(A.shape, dtype=torch.float64, device='cuda')
    for r in range(0, A.shape[0], 4096):
        E = torch.exp2(A[r:r + 4096] @ T.T - off)
        if cs is not None:
            E = E * cs.double()
        rs[r:r + 4096], o[r:r + 4096] = E.sum(1), E @ T
    return rs, o


@pytest.mark.parametrize('n_r,n_c', [(1, 1), (127, 63), (129, 65), (300, 777), (4097, 9000)])
@pytest.mark.parametrize('dim', [4, 20, 32, 36, 48, 64, 68, 124, 128])
def test_softmax_gemm_fp32_matches_float64(dim, n_r, n_c):
    from sslrec_b200 import engine
    lib, _ = _L()
    g = _gen('gemm', dim, n_r, n_c)
    off = LOG2E / 0.2
    R, _ = _operand(torch.randn(n_r, dim, generator=g).cuda(), off)
    C = _operand(torch.randn(n_c, dim, generator=g).cuda(), 1.0, garbage_from=n_c)
    cs = (torch.rand(_ceil64(n_c), generator=g) + 0.5).cuda()
    tiles = (n_c + 63) // 64
    pick = engine.choose_split((n_r + 127) // 128, tiles, slots=2 * engine.NUM_SM)
    splits = sorted({s for s in (1, 2, tiles, pick) if s <= tiles})
    refs = {on: _gemm_ref(R[:n_r], C[0][:n_c], cs[:n_c] if on else None, off) for on in (False, True)}
    for n_split in splits:
        # a partial is a sequential fp32 sum over the L columns of its split, whose rounding error grows like sqrt(L):
        # 2e-6 of the largest entry, and 1.5 sqrt(L / 1024) times that for long splits (4.9e-6 seen at L = 9024, d = 4)
        L = 64 * -(-tiles // n_split)
        k = 2e-6 * max(1.0, 1.5 * (L / 1024) ** 0.5)
        for on in (False, True):
            rs, o = _gemm(R, n_r, C, n_c, dim, cs if on else None, off, n_split, True)
            ref_rs, ref_o = refs[on]
            what = f'n_split={n_split} colscale={on}'
            _close('b softmax_gemm', rs.sum(0), ref_rs, ref_rs.abs().max(), k, 'rowsum ' + what)
            _close('b softmax_gemm', o.sum(0), ref_o, ref_o.abs().max(), k, 'O ' + what)
    # rowsum_part = NULL changes nothing else, and a second launch is bit-identical
    n_split = splits[-1]
    rs1, o1 = _gemm(R, n_r, C, n_c, dim, cs, off, n_split, True)
    _, o2 = _gemm(R, n_r, C, n_c, dim, cs, off, n_split, False)
    rs3, o3 = _gemm(R, n_r, C, n_c, dim, cs, off, n_split, True)
    assert torch.equal(o1, o2), 'rowsum_part = NULL changed O'
    assert torch.equal(rs1, rs3) and torch.equal(o1, o3), 'two launches differ'
    # rejections
    o = _nan(tiles + 1, n_r, dim)
    s = _s()
    _rejected(lib.ssl_softmax_gemm(R.data_ptr(), n_r, C[0].data_ptr(), C[1].data_ptr(), n_c, dim, None, off, tiles + 1, None,
                                   o.data_ptr(), s), 'n_split > tiles')
    for k in range(3):
        ptrs = [R.data_ptr(), C[0].data_ptr(), C[1].data_ptr()]
        ptrs[k] += 4
        _rejected(lib.ssl_softmax_gemm(ptrs[0], n_r, ptrs[1], ptrs[2], n_c, dim, None, off, 1, None, o.data_ptr(), s),
                  f'unaligned operand {k}')
    torch.cuda.synchronize()
    assert o.isnan().all(), 'a rejected call wrote its outputs'


# =====================================================================================================================
# c. epilogues
# =====================================================================================================================

@pytest.mark.parametrize('dim', [4, 20, 64, 128])
@pytest.mark.parametrize('B', [1, 7, 257])
@pytest.mark.parametrize('n_split', [1, 3, 33])
def test_nce_and_lse_finalize(n_split, B, dim):
    lib, check = _L()
    g = _gen('fin', n_split, B, dim)
    tau = float(np.float32(0.2))
    rsp = (torch.rand(n_split, B, generator=g) + 0.1).cuda()
    op = torch.randn(n_split, B, dim, generator=g).cuda()
    a_hat = (_unit(torch.randn(B, dim, generator=g)) * (LOG2E / tau)).float().cuda()
    p_hat = _unit(torch.randn(B, dim, generator=g)).float().cuda()
    s = _s()
    for eps in (0.0, 0.25):
        eps = float(np.float32(eps))
        ref_rs = rsp.double().sum(0) + eps
        ref_ob = op.double().sum(0) / ref_rs[:, None]
        rs_scale = rsp.double().sum(0) + eps
        ob_scale = op.double().abs().sum(0) / ref_rs[:, None]
        ap = (a_hat.double() * p_hat.double()).sum(1) * LN2
        ap_abs = (a_hat.double() * p_hat.double()).abs().sum(1) * LN2
        for lse in (False, True):
            rowsum, obar, loss_b = _nan(B), _nan(B, dim), _nan(B)
            if lse:
                check(lib.ssl_lse_finalize(rsp.data_ptr(), op.data_ptr(), n_split, B, dim, eps, rowsum.data_ptr(), obar.data_ptr(),
                                           loss_b.data_ptr(), s), 'ssl_lse_finalize')
                ref_loss = torch.log(ref_rs)
                loss_scale = ref_rs.log().abs() + 1.0
            else:
                check(lib.ssl_nce_finalize(rsp.data_ptr(), op.data_ptr(), n_split, B, dim, a_hat.data_ptr(), p_hat.data_ptr(), tau, eps,
                                           rowsum.data_ptr(), obar.data_ptr(), loss_b.data_ptr(), s), 'ssl_nce_finalize')
                ref_loss = -ap + 1.0 / tau + torch.log(ref_rs)
                loss_scale = ap_abs + 1.0 / tau + ref_rs.log().abs() + 1.0
            torch.cuda.synchronize()
            what = f'{"lse" if lse else "nce"} eps={eps}'
            _close('c finalize', rowsum, ref_rs, rs_scale * U, n_split + 2, 'rowsum ' + what)
            _close('c finalize', obar, ref_ob, ob_scale * U, 2 * n_split + 6, 'obar ' + what)
            _close('c finalize', loss_b, ref_loss, loss_scale * U, n_split + 24, 'loss ' + what)


@pytest.mark.parametrize('B', [1, 7, 257, 1000])
def test_nce_colscale(B):
    lib, check = _L()
    g = _gen('colscale', B)
    rowsum = (torch.rand(B, generator=g) * 50 + 0.5).cuda()
    gs = torch.tensor([0.37], **F32)
    scale = float(np.float32(1.7))
    for gscale in (None, gs):
        cs = _nan(B + 4)
        check(lib.ssl_nce_colscale(rowsum.data_ptr(), B, _p(gscale), scale, cs.data_ptr(), _s()), 'ssl_nce_colscale')
        torch.cuda.synchronize()
        ref = scale * (1.0 if gscale is None else gs.double().item()) * LN2 / rowsum.double()
        _close('c epilogue rows', cs[:B], ref, ref.abs() * U, 6, f'colscale gscale={gscale is not None}')
        assert cs[B:].isnan().all(), 'colscale wrote past batch'


def _dup_idx(g, B, n_rows):
    """Gather indices where row 5 takes every third slot (>= 64 repeats at B = 257), so the atomics collide."""
    if B == 1:
        return torch.tensor([3])
    if B == 7:
        return torch.tensor([2, 2, 2, 0, 2, 1, 2])
    idx = torch.randint(0, n_rows, (B,), generator=g)
    idx[::3] = 5
    return idx


def _prefilled(g, n_rows, dim, stride, fill_random=True):
    """A gradient table [n_rows, stride]: used columns random (or NaN), the columns past dim NaN."""
    buf = _nan(n_rows, stride)
    if fill_random:
        buf[:, :dim] = torch.randn(n_rows, dim, generator=g).cuda()
    return buf


def _index_add(n_rows, idx, rows):
    return torch.zeros(n_rows, rows.shape[1], dtype=torch.float64, device='cuda').index_add_(0, idx, rows)


@pytest.mark.parametrize('dim', [4, 20, 64, 128])
@pytest.mark.parametrize('B', [1, 7, 257])
def test_nce_bwd_rows_colliding_rows(B, dim):
    lib, check = _L()
    g = _gen('bwd_rows', B, dim)
    tau = float(np.float32(0.2))
    n_rows, stride = 40, dim + 3
    a_hat = (_unit(torch.randn(B, dim, generator=g)) * (LOG2E / tau)).float().cuda()
    p_hat = _unit(torch.randn(B, dim, generator=g)).float().cuda()
    obar = (torch.randn(B, dim, generator=g) * 0.1).cuda()
    r1, r2 = (torch.rand(B, generator=g) + 0.5).cuda(), (torch.rand(B, generator=g) + 0.5).cuda()
    idx = _dup_idx(g, B, n_rows).cuda()
    reps = int(torch.bincount(idx).max())
    gs = torch.tensor([0.8], **F32)
    scale = float(np.float32(1.3))
    for which, gscale in (('g1', None), ('g2', gs), ('both', gs)):
        g1 = _prefilled(g, n_rows, dim, stride) if which in ('g1', 'both') else None
        g2 = _prefilled(g, n_rows, dim, stride) if which in ('g2', 'both') else None
        pre1, pre2 = [None if t is None else t[:, :dim].double() for t in (g1, g2)]
        check(lib.ssl_nce_bwd_rows(a_hat.data_ptr(), p_hat.data_ptr(), obar.data_ptr(), r1.data_ptr(), r2.data_ptr(), idx.data_ptr(), B, dim,
                                   tau, _p(gscale), scale, _p(g1), stride, _p(g2), stride, _s()), 'ssl_nce_bwd_rows')
        torch.cuda.synchronize()
        gg = scale * (1.0 if gscale is None else gs.double().item()) / tau
        a = a_hat.double() * (float(np.float32(tau * LN2)))
        p, ob = p_hat.double(), obar.double()
        if g1 is not None:
            d = gg * (ob - p)
            proj = (a * d).sum(1, keepdim=True)
            c = r1.double()[:, None] * (d - a * proj)
            c_abs = r1.double()[:, None] * (d.abs() + a.abs() * (a * d).abs().sum(1, keepdim=True))
            _close('c epilogue rows', g1[:, :dim], pre1 + _index_add(n_rows, idx, c), pre1.abs() + _index_add(n_rows, idx, c_abs),
                   (reps + 24) * U, f'g1 ({which})')
            assert g1[:, dim:].isnan().all(), 'g1 written past dim'
        if g2 is not None:
            d = -gg * a
            proj = (p * d).sum(1, keepdim=True)
            c = r2.double()[:, None] * (d - p * proj)
            c_abs = r2.double()[:, None] * (d.abs() + p.abs() * (p * d).abs().sum(1, keepdim=True))
            _close('c epilogue rows', g2[:, :dim], pre2 + _index_add(n_rows, idx, c), pre2.abs() + _index_add(n_rows, idx, c_abs),
                   (reps + 24) * U, f'g2 ({which})')
            assert g2[:, dim:].isnan().all(), 'g2 written past dim'


@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('dim', [4, 20, 64, 128])
@pytest.mark.parametrize('n_split', [1, 3])
def test_nce_bwd_table(n_split, dim, accumulate):
    lib, check = _L()
    g = _gen('bwd_table', n_split, dim, accumulate)
    n, stride = 300, dim + 5
    dt = torch.randn(n_split, n, dim, generator=g).cuda()
    t_hat = _unit(torch.randn(n, dim, generator=g)).float().cuda()
    rinv = (torch.rand(n, generator=g) + 0.5).cuda()
    out = _prefilled(g, n, dim, stride, fill_random=bool(accumulate))      # accumulate = 0: every used element starts NaN
    pre = out[:, :dim].double().nan_to_num(0.0) if accumulate else 0.0
    check(lib.ssl_nce_bwd_table(dt.data_ptr(), n_split, t_hat.data_ptr(), rinv.data_ptr(), n, dim, out.data_ptr(), stride, accumulate,
                                _s()), 'ssl_nce_bwd_table')
    torch.cuda.synchronize()
    d, t, r = dt.double().sum(0), t_hat.double(), rinv.double()[:, None]
    ref = pre + r * (d - t * (t * d).sum(1, keepdim=True))
    scale = (pre.abs() if accumulate else 0.0) + r * (dt.double().abs().sum(0) + t.abs() * (t.abs() * dt.double().abs().sum(0)).sum(1, keepdim=True))
    _close('c epilogue rows', out[:, :dim], ref, scale, (n_split + 24) * U, f'g_table accumulate={accumulate}')
    assert out[:, dim:].isnan().all(), 'g_table written past dim'


@pytest.mark.parametrize('dim', [4, 20, 64, 128])
@pytest.mark.parametrize('B', [1, 7, 257])
def test_uniform_finalize_and_align_fwd(B, dim):
    lib, check = _L()
    g = _gen('ufin', B, dim)
    off = float(np.float32(4.0 * LOG2E))
    xhat = _unit(torch.randn(B, dim, generator=g)).float().cuda()
    yhat = _unit(torch.randn(B, dim, generator=g)).float().cuda()
    yhat[B // 2] = xhat[B // 2]                                      # a zero alignment distance
    r_scaled = xhat * off
    s = _s()
    for n_split in (1, 3):
        rsp = (torch.rand(n_split, B, generator=g) + 0.5).cuda()
        op = torch.randn(n_split, B, dim, generator=g).cuda()
        pair_sum, w = _nan(B), _nan(B, dim)
        check(lib.ssl_uniform_finalize(rsp.data_ptr(), op.data_ptr(), n_split, B, dim, r_scaled.data_ptr(), xhat.data_ptr(), off,
                                       pair_sum.data_ptr(), w.data_ptr(), s), 'ssl_uniform_finalize')
        torch.cuda.synchronize()
        e_ii = torch.exp2((r_scaled.double() * xhat.double()).sum(1) - off)
        _close('c epilogue rows', pair_sum, rsp.double().sum(0) - e_ii, rsp.double().sum(0) + 1.0, (n_split + 48) * U, 'pair_sum')
        _close('c epilogue rows', w, op.double().sum(0) - e_ii[:, None] * xhat.double(),
               op.double().abs().sum(0) + xhat.double().abs(), (n_split + 48) * U, 'w')
    loss_b = _nan(B + 4)
    check(lib.ssl_align_fwd(xhat.data_ptr(), yhat.data_ptr(), B, dim, loss_b.data_ptr(), s), 'ssl_align_fwd')
    torch.cuda.synchronize()
    diff = xhat.double() - yhat.double()
    ref = (diff * diff).sum(1)
    _close('c epilogue rows', loss_b[:B], ref, ref + 1e-300, 16 * U, 'align loss_b')
    assert loss_b[B:].isnan().all()


@pytest.mark.parametrize('dim', [4, 20, 64, 128])
@pytest.mark.parametrize('B', [1, 257])
def test_unit_rows_bwd(B, dim):
    lib, check = _L()
    g = _gen('unit_bwd', B, dim)
    xhat = _unit(torch.randn(B, dim, generator=g)).float().cuda()
    rinv = (torch.rand(B, generator=g) + 0.5).cuda()
    d1, d2 = torch.randn(B, dim, generator=g).cuda(), torch.randn(B, dim, generator=g).cuda()
    c1, c2 = float(np.float32(0.7)), float(np.float32(-1.9))
    gs = torch.tensor([1.25], **F32)
    scale = float(np.float32(0.5))
    n_rows = 40
    for with_d2, with_idx, gscale in ((False, False, None), (True, False, gs), (False, True, gs), (True, True, None)):
        idx = _dup_idx(g, B, n_rows).cuda() if with_idx else None
        rows = n_rows if with_idx else B
        stride = dim + 2
        out = _prefilled(g, rows, dim, stride)
        pre = out[:, :dim].double()
        check(lib.ssl_unit_rows_bwd(xhat.data_ptr(), rinv.data_ptr(), _p(idx), B, dim, d1.data_ptr(), c1, _p(d2 if with_d2 else None), c2,
                                    _p(gscale), scale, out.data_ptr(), stride, _s()), 'ssl_unit_rows_bwd')
        torch.cuda.synchronize()
        gg = scale * (1.0 if gscale is None else gs.double().item())
        d = gg * c1 * d1.double() + (gg * c2 * d2.double() if with_d2 else 0.0)
        d_abs = abs(gg * c1) * d1.double().abs() + (abs(gg * c2) * d2.double().abs() if with_d2 else 0.0)
        x = xhat.double()
        c = rinv.double()[:, None] * (d - x * (x * d).sum(1, keepdim=True))
        c_abs = rinv.double()[:, None] * (d_abs + x.abs() * (x.abs() * d_abs).sum(1, keepdim=True))
        ii = idx if with_idx else torch.arange(B, device='cuda')
        reps = int(torch.bincount(ii).max())
        _close('c epilogue rows', out[:, :dim], pre + _index_add(rows, ii, c), pre.abs() + _index_add(rows, ii, c_abs), (reps + 24) * U,
               f'unit_rows_bwd d2={with_d2} idx={with_idx}')
        assert out[:, dim:].isnan().all(), 'written past dim'


MARGINS = [-100.0, -20.0, 0.0, 19.9, 20.0, 20.1, 100.0]


@pytest.mark.parametrize('dim', [4, 20, 64, 128])
def test_bpr_forward_backward(dim):
    """Margins z = a.n - a.p set exactly (anchor e_0, positive 0, negative z e_0) around softplus's threshold of 20 and far
    past it, plus random rows with repeated users / items (one row has pos == neg); tables and gradients are strided views."""
    lib, check = _L()
    g = _gen('bpr', dim)
    nu, ni, n_rand = 50, 70, 250
    users = _nan(nu, 2, dim)
    items = _nan(ni, 3, dim)
    users[:, 0] = (torch.randn(nu, dim, generator=g) * 0.3).cuda()
    items[:, 2] = (torch.randn(ni, dim, generator=g) * 0.3).cuda()
    users[0, 0] = 0.0
    users[0, 0, 0] = 1.0
    items[0, 2] = 0.0
    for k, z in enumerate(MARGINS):
        items[1 + k, 2] = 0.0
        items[1 + k, 2, 0] = z
    ancs = torch.cat([torch.zeros(len(MARGINS), dtype=torch.int64), torch.randint(1, nu, (n_rand,), generator=g)])
    poss = torch.cat([torch.zeros(len(MARGINS), dtype=torch.int64), torch.randint(8, ni, (n_rand,), generator=g)])
    negs = torch.cat([torch.arange(1, 1 + len(MARGINS)), torch.randint(8, ni, (n_rand,), generator=g)])
    negs[-1] = poss[-1]
    ancs[::5] = 3                                          # repeated users
    ancs[:len(MARGINS)] = 0
    ancs, poss, negs = ancs.cuda(), poss.cuda(), negs.cuda()
    B = ancs.numel()
    U_, I_ = users[:, 0], items[:, 2]
    loss_b, coef_b = _nan(B), _nan(B)
    s = _s()
    check(lib.ssl_bpr_fwd(U_.data_ptr(), 2 * dim, I_.data_ptr(), 3 * dim, ancs.data_ptr(), poss.data_ptr(), negs.data_ptr(), B, dim,
                          loss_b.data_ptr(), coef_b.data_ptr(), s), 'ssl_bpr_fwd')
    torch.cuda.synchronize()
    a, p, n = U_.double()[ancs], I_.double()[poss], I_.double()[negs]
    z = (a * n).sum(1) - (a * p).sum(1)
    assert torch.equal(z[:len(MARGINS)].float().cpu(), torch.tensor(MARGINS, dtype=torch.float32))
    zs = (a * n).abs().sum(1) + (a * p).abs().sum(1)
    ref_loss = torch.where(z > 20, z, torch.log1p(torch.exp(z)))
    ref_coef = torch.sigmoid(z)
    _close('c bpr', loss_b, ref_loss, zs + ref_loss.abs() + 1e-300, 24 * U, 'bpr loss')
    _close('c bpr', coef_b, ref_coef, zs + ref_coef + 1e-300, 24 * U, 'bpr coef')
    gs = torch.tensor([0.6], **F32)
    scale = float(np.float32(1.0 / B))
    for gscale in (None, gs):
        gu, gi = _nan(nu, 2, dim), _nan(ni, 3, dim)
        gu[:, 0] = torch.randn(nu, dim, generator=g).cuda()
        gi[:, 2] = torch.randn(ni, dim, generator=g).cuda()
        pre_u, pre_i = gu[:, 0].double(), gi[:, 2].double()
        check(lib.ssl_bpr_bwd(U_.data_ptr(), 2 * dim, I_.data_ptr(), 3 * dim, ancs.data_ptr(), poss.data_ptr(), negs.data_ptr(), B, dim,
                              coef_b.data_ptr(), _p(gscale), scale, gu[:, 0].data_ptr(), 2 * dim, gi[:, 2].data_ptr(), 3 * dim, s),
              'ssl_bpr_bwd')
        torch.cuda.synchronize()
        gg = (scale * (1.0 if gscale is None else gs.double().item()) * coef_b.double())[:, None]
        ref_u = pre_u + _index_add(nu, ancs, gg * (n - p))
        ref_i = pre_i + _index_add(ni, poss, -gg * a) + _index_add(ni, negs, gg * a)
        sc_u = pre_u.abs() + _index_add(nu, ancs, gg.abs() * (n.abs() + p.abs()))
        sc_i = pre_i.abs() + _index_add(ni, poss, gg.abs() * a.abs()) + _index_add(ni, negs, gg.abs() * a.abs())
        reps_u = int(torch.bincount(ancs).max())
        reps_i = int((torch.bincount(poss, minlength=ni) + torch.bincount(negs, minlength=ni)).max())
        _close('c bpr', gu[:, 0], ref_u, sc_u, (reps_u + 8) * U, f'bpr g_users gscale={gscale is not None}')
        _close('c bpr', gi[:, 2], ref_i, sc_i, (reps_i + 8) * U, f'bpr g_items gscale={gscale is not None}')
        assert gu[:, 1].isnan().all() and gi[:, :2].isnan().all(), 'bpr_bwd wrote outside its strided view'


# =====================================================================================================================
# d. reductions and axpy
# =====================================================================================================================

@pytest.mark.parametrize('n', [0, 1, 2, 3, 4, 5, 1023, 606208, 606209, 606211, 10000003])
def test_sum_and_sumsq(n):
    """606 208 = 592 blocks x 256 threads x 4: one full pass of the grid-stride loop.  The slack past n holds NaN."""
    lib, check = _L()
    g = torch.Generator(device='cuda').manual_seed(n + 1)
    buf = _nan(n + 8)
    buf[:n] = torch.randn(n, generator=g, **F32) + 0.5
    x = buf[:n]
    alpha = float(np.float32(1.0 / 3.0))
    chain = min(n, 128) + 2            # no element passes through more than ~75 fp32 additions in the two-stage tree
    for sq in (False, True):
        outs = []
        for _ in range(2):
            out = _nan(1)
            if sq:
                check(lib.ssl_sumsq(buf.data_ptr(), n, out.data_ptr(), _s()), 'ssl_sumsq')
            else:
                check(lib.ssl_sum(buf.data_ptr(), n, alpha, out.data_ptr(), _s()), 'ssl_sum')
            torch.cuda.synchronize()
            outs.append(out)
        xd = x.double()
        ref = (xd * xd).sum() if sq else alpha * xd.sum()
        scale = (xd * xd).sum() if sq else alpha * xd.abs().sum()
        _close('d reductions', outs[0], ref.reshape(1), scale + 1e-300, chain * U, f'{"sumsq" if sq else "sum"} n={n}')
        assert torch.equal(outs[0], outs[1]), 'two runs differ'
    _rejected(lib.ssl_sum(buf.data_ptr() + 4, n, 1.0, buf.data_ptr(), _s()), 'ssl_sum at a 4-byte offset')
    _rejected(lib.ssl_sumsq(buf.data_ptr() + 4, n, buf.data_ptr(), _s()), 'ssl_sumsq at a 4-byte offset')


@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 6, 7, 8, 9, 1027])
def test_axpy(n):
    lib, check = _L()
    g = torch.Generator().manual_seed(n)
    xb, gs = _nan(n + 8), torch.tensor([0.6], **F32)
    xb[:n] = torch.randn(n, generator=g).cuda()
    alpha = float(np.float32(-0.7))
    for gscale in (None, gs):
        yb = torch.full((n + 8,), 5.0, **F32)
        yb[:n] = torch.randn(n, generator=g).cuda()
        y0 = yb[:n].double().clone()
        check(lib.ssl_axpy(xb.data_ptr(), yb.data_ptr(), n, _p(gscale), alpha, _s()), 'ssl_axpy')
        torch.cuda.synchronize()
        a = torch.tensor(alpha, dtype=torch.float32) * (1.0 if gscale is None else gs.cpu()[0])
        ref = y0 + float(a) * xb[:n].double()
        _close('d axpy (ulp)', yb[:n], ref, 2.0 ** -23 * ref.abs() + 1e-300, 1.0, f'axpy gscale={gscale is not None}')
        assert torch.equal(yb[n:], torch.full((8,), 5.0, **F32)), 'axpy wrote past n'


# =====================================================================================================================
# e. Adam
# =====================================================================================================================

LR, BETAS, EPS, WD = 1e-3, (0.9, 0.999), 1e-8, 0.01


def _peer_array(peers):
    return (ctypes.c_void_p * len(peers))(*[t.data_ptr() for t in peers])


@pytest.mark.parametrize('step', [1, 1000])
@pytest.mark.parametrize('n', [1001, 1002, 1003])
def test_adam_device_step_equals_host_step(n, step):
    """ssl_adam_step_dev (bias corrections from a device step count, the CUDA-graph path) against ssl_adam_step_peers at the
    same step: both evaluate the corrections in double and round them to float, so p, m and v agree bit for bit.  Two
    stand-in peer buffers receive p, the n & 3 tail included."""
    lib, check = _L()
    g = torch.Generator().manual_seed(n * 7 + step)
    p0, grad = torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()
    m0, v0 = (torch.randn(n, generator=g) * 0.1).cuda(), (torch.rand(n, generator=g) * 0.01).cuda()
    res = {}
    for mode in ('host', 'host_peers', 'dev'):
        p, m, v = p0.clone(), m0.clone(), v0.clone()
        peers = [_nan(n), _nan(n)] if mode != 'host' else []
        if mode == 'dev':
            step_dev, scratch = torch.tensor([step], dtype=torch.int64, device='cuda'), _nan(2)
            check(lib.ssl_adam_step_dev(p.data_ptr(), _peer_array(peers), 2, grad.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                        step_dev.data_ptr(), scratch.data_ptr(), LR, BETAS[0], BETAS[1], EPS, WD, _s()), 'ssl_adam_step_dev')
        elif mode == 'host_peers':
            check(lib.ssl_adam_step_peers(p.data_ptr(), _peer_array(peers), 2, grad.data_ptr(), m.data_ptr(), v.data_ptr(), n, step,
                                          LR, BETAS[0], BETAS[1], EPS, WD, _s()), 'ssl_adam_step_peers')
        else:
            check(lib.ssl_adam_step(p.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), n, step, LR, BETAS[0], BETAS[1], EPS, WD,
                                    _s()), 'ssl_adam_step')
        torch.cuda.synchronize()
        for q, peer in enumerate(peers):
            assert torch.equal(peer, p), f'{mode}: peer {q} differs from p at {(peer != p).nonzero().flatten()[:8].tolist()}'
        res[mode] = (p, m, v)
    for mode in ('host_peers', 'dev'):
        for a, b, name in zip(res['host'], res[mode], 'pmv'):
            assert torch.equal(a, b), f'{mode} {name} differs from the host step: max |d| {(a - b).abs().max().item():.3e}'


@pytest.mark.parametrize('n', [1001, 1003])
def test_adam_three_steps_match_float64(n):
    """Three steps against a float64 restatement of torch.optim.Adam (L2 weight decay added to the gradient)."""
    lib, check = _L()
    g = torch.Generator().manual_seed(n)
    p = torch.randn(n, generator=g).cuda()
    m, v = torch.zeros(n, **F32), torch.zeros(n, **F32)
    rp, rm, rv = p.double(), torch.zeros(n, dtype=torch.float64, device='cuda'), torch.zeros(n, dtype=torch.float64, device='cuda')
    am, ap = torch.zeros_like(rm), rp.abs()
    b1, b2 = BETAS
    for step in (1, 2, 3):
        grad = torch.randn(n, generator=g).cuda()
        check(lib.ssl_adam_step(p.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), n, step, LR, b1, b2, EPS, WD, _s()),
              'ssl_adam_step')
        ge = grad.double() + WD * rp
        rm = b1 * rm + (1 - b1) * ge
        rv = b2 * rv + (1 - b2) * ge * ge
        am = b1 * am + (1 - b1) * ge.abs()
        upd = LR / (1 - b1 ** step) * rm / (rv.sqrt() / (1 - b2 ** step) ** 0.5 + EPS)
        rp = rp - upd
        ap = ap + upd.abs()
    torch.cuda.synchronize()
    _close('e adam', m, rm, am, 16 * U, 'exp_avg')
    _close('e adam', v, rv, rv, 16 * U, 'exp_avg_sq')
    _close('e adam', p, rp, ap, 16 * U, 'param')


# =====================================================================================================================
# f. uniformity at small batches
# =====================================================================================================================

def _uniformity_rows(B, dim, kind, g):
    x = torch.randn(B, dim, generator=g) * 0.3
    if kind == 'antipodal':                      # rows in pairs pointing in nearly opposite directions
        for k in range(0, B - 1, 2):
            x[k + 1] = -x[k] + 0.05 * torch.randn(dim, generator=g)
    elif kind == 'duplicated':                   # the same row twice in a batch: pair distance 0
        x[1] = x[0]
        if B >= 8:
            x[B - 1] = x[2]
    return x


@pytest.mark.parametrize('kind', ['random', 'antipodal', 'duplicated'])
@pytest.mark.parametrize('dim', [32, 64, 128])
@pytest.mark.parametrize('B', [2, 3, 4, 8, 64, 255, 256])
def test_uniformity_small_batches(B, dim, kind):
    """log mean_{i<j} exp(-2 |x^_i - x^_j|^2) and its gradient against the float64 oracle.  Below 256 rows the pair sums come
    from the difference vectors; the contraction's rowsum_i - e_ii lost most of its digits at B = 2-3 and for
    near-antipodal rows, where the off-diagonal sum is small next to e_ii = 1."""
    from sslrec_b200 import loss_utils as LU
    x = _uniformity_rows(B, dim, kind, _gen('unif', B, dim, kind))
    xs = x.clone().cuda().requires_grad_(True)
    got = LU.uniformity(xs)
    got.backward()
    ref_x = x.double().clone().requires_grad_(True)
    want = O.uniformity(ref_x)
    want.backward()
    err = abs(got.item() - want.item())
    _WORST['f uniformity'] = max(_WORST.get('f uniformity', 0.0), err / max(1.0, abs(want.item())))
    assert err <= 1e-5 * max(1.0, abs(want.item())), (got.item(), want.item())
    gmax = ref_x.grad.abs().max().item()
    # all rows equal (B = 2, duplicated): the exact gradient is 0 and ours is the rounding residue of projecting x^_i off itself
    atol = 2e-5 * gmax if gmax > 0 else 1e-5
    H.close(xs.grad, ref_x.grad, 2e-4, atol, 'grad')
    if gmax > 0:
        _WORST['f uniformity grad'] = max(_WORST.get('f uniformity grad', 0.0), (xs.grad.cpu().double() - ref_x.grad).abs().max().item() / gmax)
