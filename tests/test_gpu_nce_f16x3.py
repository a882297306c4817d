"""The 3xFP16 tensor-core InfoNCE contraction (ssl_softmax_gemm_f16x3[_live]) and its operand writer
(ssl_rows_normalize_f16x3) through the C ABI: against float64 at the bench shapes and at ragged ones, n_split from 1 to
its maximum, d = 32 and 64, colscale at the backward role's magnitude, tau = 0.1 and 0.2, special operands (exact zeros,
entries below 2^-14, entries at the bound), both live roles, relaunch bit-identity, agreement with 3xTF32, and rejected
arguments."""
import numpy as np
import pytest
import torch

import ssl_test_helpers as H
from test_host_f16x3_split import f16x3_split

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
F32 = dict(device='cuda', dtype=torch.float32)
F16 = dict(device='cuda', dtype=torch.float16)
LIVE_ROWS, LIVE_COLS = 1, 2


def _s():
    return torch.cuda.current_stream().cuda_stream


def _operand(x, alpha, norm_mode=0):
    """Rows of x normalised and scaled by alpha: (fp32 rows, fp16 hi, fp16 lo, rinv)."""
    from sslrec_b200._lib import lib, check
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, hi, lo, rinv = torch.empty(npad, d, **F32), torch.empty(npad, d, **F16), torch.empty(npad, d, **F16), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize_f16x3(x.data_ptr(), d, None, n, d, norm_mode, alpha, hat.data_ptr(), rinv.data_ptr(), hi.data_ptr(),
                                       lo.data_ptr(), _s()), 'ssl_rows_normalize_f16x3')
    return hat, hi, lo, rinv


def _contract(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum=True, live=None, role=0):
    from sslrec_b200._lib import lib, check
    rs = torch.zeros(n_split, n_r, **F32) if with_rowsum else None
    o = torch.zeros(n_split, n_r, d, **F32)
    args = (R[1].data_ptr(), R[2].data_ptr(), n_r, C[1].data_ptr(), C[2].data_ptr(), n_c, d, None if cs is None else cs.data_ptr(), off,
            n_split, None if rs is None else rs.data_ptr(), o.data_ptr())
    if live is None:
        check(lib.ssl_softmax_gemm_f16x3(*args, _s()), 'ssl_softmax_gemm_f16x3')
    else:
        check(lib.ssl_softmax_gemm_f16x3_live(*args, live.data_ptr(), role, _s()), 'ssl_softmax_gemm_f16x3_live')
    torch.cuda.synchronize()
    return rs, o


def _reference(A, T, cs, off):
    """rowsum_i = sum_j exp2(a_i . t_j - off) cs_j and O_i = sum_j exp2(...) cs_j t_j in float64, in row chunks."""
    A, T = A.double(), T.double()
    rs, o = torch.empty(A.shape[0], dtype=torch.float64, device='cuda'), torch.empty(A.shape, dtype=torch.float64, device='cuda')
    for r in range(0, A.shape[0], 4096):
        E = torch.exp2(A[r:r + 4096] @ T.T - off)
        if cs is not None:
            E = E * cs.double()
        rs[r:r + 4096], o[r:r + 4096] = E.sum(1), E @ T
    return rs, o


def _colscale(n, mag, g):
    """colscale at magnitude ``mag`` with a max / min ratio of 2^12 (log-uniform), as g ln2 / rowsum is in the backward."""
    return (mag * torch.exp2(-12.0 * torch.rand(n, generator=g, dtype=torch.float64))).float().cuda()


def _check(rs, o, ref_rs, ref_o):
    if rs is not None:
        H.close(rs.sum(0), ref_rs, 2e-4, 1e-5 * ref_rs.abs().max().item(), 'rowsum')
    H.close(o.sum(0), ref_o, 2e-4, 1e-5 * ref_o.abs().max().item(), 'O')


@pytest.mark.parametrize('n_r,n_c,d,n_split,cs_mag,tau', [
    (4096, 83761, 64, 4, None, 0.2),       # the amazon forward role
    (4096, 83761, 64, 4, None, 0.1),
    (83761, 4096, 64, 1, 1e-9, 0.2),       # the amazon backward role: colscale ~ g ln2 / rowsum
    (83761, 4096, 64, 1, 1e-12, 0.1),
    (83761, 4096, 64, 64, 1e-6, 0.2),      # n_split at its maximum
    (300, 1000, 64, 1, None, 0.2),         # n_r not a multiple of 128, n_c not a multiple of 64
    (300, 1000, 64, 16, 1e-9, 0.1),        # n_split at its maximum (one C tile per unit)
    (300, 1000, 32, 1, 1e-9, 0.2),
    (300, 1000, 32, 16, None, 0.1),
    (1000, 777, 32, 13, 1e-6, 0.2),        # n_c not a multiple of 8
    (200, 778, 64, 1, 1e-12, 0.2),
    (300, 1003, 32, 2, None, 0.1),
    (4096, 9000, 32, 5, None, 0.2),
])
def test_f16x3_matches_float64(n_r, n_c, d, n_split, cs_mag, tau):
    g = torch.Generator().manual_seed(n_r + n_c + d + n_split)
    off = LOG2E / tau
    R = _operand(torch.randn(n_r, d, generator=g).cuda(), off)
    C = _operand(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    cs = None if cs_mag is None else _colscale((n_c + 63) // 64 * 64, cs_mag, g)
    rs, o = _contract(R, n_r, C, n_c, d, cs, off, n_split)
    ref_rs, ref_o = _reference(R[0][:n_r], C[0][:n_c], None if cs is None else cs[:n_c], off)
    _check(rs, o, ref_rs, ref_o)


@pytest.mark.parametrize('d', [32, 64])
@pytest.mark.parametrize('backward', [False, True])
def test_f16x3_special_operands(d, backward):
    """Exact zeros, entries below 2^-14 (hi = 0, lo carries them) and entries at the bound (|x| = alpha = offset = 16)."""
    g = torch.Generator().manual_seed(d + 7 * backward)
    off = 16.0
    n_a, n_t = 700, 1500
    a = torch.randn(n_a, d, generator=g)
    t = torch.randn(n_t, d, generator=g)
    for x in (a, t):
        x[::5, : d // 2] = 0.0                                    # exact zeros
        x[1::5, 1:] *= 1e-6                                       # one large entry, the others normalise to < 2^-14
        x[2::5] = 0.0
        x[2::5, 3] = 1.0                                          # one-hot: the entry is alpha itself after normalising
        x[3::5, 0] = 0.0
        x[3::5, 1:4] = x[3::5, 1:4].sign() * 3e-5 * x[3::5].norm(dim=1, keepdim=True)   # entries straddling 2^-14
    A, T = _operand(a.cuda(), off), _operand(t.cuda(), 1.0)
    hi, lo = f16x3_split(A[0].cpu().numpy())
    assert (hi == 0).sum() > 0 and ((np.abs(A[0].cpu().numpy()) < 2.0 ** -14) & (A[0].cpu().numpy() != 0)).sum() > 0
    assert A[0].abs().max().item() >= 15.99
    if backward:                                                  # R = table rows, C = scaled anchors, colscale
        cs = _colscale((n_a + 63) // 64 * 64, 1e-9, g)
        rs, o = _contract(T, n_t, A, n_a, d, cs, off, 1, with_rowsum=True)
        ref_rs, ref_o = _reference(T[0][:n_t], A[0][:n_a], cs[:n_a], off)
    else:
        rs, o = _contract(A, n_a, T, n_t, d, None, off, 4)
        ref_rs, ref_o = _reference(A[0][:n_a], T[0][:n_t], None, off)
    _check(rs, o, ref_rs, ref_o)


@pytest.mark.parametrize('d', [32, 64])
@pytest.mark.parametrize('norm_mode', [0, 1, 2])
def test_operand_writer_matches_split_and_rows_normalize(d, norm_mode):
    """ssl_rows_normalize_f16x3: out and rinv bit-identical to ssl_rows_normalize, hi / lo equal to the split rule bit for
    bit (including entries below 2^-14), padding rows zero."""
    from sslrec_b200._lib import lib, check
    g = torch.Generator().manual_seed(d + norm_mode)
    n = 1000
    x = torch.randn(n, d, generator=g)
    x[::3, 1:] *= 1e-6
    x[5] = 0.0
    x = x.cuda()
    alpha = LOG2E / 0.1
    hat, hi, lo, rinv = _operand(x, alpha, norm_mode)
    npad = hat.shape[0]
    ref, ref_rinv = torch.empty(npad, d, **F32), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, norm_mode, alpha, ref.data_ptr(), None, ref_rinv.data_ptr(), None, None,
                                 None, None, 0, _s()), 'ssl_rows_normalize')
    torch.cuda.synchronize()
    assert torch.equal(hat[:n], ref[:n]) and torch.equal(rinv, ref_rinv)
    assert (hat[n:] == 0).all() and (hi[n:] == 0).all() and (lo[n:] == 0).all()
    nh, nl = f16x3_split(hat.cpu().numpy())
    np.testing.assert_array_equal(hi.cpu().numpy().view(np.uint16), nh.view(np.uint16))
    np.testing.assert_array_equal(lo.cpu().numpy().view(np.uint16), nl.view(np.uint16))
    assert (np.abs(hat.cpu().numpy()) < 2.0 ** -14).sum() > 0


@pytest.mark.parametrize('n_r,n_c,d,n_split', [(83761, 4096, 64, 1), (4096, 83761, 64, 4), (4096, 9000, 32, 4)])
def test_f16x3_is_bit_stable(n_r, n_c, d, n_split):
    g = torch.Generator().manual_seed(11)
    off = LOG2E / 0.2
    R = _operand(torch.randn(n_r, d, generator=g).cuda(), off)
    C = _operand(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    cs = _colscale((n_c + 63) // 64 * 64, 1e-9, g)
    rs1, o1 = _contract(R, n_r, C, n_c, d, cs, off, n_split)
    rs2, o2 = _contract(R, n_r, C, n_c, d, cs, off, n_split)
    assert torch.equal(rs1, rs2) and torch.equal(o1, o2)


@pytest.mark.parametrize('n_r,n_c,d,n_split,colscale', [(83761, 4096, 64, 1, True), (4096, 83761, 64, 4, False), (300, 1003, 32, 2, True)])
def test_f16x3_agrees_with_tf32x3(n_r, n_c, d, n_split, colscale):
    """Both kernels on the same rows agree at the level of the tensor core's fp32 accumulation, which truncates rather than
    rounds: over the ~1300 k-steps of a unit at the bench shapes that is ~1e-5 relative, ten times below either kernel's
    tolerance against float64."""
    from sslrec_b200._lib import lib, check
    g = torch.Generator().manual_seed(3)
    off = LOG2E / 0.2
    xr, xc = torch.randn(n_r, d, generator=g).cuda(), torch.randn(n_c, d, generator=g).cuda()
    R, C = _operand(xr, off), _operand(xc, 1.0)
    cs = _colscale((n_c + 63) // 64 * 64, 1e-9, g) if colscale else None
    rs16, o16 = _contract(R, n_r, C, n_c, d, cs, off, n_split)

    def tf32_operand(x, alpha):
        n = x.shape[0]
        npad = (n + 63) // 64 * 64
        hat, hi, lo = torch.empty(npad, d, **F32), torch.empty(npad, d, **F32), torch.empty(npad, d, **F32)
        thi, tlo = torch.empty(d, npad, **F32), torch.empty(d, npad, **F32)
        check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), None, None, hi.data_ptr(), lo.data_ptr(),
                                     thi.data_ptr(), tlo.data_ptr(), npad, _s()), 'ssl_rows_normalize')
        return hi, lo, thi, tlo, npad
    Rt, Ct = tf32_operand(xr, off), tf32_operand(xc, 1.0)
    rs32, o32 = torch.zeros(n_split, n_r, **F32), torch.zeros(n_split, n_r, d, **F32)
    check(lib.ssl_softmax_gemm_tf32x3(Rt[0].data_ptr(), Rt[1].data_ptr(), n_r, Ct[0].data_ptr(), Ct[1].data_ptr(), Ct[2].data_ptr(),
                                      Ct[3].data_ptr(), Ct[4], n_c, d, None if cs is None else cs.data_ptr(), off, n_split,
                                      rs32.data_ptr(), o32.data_ptr(), _s()), 'ssl_softmax_gemm_tf32x3')
    torch.cuda.synchronize()
    rs32, o32, rs16, o16 = rs32.sum(0), o32.sum(0), rs16.sum(0), o16.sum(0)
    print(f'f16x3 vs tf32x3: rowsum max rel {((rs16 - rs32).abs() / rs32.abs()).max().item():.2e}, '
          f'O max abs / max|O| {((o16 - o32).abs().max() / o32.abs().max()).item():.2e}')
    H.close(rs16, rs32, 2e-5, 0.0, 'rowsum f16x3 vs tf32x3')
    H.close(o16, o32, 1e-4, 1e-6 * o32.abs().max().item(), 'O f16x3 vs tf32x3')


@pytest.mark.parametrize('d', [32, 64])
def test_f16x3_live_roles(d):
    """LIVE_ROWS / LIVE_COLS equal the plain call at n = live bit for bit, for live = 0, a ragged count and the capacity;
    zero live rows write nothing (rows) or zero partials (columns)."""
    g = torch.Generator().manual_seed(d)
    off = LOG2E / 0.2
    cap_a, n_t = 1000, 3000
    A = _operand(torch.randn(cap_a, d, generator=g).cuda(), off)
    T = _operand(torch.randn(n_t, d, generator=g).cuda(), 1.0)
    cs = _colscale((cap_a + 63) // 64 * 64, 1e-9, g)
    for live_n in (0, 1, 333, cap_a):
        live = torch.tensor([live_n], dtype=torch.int64, device='cuda')
        # forward: R = anchors, live rows
        rs = torch.full((4, cap_a), float('nan'), **F32)
        o = torch.full((4, cap_a, d), float('nan'), **F32)
        from sslrec_b200._lib import lib, check
        check(lib.ssl_softmax_gemm_f16x3_live(A[1].data_ptr(), A[2].data_ptr(), cap_a, T[1].data_ptr(), T[2].data_ptr(), n_t, d, None, off,
                                              4, rs.data_ptr(), o.data_ptr(), live.data_ptr(), LIVE_ROWS, _s()), 'live rows')
        torch.cuda.synchronize()
        assert torch.isnan(rs[:, live_n:]).all() and torch.isnan(o[:, live_n:]).all()
        if live_n:
            rs_p, o_p = _contract(A, live_n, T, n_t, d, None, off, 4)
            assert torch.equal(rs[:, :live_n], rs_p) and torch.equal(o[:, :live_n], o_p)
        # backward: C = anchors, live columns, colscale past the count never read
        cs_l = cs.clone()
        cs_l[live_n:] = float('nan')
        o = torch.full((1, n_t, d), float('nan'), **F32)
        check(lib.ssl_softmax_gemm_f16x3_live(T[1].data_ptr(), T[2].data_ptr(), n_t, A[1].data_ptr(), A[2].data_ptr(), cap_a, d,
                                              cs_l.data_ptr(), off, 1, None, o.data_ptr(), live.data_ptr(), LIVE_COLS, _s()), 'live cols')
        torch.cuda.synchronize()
        if live_n == 0:
            assert (o == 0).all()
        else:
            _, o_p = _contract(T, n_t, A, live_n, d, cs, off, 1, with_rowsum=False)
            assert torch.equal(o, o_p)


def test_f16x3_rejects_bad_arguments():
    """Rejected arguments return SSL_E_ARG before any write: the NaN sentinels stay."""
    from sslrec_b200._lib import lib
    d, n = 64, 256
    g = torch.Generator().manual_seed(5)
    R, C = _operand(torch.randn(n, d, generator=g).cuda(), 7.0), _operand(torch.randn(n, d, generator=g).cuda(), 1.0)
    rs, o = torch.full((1, n), float('nan'), **F32), torch.full((1, n, d), float('nan'), **F32)
    live = torch.tensor([n], dtype=torch.int64, device='cuda')
    base = dict(rh=R[1].data_ptr(), rl=R[2].data_ptr(), ch=C[1].data_ptr(), cl=C[2].data_ptr(), d=d, off=7.0, ns=1, cs=None)
    bad = [dict(off=16.5), dict(off=-0.5), dict(off=float('nan')), dict(d=48), dict(ns=5), dict(rh=R[1].data_ptr() + 2),
           dict(cl=C[2].data_ptr() + 8), dict(ch=None), dict(cs=torch.zeros(n + 2, **F32).data_ptr() + 4)]
    for b in bad:
        a = {**base, **b}
        args = (a['rh'], a['rl'], n, a['ch'], a['cl'], n, a['d'], a['cs'], a['off'], a['ns'], rs.data_ptr(), o.data_ptr())
        assert lib.ssl_softmax_gemm_f16x3(*args, _s()) != 0, b
        assert lib.ssl_softmax_gemm_f16x3_live(*args, live.data_ptr(), LIVE_ROWS, _s()) != 0, b
    args = (base['rh'], base['rl'], n, base['ch'], base['cl'], n, d, None, 7.0, 1, rs.data_ptr(), o.data_ptr())
    assert lib.ssl_softmax_gemm_f16x3_live(*args, None, LIVE_ROWS, _s()) != 0
    assert lib.ssl_softmax_gemm_f16x3_live(*args, live.data_ptr(), 3, _s()) != 0
    torch.cuda.synchronize()
    assert torch.isnan(rs).all() and torch.isnan(o).all()
    # the operand writer: raw rows (norm_mode 3), |alpha| > 16, dims other than 32 / 64
    x = torch.randn(n, d, generator=g).cuda()
    out, ri = torch.full((n, d), float('nan'), **F32), torch.full((n,), float('nan'), **F32)
    hi, lo = torch.full((n, d), float('nan'), **F16), torch.full((n, d), float('nan'), **F16)
    for mode, alpha, dd in ((3, 1.0, d), (0, 16.5, d), (0, -17.0, d), (0, 1.0, 48)):
        assert lib.ssl_rows_normalize_f16x3(x.data_ptr(), d, None, n, dd, mode, alpha, out.data_ptr(), ri.data_ptr(), hi.data_ptr(),
                                            lo.data_ptr(), _s()) != 0
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and torch.isnan(ri).all() and torch.isnan(hi).all() and torch.isnan(lo).all()
