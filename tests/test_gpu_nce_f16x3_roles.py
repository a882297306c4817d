"""The role-specialised exp phase of the 3xFP16 InfoNCE contraction (ssl_softmax_gemm_f16x3[_live]) through the C ABI.

Each launch takes one of three exp phases, picked from its arguments: the forward (no colscale: the 2^14 bias folded
into the offset, the flush rule only above offset 13.5), the backward (colscale, no row sums) and the general one
(colscale and row sums).  Checked here against float64 at the bench shapes and at ragged ones, in both roles and both
live modes, at offsets 0, 7.2 (the bench's tau = 0.2), 13.5 (the last offset without the flush rule) and 16 (the
largest the ABI accepts), with the bounds of test_gpu_nce_f16x3.py; and that the forward's folded exp phase agrees with
the general one (a colscale of ones), and that dropping the backward's row sums leaves O bit for bit as it was."""
import pytest
import torch

from test_gpu_nce_f16x3 import F32, LIVE_COLS, LIVE_ROWS, _check, _colscale, _contract, _operand, _reference

pytestmark = pytest.mark.gpu


def _operands(n_r, n_c, d, off, g):
    """R rows scaled by ``off`` and C rows of unit norm, so |S| <= off.  At off = 0 both keep unit norm and opposite
    signs (R <= 0 <= C entrywise), so that S <= 0 = off still holds."""
    xr, xc = torch.randn(n_r, d, generator=g), torch.randn(n_c, d, generator=g)
    if off == 0.0:
        return _operand(-xr.abs().cuda(), 1.0), _operand(xc.abs().cuda(), 1.0)
    return _operand(xr.cuda(), off), _operand(xc.cuda(), 1.0)


@pytest.mark.parametrize('off', [0.0, 7.2, 13.5, 16.0])
@pytest.mark.parametrize('n_r,n_c,d,n_split', [
    (4096, 83761, 64, 4),        # the amazon forward: 83761 = 1308 x 64 + 49, a ragged last tile
    (4096, 76469, 64, 4),
    (300, 1003, 32, 2),
])
def test_forward_role_matches_float64(n_r, n_c, d, n_split, off):
    g = torch.Generator().manual_seed(n_c + int(4 * off))
    R, C = _operands(n_r, n_c, d, off, g)
    rs, o = _contract(R, n_r, C, n_c, d, None, off, n_split)
    _check(rs, o, *_reference(R[0][:n_r], C[0][:n_c], None, off))


@pytest.mark.parametrize('off', [0.0, 7.2, 16.0])
@pytest.mark.parametrize('n_r,n_c,d,cs_mag', [
    (83761, 4096, 64, 1e-9),     # the amazon backward
    (76469, 4096, 64, 1e-12),
    (1000, 777, 32, 1e-6),       # n_c not a multiple of 8
])
def test_backward_role_matches_float64(n_r, n_c, d, cs_mag, off):
    """O from the backward's exp phase (no row sums) against float64, and bit for bit against the general exp phase of
    the same launch with row sums, whose row sums are checked too."""
    g = torch.Generator().manual_seed(n_r + int(4 * off))
    R, C = _operands(n_r, n_c, d, off, g)
    cs = _colscale((n_c + 63) // 64 * 64, cs_mag, g)
    _, o = _contract(R, n_r, C, n_c, d, cs, off, 1, with_rowsum=False)
    rs_g, o_g = _contract(R, n_r, C, n_c, d, cs, off, 1, with_rowsum=True)
    assert torch.equal(o, o_g)
    _check(rs_g, o, *_reference(R[0][:n_r], C[0][:n_c], cs[:n_c], off))


@pytest.mark.parametrize('off', [0.0, 7.2, 13.5, 16.0])
@pytest.mark.parametrize('n_r,n_c,d,n_split', [(4096, 83761, 64, 4), (300, 1003, 32, 2)])
def test_forward_fold_matches_unit_colscale(n_r, n_c, d, n_split, off):
    """A forward launch with a colscale of ones (M = 1: E' = exp2(S - offset) 2^14, the general exp phase) and the
    null-colscale launch (E' = exp2(S - (offset - 14))) agree within the float64 bounds."""
    g = torch.Generator().manual_seed(7 + n_c + int(4 * off))
    R, C = _operands(n_r, n_c, d, off, g)
    ones = torch.ones((n_c + 63) // 64 * 64, **F32)
    rs, o = _contract(R, n_r, C, n_c, d, None, off, n_split)
    rs1, o1 = _contract(R, n_r, C, n_c, d, ones, off, n_split)
    _check(rs, o, rs1.sum(0).double(), o1.sum(0).double())


@pytest.mark.parametrize('off', [0.0, 7.2, 16.0])
@pytest.mark.parametrize('d', [32, 64])
def test_live_roles_match_float64(d, off):
    """LIVE_ROWS in the forward role and LIVE_COLS in the backward role at a ragged live count, against float64 over the
    live rows / columns."""
    from sslrec_b200._lib import check, lib
    g = torch.Generator().manual_seed(d + int(4 * off))
    cap_a, n_t, live_n = 1000, 3001, 333
    A, T = _operands(cap_a, n_t, d, off, g)
    live = torch.tensor([live_n], dtype=torch.int64, device='cuda')
    s = torch.cuda.current_stream().cuda_stream
    # forward: R = anchors, the first live_n rows live
    rs, o = torch.zeros(4, cap_a, **F32), torch.zeros(4, cap_a, d, **F32)
    check(lib.ssl_softmax_gemm_f16x3_live(A[1].data_ptr(), A[2].data_ptr(), cap_a, T[1].data_ptr(), T[2].data_ptr(), n_t, d, None, off,
                                          4, rs.data_ptr(), o.data_ptr(), live.data_ptr(), LIVE_ROWS, s), 'live rows')
    torch.cuda.synchronize()
    _check(rs[:, :live_n], o[:, :live_n], *_reference(A[0][:live_n], T[0][:n_t], None, off))
    # backward: C = anchors, the first live_n columns live; no row sums
    cs = _colscale((cap_a + 63) // 64 * 64, 1e-9, g)
    o = torch.zeros(1, n_t, d, **F32)
    check(lib.ssl_softmax_gemm_f16x3_live(T[1].data_ptr(), T[2].data_ptr(), n_t, A[1].data_ptr(), A[2].data_ptr(), cap_a, d,
                                          cs.data_ptr(), off, 1, None, o.data_ptr(), live.data_ptr(), LIVE_COLS, s), 'live cols')
    torch.cuda.synchronize()
    _check(None, o, None, _reference(T[0][:n_t], A[0][:live_n], cs[:live_n], off)[1])
