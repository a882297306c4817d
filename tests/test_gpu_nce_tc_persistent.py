"""The persistent tensor-core InfoNCE contraction (ssl_softmax_gemm_tf32x3) through the C ABI against a float64
restatement: more (R tile, C chunk) units than CTAs, ragged n_r / n_c, n_split from 1 to its maximum, the colscale path,
d = 32 and 64, and run-to-run bit stability of the partial outputs."""
import pytest
import torch

import ssl_test_helpers as H

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
F32 = dict(device='cuda', dtype=torch.float32)


def _operand(x, alpha):
    """Rows of x normalised and scaled by alpha, with the hi / lo and transposed hi / lo copies the kernel reads."""
    from sslrec_b200._lib import lib, check
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, t, hi, lo = torch.empty(npad, d, **F32), torch.empty(npad // 64, d, 64, **F32), torch.empty(npad, d, **F32), torch.empty(npad, d, **F32)
    thi, tlo, rinv = torch.empty(d, npad, **F32), torch.empty(d, npad, **F32), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), t.data_ptr(), rinv.data_ptr(), hi.data_ptr(),
                                 lo.data_ptr(), thi.data_ptr(), tlo.data_ptr(), npad, torch.cuda.current_stream().cuda_stream), 'rows_normalize')
    return hat, hi, lo, thi, tlo, npad


def _contract(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum):
    from sslrec_b200._lib import lib, check
    rs = torch.zeros(n_split, n_r, **F32) if with_rowsum else None
    o = torch.zeros(n_split, n_r, d, **F32)
    check(lib.ssl_softmax_gemm_tf32x3(R[1].data_ptr(), R[2].data_ptr(), n_r, C[1].data_ptr(), C[2].data_ptr(), C[3].data_ptr(), C[4].data_ptr(),
                                      C[5], n_c, d, None if cs is None else cs.data_ptr(), off, n_split,
                                      None if rs is None else rs.data_ptr(), o.data_ptr(), torch.cuda.current_stream().cuda_stream),
          'ssl_softmax_gemm_tf32x3')
    torch.cuda.synchronize()
    return rs, o


def _reference(A, T, cs, off):
    """rowsum_i = sum_j exp2(a_i . t_j - off) cs_j and O_i = sum_j exp2(...) cs_j t_j in float64, in row chunks."""
    A, T = A.double(), T.double()
    rs, o = torch.empty(A.shape[0], dtype=torch.float64, device='cuda'), torch.empty(A.shape, dtype=torch.float64, device='cuda')
    for r in range(0, A.shape[0], 8192):
        E = torch.exp2(A[r:r + 8192] @ T.T - off)
        if cs is not None:
            E = E * cs.double()
        rs[r:r + 8192], o[r:r + 8192] = E.sum(1), E @ T
    return rs, o


@pytest.mark.parametrize('n_r,n_c,d,n_split,colscale', [
    (83761, 4096, 64, 1, True),          # the amazon backward role: 655 units on one CTA per SM
    (83761, 4096, 64, 3, False),
    (300, 1000, 64, 1, False),           # n_r not a multiple of 128, n_c not a multiple of 64
    (300, 1000, 64, 16, True),           # n_split at its maximum (one C tile per unit)
    (300, 1000, 32, 1, True),
    (300, 1000, 32, 16, False),
    (4096, 9000, 64, 5, False),          # forward role: fewer units than SMs
    (1000, 777, 32, 13, True),
    (200, 778, 64, 1, True),             # n_c % 8 = 2 and 3: the last column group of the transposed copy is partly
    (300, 1003, 32, 2, False),           # past n_c, and its valid columns are spread over the group
])
def test_persistent_contraction_matches_float64(n_r, n_c, d, n_split, colscale):
    g = torch.Generator().manual_seed(n_r + n_c + d + n_split)
    off = LOG2E / 0.2
    R = _operand(torch.randn(n_r, d, generator=g).cuda(), off)
    C = _operand(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    cs = (torch.rand(C[5], generator=g) + 0.5).cuda() if colscale else None
    rs, o = _contract(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum=True)
    ref_rs, ref_o = _reference(R[0][:n_r], C[0][:n_c], None if cs is None else cs[:n_c], off)
    H.close(rs.sum(0), ref_rs, 2e-4, 1e-5 * ref_rs.abs().max().item(), 'rowsum')
    H.close(o.sum(0), ref_o, 2e-4, 1e-5 * ref_o.abs().max().item(), 'O')


@pytest.mark.parametrize('n_r,n_c,d,n_split', [(83761, 4096, 64, 1), (4096, 9000, 32, 4)])
def test_persistent_contraction_is_bit_stable(n_r, n_c, d, n_split):
    g = torch.Generator().manual_seed(11)
    off = LOG2E / 0.2
    R = _operand(torch.randn(n_r, d, generator=g).cuda(), off)
    C = _operand(torch.randn(n_c, d, generator=g).cuda(), 1.0)
    cs = (torch.rand(C[5], generator=g) + 0.5).cuda()
    rs1, o1 = _contract(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum=True)
    rs2, o2 = _contract(R, n_r, C, n_c, d, cs, off, n_split, with_rowsum=True)
    assert torch.equal(rs1, rs2) and torch.equal(o1, o2)
