"""Time ssl_softmax_gemm_tf32x3 vs ssl_softmax_gemm at the bench's forward / backward shapes (GPU box)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sslrec_b200._lib import lib, check
from sslrec_b200 import engine as E
from sslrec_b200.engine import choose_split
f = dict(device='cuda', dtype=torch.float32)
def prep(x, n, d, alpha):
    npad = (n + 63) // 64 * 64
    hat, t, hi, lo, thi, tlo, r = (torch.empty(npad, d, **f), torch.empty(npad // 64, d, 64, **f), torch.empty(npad, d, **f), torch.empty(npad, d, **f),
                                   torch.empty(d, npad, **f), torch.empty(d, npad, **f), torch.empty(n, **f))
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), t.data_ptr(), r.data_ptr(), hi.data_ptr(), lo.data_ptr(), thi.data_ptr(), tlo.data_ptr(), npad, torch.cuda.current_stream().cuda_stream))
    return hat, t, hi, lo, thi, tlo, npad
def run(nr, nc, d, tc, reps=10, split=None):
    g = torch.Generator().manual_seed(0)
    R = prep(torch.randn(nr, d, generator=g).cuda(), nr, d, 7.2); C = prep(torch.randn(nc, d, generator=g).cuda(), nc, d, 1.0)
    ns = split or choose_split((nr + 127) // 128, C[6] // 64, slots=E.NUM_SM if tc else 2 * E.NUM_SM, prefer_few=tc)
    rs, o = torch.zeros(ns, nr, **f), torch.zeros(ns, nr, d, **f)
    s = torch.cuda.current_stream().cuda_stream
    def call():
        if tc:
            check(lib.ssl_softmax_gemm_tf32x3(R[2].data_ptr(), R[3].data_ptr(), nr, C[2].data_ptr(), C[3].data_ptr(), C[4].data_ptr(), C[5].data_ptr(), C[6], nc, d, None, 7.2, ns, rs.data_ptr(), o.data_ptr(), s))
        else:
            check(lib.ssl_softmax_gemm(R[0].data_ptr(), nr, C[0].data_ptr(), C[1].data_ptr(), nc, d, None, 7.2, ns, rs.data_ptr(), o.data_ptr(), s))
    for _ in range(3): call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): call()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print(f'nr={nr} nc={nc} d={d} tc={tc} split={ns}: {ms:.3f} ms  {4.0 * nr * nc * d / ms / 1e9:.1f} TFLOP/s(fp32-equivalent)', flush=True)
if len(sys.argv) > 1 and sys.argv[1] == 'sweep':
    # n_split sweep at the bench's shapes: forward role (anchors resident, table streamed) and backward role (table resident)
    for nr, nc, splits in ((4096, 76469, (5, 7, 9, 14, 18, 23)), (4096, 83761, (5, 7, 9, 14, 18, 23)), (76469, 4096, (1, 2, 3, 4, 6, 8)), (83761, 4096, (1, 2, 3, 4, 6, 8)),
                           (4096, 25557, (3, 5, 9, 14)), (25557, 4096, (1, 2, 3, 4, 8))):
        print('heuristic:', end=' ')
        run(nr, nc, 64, True, reps=20)
        for sp in splits:
            run(nr, nc, 64, True, reps=20, split=sp)
    sys.exit(0)
quick = len(sys.argv) > 1
for tc in ((True,) if quick else (True, False)):
    run(4096, 83761, 64, tc)
    if not quick:
        run(83761, 4096, 64, tc)
        run(4096, 83761, 64, tc, split=9)     # fewer, longer CTAs
        run(4096, 83761, 32, tc)
