"""Time the two tensor-core InfoNCE contractions, ssl_softmax_gemm_tf32x3 and ssl_softmax_gemm_f16x3, alternately at the
bench's four contraction shapes while sampling the SM clock and board power (nvidia-smi, every 0.1 s), and report each
kernel's MMA rate against its own data-sheet peak and against its peak at the sampled clock (132 SMs x 1024 tf32 or
2048 fp16 FMA / clk x 2).  A power-capped card runs these kernels well below its maximum clock, so the clock-adjusted
share is the one that says how much of the hardware a kernel uses (GPU box).

    python tools/perf_tc_clock.py [reps] [rounds]          # A/B, ``rounds`` alternations per shape (default 2)
    python tools/perf_tc_clock.py --sweep [reps]           # f16x3 n_split sweep at the four shapes
"""
import os
import statistics
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from sslrec_b200 import engine as E
from sslrec_b200._lib import check, lib
from sslrec_b200.engine import choose_split

F32 = dict(device='cuda', dtype=torch.float32)
F16 = dict(device='cuda', dtype=torch.float16)
DATASHEET = {'tf32x3': 494.7e12, 'f16x3': 989.4e12}
FMA_PER_CLK = {'tf32x3': 1024, 'f16x3': 2048}
SHAPES = ((4096, 76469), (4096, 83761), (76469, 4096), (83761, 4096))     # forward (anchors resident) x 2, backward x 2
OFF = 7.2                                                                 # LOG2E / 0.2


def smi(query):
    return subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits'], capture_output=True, text=True).stdout.strip()


def prep_tf32(x, alpha):
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, hi, lo = torch.empty(npad, d, **F32), torch.empty(npad, d, **F32), torch.empty(npad, d, **F32)
    thi, tlo, r = torch.empty(d, npad, **F32), torch.empty(d, npad, **F32), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), None, r.data_ptr(), hi.data_ptr(), lo.data_ptr(),
                                 thi.data_ptr(), tlo.data_ptr(), npad, torch.cuda.current_stream().cuda_stream))
    return hi, lo, thi, tlo, npad


def prep_f16(x, alpha):
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, hi, lo, r = torch.empty(npad, d, **F32), torch.empty(npad, d, **F16), torch.empty(npad, d, **F16), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize_f16x3(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), r.data_ptr(), hi.data_ptr(), lo.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    return hi, lo, npad


def make_call(kind, nr, nc, d, ns=None):
    """A closure launching one contraction (R = scaled rows, C = unit rows; the backward shapes carry a colscale of the
    backward's magnitude) and its split."""
    g = torch.Generator().manual_seed(0)
    xr, xc = torch.randn(nr, d, generator=g).cuda(), torch.randn(nc, d, generator=g).cuda()
    npad = (nc + 63) // 64 * 64
    cs = (1e-9 * (torch.rand(npad, generator=g) + 0.5)).cuda() if nr > nc else None
    csp = None if cs is None else cs.data_ptr()
    ns = ns or choose_split((nr + 127) // 128, npad // 64, slots=E.NUM_SM, prefer_few=True)
    rs, o = torch.zeros(ns, nr, **F32), torch.zeros(ns, nr, d, **F32)
    s = torch.cuda.current_stream().cuda_stream
    if kind == 'tf32x3':
        R, C = prep_tf32(xr, OFF), prep_tf32(xc, 1.0)

        def call():
            check(lib.ssl_softmax_gemm_tf32x3(R[0].data_ptr(), R[1].data_ptr(), nr, C[0].data_ptr(), C[1].data_ptr(), C[2].data_ptr(),
                                              C[3].data_ptr(), C[4], nc, d, csp, OFF, ns, rs.data_ptr(), o.data_ptr(), s))
    else:
        R, C = prep_f16(xr, OFF), prep_f16(xc, 1.0)

        def call():
            check(lib.ssl_softmax_gemm_f16x3(R[0].data_ptr(), R[1].data_ptr(), nr, C[0].data_ptr(), C[1].data_ptr(), nc, d, csp, OFF, ns,
                                             rs.data_ptr(), o.data_ptr(), s))
    return call, ns


def timed(call, reps):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    samples, stop = [], threading.Event()

    def sampler():
        while not stop.is_set():
            samples.append(smi('clocks.sm,power.draw'))
            time.sleep(0.1)
    th = threading.Thread(target=sampler)
    th.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    stop.set()
    th.join()
    vals = [tuple(float(v) for v in x.split(',')) for x in samples if x]
    mhz = statistics.median(v[0] for v in vals) if vals else float('nan')
    watts = max(v[1] for v in vals) if vals else float('nan')
    return e0.elapsed_time(e1) / reps, mhz, watts


def report(kind, nr, nc, d, ns, ms, mhz, watts):
    rate = 2.0 * 3 * 2 * nr * nc * d / (ms * 1e-3)               # two GEMMs x three products x 2 flop per FMA
    peak_clk = 132 * FMA_PER_CLK[kind] * 2 * mhz * 1e6
    print(f'{kind:6s} nr={nr:6d} nc={nc:6d} d={d} split={ns:2d}: {ms:.4f} ms  {rate / 1e12:.1f} TFLOP/s  {rate / DATASHEET[kind]:.3f} of '
          f'its data sheet  median SM clock {mhz:.0f} MHz -> {rate / peak_clk:.3f} of its clock-adjusted peak  (max {watts:.0f} W)',
          flush=True)


if __name__ == '__main__':
    args = [a for a in sys.argv[1:] if not a.startswith('--')]
    reps = int(args[0]) if args else 2000
    print(smi('name,power.limit,clocks.max.sm'))
    if '--sweep' in sys.argv:
        for nr, nc in SHAPES:
            max_split = max(1, min(((nc + 63) // 64) // 4, 64))
            for ns in sorted({1, 2, 3, 4, 5, 6, 8, 9, 12, 16, 18} & set(range(1, max_split + 1))):
                call, _ = make_call('f16x3', nr, nc, 64, ns)
                report('f16x3', nr, nc, 64, ns, *timed(call, reps))
        sys.exit(0)
    rounds = int(args[1]) if len(args) > 1 else 2
    for nr, nc in SHAPES:
        calls = {k: make_call(k, nr, nc, 64) for k in ('tf32x3', 'f16x3')}
        for _ in range(rounds):
            for k, (call, ns) in calls.items():
                report(k, nr, nc, 64, ns, *timed(call, reps))
