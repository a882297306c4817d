"""Time ssl_softmax_gemm_tf32x3 at the bench's four contraction shapes while sampling the SM clock and board power
(nvidia-smi, every 0.1 s), and report the tf32 MMA rate against the data-sheet peak and against the peak at the
sampled clock (132 SMs x 1024 tf32 FMA / clk x 2).  A power-capped card runs this kernel well below its maximum
clock, so the clock-adjusted share is the one that says how much of the hardware the kernel uses (GPU box).

    python tools/perf_tc_clock.py [reps]
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
DATASHEET_TF32 = 494.7e12
SHAPES = ((4096, 76469), (4096, 83761), (76469, 4096), (83761, 4096))     # forward (anchors resident) x 2, backward x 2


def smi(query):
    return subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader,nounits'], capture_output=True, text=True).stdout.strip()


def prep(x, alpha):
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, t, hi, lo = torch.empty(npad, d, **F32), torch.empty(npad // 64, d, 64, **F32), torch.empty(npad, d, **F32), torch.empty(npad, d, **F32)
    thi, tlo, r = torch.empty(d, npad, **F32), torch.empty(d, npad, **F32), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), t.data_ptr(), r.data_ptr(), hi.data_ptr(), lo.data_ptr(),
                                 thi.data_ptr(), tlo.data_ptr(), npad, torch.cuda.current_stream().cuda_stream))
    return hi, lo, thi, tlo, npad


def run(nr, nc, d, reps):
    g = torch.Generator().manual_seed(0)
    R, C = prep(torch.randn(nr, d, generator=g).cuda(), 7.2), prep(torch.randn(nc, d, generator=g).cuda(), 1.0)
    ns = choose_split((nr + 127) // 128, C[4] // 64, slots=E.NUM_SM, prefer_few=True)
    rs, o = torch.zeros(ns, nr, **F32), torch.zeros(ns, nr, d, **F32)
    s = torch.cuda.current_stream().cuda_stream

    def call():
        check(lib.ssl_softmax_gemm_tf32x3(R[0].data_ptr(), R[1].data_ptr(), nr, C[0].data_ptr(), C[1].data_ptr(), C[2].data_ptr(), C[3].data_ptr(),
                                          C[4], nc, d, None, 7.2, ns, rs.data_ptr(), o.data_ptr(), s))
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
    ms = e0.elapsed_time(e1) / reps
    vals = [tuple(float(v) for v in x.split(',')) for x in samples if x]
    mhz = statistics.median(v[0] for v in vals) if vals else float('nan')
    watts = max(v[1] for v in vals) if vals else float('nan')
    rate = 2.0 * 3 * 2 * nr * nc * d / (ms * 1e-3)               # two GEMMs x three tf32 products x 2 flop per FMA
    peak_clk = 132 * 1024 * 2 * mhz * 1e6
    print(f'nr={nr:6d} nc={nc:6d} d={d} split={ns:2d}: {ms:.4f} ms  {rate / 1e12:.1f} TFLOP/s tf32  {rate / DATASHEET_TF32:.3f} of the '
          f'data sheet  median SM clock {mhz:.0f} MHz -> {rate / peak_clk:.3f} of the clock-adjusted peak  (max {watts:.0f} W)', flush=True)


if __name__ == '__main__':
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    print(smi('name,power.limit,clocks.max.sm'))
    for nr, nc in SHAPES:
        run(nr, nc, 64, reps)
