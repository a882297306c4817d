"""Where the 3xFP16 InfoNCE contraction (softmax_gemm_f16x3_kernel, d = 64) spends its cycles, phase by phase, at the
bench's four contraction shapes (GPU box).

The kernel source has an instrumented form (-DSSL_NCE_PHASES, never part of the library): each consumer warpgroup sums
the clock64() cycles of each phase of its tile loop and writes the sums to a device buffer, read back once per launch.
This tool compiles that form with nvcc into a temporary directory (or loads one given with --lib), prepares the
operands with the library's own operand writer, and prints, per shape, the mean cycles per C tile per warpgroup:

  full    waiting for the TMA ring stage (mbarrier)
  bar1    waiting for this warpgroup's turn to issue GEMM1 (named barrier)
  issue1  issuing GEMM1's 12 wgmmas
  wait1   waiting for GEMM1's results (wgmma.wait_group)
  exp     the exp phase: E', row sums, the f16x3 split into GEMM2's A fragments
  bar2    waiting for this warpgroup's turn to issue GEMM2
  issue2  issuing GEMM2's 12 wgmmas
  wait2   waiting for GEMM2's results
  other   the rest (unit prologue / epilogue, loop overhead), spread over the unit's tiles

Each GEMM of one warpgroup's tile is 12 m64n64k16 wgmmas, 3 x 64^3 FMA: 384 clocks at the 2048 dense fp16 FMA / clk / SM
of the data sheet (989.4 TFLOP/s over 132 SMs at 1830 MHz).  While one warpgroup runs its exp phase, the tensor cores
run the other's GEMM2 and GEMM1: a window of 768 clocks.  Both warpgroups' tiles need 1536 tensor-core clocks per
round, so 1536 / total is the share of the round the tensor cores can be busy.  The clock64() reads add a few cycles
per mark.

    python tools/nce_phases.py [--lib libnce_phases.so] [--csrc DIR] [--launches N] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from sslrec_b200._lib import check, lib

PHASES = ('full', 'bar1', 'issue1', 'wait1', 'exp', 'bar2', 'issue2', 'wait2', 'other')
N_CTAS, N_SLOTS = 256, len(PHASES) + 1           # kPhaseCtas, kNumPhases (the last slot counts tiles)
MMA_CLK = 384                                    # one GEMM of one warpgroup's tile at 2048 FMA / clk / SM
OFF = 7.2                                        # LOG2E / 0.2, the bench's temperature
# (n_r, n_c, n_split, role): the forward keeps the 4096 anchors resident, the backward the table rows
SHAPES = ((4096, 76469, 4, 'fwd'), (4096, 83761, 4, 'fwd'), (76469, 4096, 1, 'bwd'), (83761, 4096, 1, 'bwd'))
F32 = dict(device='cuda', dtype=torch.float32)
F16 = dict(device='cuda', dtype=torch.float16)


def smi(query):
    return subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()


def build(csrc):
    out = os.path.join(tempfile.mkdtemp(prefix='nce_phases_'), 'libnce_phases.so')
    nvcc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')
    cmd = [nvcc if os.path.exists(nvcc) else 'nvcc', '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-Xcompiler', '-fPIC',
           '--expt-relaxed-constexpr', '-DSSL_NCE_PHASES', '-shared', os.path.join(csrc, 'nce_gemm_f16x3.cu'), os.path.join(csrc, 'api.cu'),
           '-o', out]
    subprocess.run(cmd, check=True)
    return out


def load(path):
    ilib = C.CDLL(path)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    ilib.ssl_softmax_gemm_f16x3.restype = C.c_int
    ilib.ssl_softmax_gemm_f16x3.argtypes = [vp, vp, i64, vp, vp, i64, i32, vp, f32, i32, vp, vp, vp]
    ilib.ssl_nce_phases_read.restype = C.c_int
    ilib.ssl_nce_phases_read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    ilib.ssl_last_error.restype = C.c_char_p
    return ilib


def operand(x, alpha):
    n, d = x.shape
    npad = (n + 63) // 64 * 64
    hat, hi, lo, r = torch.empty(npad, d, **F32), torch.empty(npad, d, **F16), torch.empty(npad, d, **F16), torch.empty(n, **F32)
    check(lib.ssl_rows_normalize_f16x3(x.data_ptr(), d, None, n, d, 0, alpha, hat.data_ptr(), r.data_ptr(), hi.data_ptr(), lo.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), 'ssl_rows_normalize_f16x3')
    return hi, lo


def measure(ilib, nr, nc, ns, role, launches, d=64):
    """Mean cycles per tile per warpgroup of each phase, per launch; the median over ``launches`` launches."""
    g = torch.Generator().manual_seed(0)
    R, Cc = operand(torch.randn(nr, d, generator=g).cuda(), OFF), operand(torch.randn(nc, d, generator=g).cuda(), 1.0)
    npad = (nc + 63) // 64 * 64
    cs = (1e-9 * (torch.rand(npad, generator=g) + 0.5)).cuda() if role == 'bwd' else None
    rs = torch.zeros(ns, nr, **F32) if role == 'fwd' else None       # the backward does not read its row sums
    o = torch.zeros(ns, nr, d, **F32)
    buf = (C.c_ulonglong * (N_CTAS * 2 * N_SLOTS))()
    s = torch.cuda.current_stream().cuda_stream

    def launch():
        rc = ilib.ssl_softmax_gemm_f16x3(R[0].data_ptr(), R[1].data_ptr(), nr, Cc[0].data_ptr(), Cc[1].data_ptr(), nc, d,
                                         None if cs is None else cs.data_ptr(), OFF, ns, None if rs is None else rs.data_ptr(),
                                         o.data_ptr(), s)
        if rc != 0:
            raise RuntimeError(ilib.ssl_last_error().decode())
    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    per_launch = []
    for _ in range(launches):
        launch()
        torch.cuda.synchronize()
        if ilib.ssl_nce_phases_read(buf, len(buf)) != 0:
            raise RuntimeError(ilib.ssl_last_error().decode())
        v = torch.tensor(list(buf), dtype=torch.float64).view(N_CTAS, 2, N_SLOTS)
        live = v[:, :, -1] > 0
        tiles = v[:, :, -1][live].sum().item()
        per_launch.append({p: v[:, :, k][live].sum().item() / tiles for k, p in enumerate(PHASES)})
    return {p: statistics.median(x[p] for x in per_launch) for p in PHASES}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--lib', help='a prebuilt instrumented library (default: compile csrc/nce_gemm_f16x3.cu with -DSSL_NCE_PHASES)')
    ap.add_argument('--csrc', default=os.path.join(ROOT, 'sslrec_b200', 'csrc'), help='the kernel sources to compile')
    ap.add_argument('--launches', type=int, default=9)
    ap.add_argument('--json', help='write the table as JSON to this path')
    args = ap.parse_args()
    ilib = load(args.lib or build(args.csrc))
    card = smi('name,power.limit,clocks.max.sm')
    print(f'card: {card}', flush=True)
    print(f'{"shape":28s} ' + ' '.join(f'{p:>7s}' for p in PHASES) + '    total  exp/window  MMA/total', flush=True)
    rows = []
    for nr, nc, ns, role in SHAPES:
        ph = measure(ilib, nr, nc, ns, role, args.launches)
        total = sum(ph.values())
        name = f'{role} {nr} x {nc} ({ns})'
        print(f'{name:28s} ' + ' '.join(f'{ph[p]:7.0f}' for p in PHASES) + f' {total:8.0f}  {ph["exp"] / (2 * MMA_CLK):10.2f}  {4 * MMA_CLK / total:9.2f}',
              flush=True)
        rows.append(dict(shape=name, cycles_per_tile=ph, total=total))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(dict(card=card, mma_clk_per_gemm=MMA_CLK, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
