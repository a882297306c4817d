"""The ordered scatter of train.deterministic (csrc/ordered_scatter.cuh, the kernel of ssl_scatter_rows_ordered) executed on the
host under AddressSanitizer (tests/emu/cuda_emu.h: one pthread per CUDA thread) and compared bit for bit with a sequential
float32 restatement of its contract, sink[r] = sink[r] + (((c_p1 + c_p2) + c_p3) + ...) over the positions of r in order
(tests/emu/ordered_scatter_emu.cpp).  Ragged sizes around the warp width, every supported row width, strided sinks, a nonzero
prior sink, all-distinct ids, one id repeated P times, ids at 0 and N - 1 only, and dead positions (id -1).  The kernel is
grid-agnostic; the emulation runs it on a few warps, so every warp walks many units."""
import itertools
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RANDOM, DISTINCT, ONE_ID, ENDS, DEAD = range(5)


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'ordered_scatter_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'ordered_scatter_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _cases():
    # (P, dim, stride - dim, prior sink, id pattern, grid, warps per block): every (P, dim) pair once, the patterns, strides and
    # prior sinks rotating over them, then the patterns that matter most at the largest sizes
    out = []
    for i, (P, d) in enumerate(itertools.product((0, 1, 31, 33, 4096, 3 * 4096 + 5), (4, 36, 64, 128))):
        out.append((P, d, (0, 3, d, 64)[i % 4], i % 2, i % 5, 1 + i % 3, 1 + i % 4))
    out += [(4096, 128, 0, 1, ONE_ID, 2, 4), (3 * 4096 + 5, 64, 64, 1, ONE_ID, 3, 2), (3 * 4096 + 5, 128, 5, 0, DISTINCT, 2, 4),
            (33, 4, 0, 1, ENDS, 1, 1), (3 * 4096 + 5, 36, 0, 1, DEAD, 2, 4), (31, 128, 128, 1, DEAD, 1, 2)]
    return out


@pytest.mark.parametrize('case', _cases(), ids=lambda c: 'P%d-d%d-x%d-prior%d-pat%d-g%dw%d' % c)
def test_ordered_scatter_kernel_matches_its_sequential_restatement_on_the_host(emulator, case):
    P, d, extra, prior, pattern, grid, warps = case
    r = subprocess.run([emulator] + [str(v) for v in (P, d, extra, prior, pattern, 1000 + P + d, grid, warps)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
