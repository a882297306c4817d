"""The MixGCF kernels (csrc/mixgcf.cuh: ssl_mixgcf_bpr_fwd / ssl_mixgcf_bpr_bwd) executed on the host under AddressSanitizer
(tests/emu/cuda_emu.h: one pthread per CUDA thread) and compared bit for bit with a sequential float32 restatement of their
documented arithmetic (tests/emu/mixgcf_emu.cpp): the picks, alpha (drawn from the seed and injected), nhat, loss_b and coef_b
of the forward, and every per-position contribution of the backward run on identity ids into -0.0 stages.  Ragged batch sizes
around the warp and block widths; M = 1, 2, 33, 256; 1 to 8 layers; every listed row width; strided tables and views of
interleaved [N, 3, d] tables; exact ties between distinct candidates; NaN rows; alpha = 0 and alpha just below 1."""
import itertools
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RANDOM, TIES, NAN_ROWS, ALL_NAN = range(4)
DRAWN, INJECTED, ZERO, BELOW_ONE = range(4)


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'mixgcf_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'mixgcf_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _cases():
    # (B, M, n_layers, dim, stride - dim, view, pattern, alpha): every (M, dim) pair once with the batch sizes, layer counts,
    # strides, layouts, patterns and alpha modes rotating over them, then the named edge cases
    out = []
    for i, (M, d) in enumerate(itertools.product((1, 2, 33, 256), (4, 32, 60, 64, 128))):
        out.append(((1, 31, 33, 37, 70)[i % 5], M, 1 + i % 8, d, (0, 3, 4, d)[i % 4], int(i % 3 == 2), i % 4 if M > 1 else i % 2 * 2,
                    i % 4))
    out += [(300, 2, 4, 64, 0, 1, TIES, DRAWN), (37, 256, 8, 128, 4, 1, TIES, INJECTED), (33, 33, 3, 60, 0, 0, NAN_ROWS, DRAWN),
            (40, 3, 4, 32, 0, 0, ALL_NAN, DRAWN), (9, 256, 2, 4, 0, 1, ALL_NAN, BELOW_ONE), (65, 8, 8, 64, 0, 1, RANDOM, ZERO),
            (65, 1, 4, 64, 4, 0, RANDOM, ZERO), (65, 8, 4, 64, 0, 0, RANDOM, BELOW_ONE), (0, 8, 4, 32, 0, 0, RANDOM, DRAWN)]
    return out


@pytest.mark.parametrize('case', _cases(), ids=lambda c: 'B%d-M%d-L%d-d%d-x%d-view%d-pat%d-alpha%d' % c)
def test_mixgcf_kernels_match_their_sequential_restatement_on_the_host(emulator, case):
    r = subprocess.run([emulator] + [str(v) for v in case] + [str(7 + sum(case))], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
