"""The score-argmax selection of dynamic negative sampling (csrc/hard_negs.cuh, the kernel of ssl_neg_select) executed on the
host under AddressSanitizer (tests/emu/cuda_emu.h: one pthread per CUDA thread) and compared bit for bit with a sequential
float32 restatement of its documented order: each score one FMA chain over k = 0 .. dim-1, the lowest j among equal largest
scores, NaN scores never chosen, candidate 0 when all are NaN (tests/emu/neg_select_emu.cpp).  Ragged batch sizes around the
warp and block widths, M from 2 to 256 (one to eight candidates per lane), every listed row width, strided tables and views of
an interleaved [N, 3, d] layer sum, exact ties between distinct candidates, NaN rows and pairs whose every score is NaN."""
import itertools
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RANDOM, TIES, NAN_ROWS, ALL_NAN = range(4)


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'neg_select_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'neg_select_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _cases():
    # (B, M, dim, user stride - dim, item stride - dim, view, pattern): every (M, dim) pair once with the batch sizes, strides,
    # layouts and patterns rotating over them, then each pattern at the extremes of M
    out = []
    for i, (M, d) in enumerate(itertools.product((2, 3, 32, 256), (4, 32, 60, 64, 128))):
        view = i % 3 == 2
        ue = (0, 3, 4, d)[i % 4]
        out.append(((1, 31, 33, 37, 300)[i % 5], M, d, ue, ue if view else (0, 5, 0, 64)[i % 4], int(view), i % 4))
    out += [(300, 2, 64, 0, 0, 1, TIES), (37, 256, 128, 4, 4, 1, TIES), (33, 256, 60, 0, 4, 0, NAN_ROWS), (300, 3, 32, 0, 0, 0, ALL_NAN),
            (9, 256, 4, 0, 0, 1, ALL_NAN), (0, 8, 32, 0, 0, 0, RANDOM)]
    return out


@pytest.mark.parametrize('case', _cases(), ids=lambda c: 'B%d-M%d-d%d-u%d-i%d-view%d-pat%d' % c)
def test_neg_select_kernel_matches_its_sequential_restatement_on_the_host(emulator, case):
    r = subprocess.run([emulator] + [str(v) for v in case] + [str(7 + sum(case))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
