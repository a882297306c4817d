"""The fused score + mask + top-k kernels (sslrec_b200/csrc/predict_topk.cuh) executed ON THE HOST: the same source the library compiles
for sm_90a, run thread by thread (tests/emu/cuda_emu.h + cuda_emu_warp.h) under AddressSanitizer, and compared bit for bit (item ids and value bits) with a
host restatement of ssl_predict_mask + ssl_topk: one sequential fp32 FMA chain per score, the mask formula, a sort by (value descending,
item ascending).  The cases cut tiles by n_b and n_item, give a chunk several tiles, shrink the candidate lists to k + 128 keys so that
they are compacted over and over, use k = 1, 7, 40 and 256 (up to k = n_item), strided tables, repeated users, duplicated item rows,
an all-zero user, a user with fewer than k unmasked items, and the three mask modes.  The workspace starts as garbage.  No GPU involved."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

#        n_b  n_item dim u_stride i_stride mode(0 none, 1 dense, 2 CSR) k  chunks cap  seed
CASES = [(1, 1, 4, 4, 4, 0, 1, 1, 129, 1),
         (3, 300, 4, 4, 4, 2, 1, 3, 129, 2),
         (130, 1000, 36, 36, 108, 2, 7, 3, 135, 3),
         (129, 700, 64, 64, 64, 1, 40, 2, 168, 4),
         (5, 1500, 128, 160, 128, 2, 256, 2, 384, 5),
         (40, 900, 32, 32, 32, 0, 40, 2, 208, 6),
         (3, 256, 20, 20, 20, 1, 256, 1, 640, 7)]


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'predict_topk_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'predict_topk_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and 'asan' in (r.stderr or '').lower():
        r = subprocess.run([c for c in cmd if not c.startswith('-fsanitize')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'b%d_i%d_d%d_m%d_k%d_c%d' % (c[0], c[1], c[2], c[5], c[6], c[7]))
def test_predict_topk_kernels_on_the_host(emulator, case):
    r = subprocess.run([emulator] + [str(v) for v in case], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'bad=0' in r.stdout, r.stdout[-500:] + '\n' + r.stderr[-2000:]
