"""The sampled softmax kernels (csrc/ssm.cuh: ssl_ssm_fwd / ssl_ssm_bwd) executed on the host under AddressSanitizer
(tests/emu/cuda_emu.h: one pthread per CUDA thread; tests/emu/ssm_emu.cpp) and compared bit for bit with the sequential float32
restatement of their documented arithmetic (tests/ssm_oracle.forward32 / backward32, the same C library expf and logf): loss_b,
s, w and the norms of the forward, and every per-position contribution of the backward run on identity ids into -0.0 stages.
The backward on the tables themselves (float atomics, any order) is checked against the restatement's contributions summed per
row.  Ragged batch sizes around the group, warp and block widths; M = 1, 2, 31, 32, 33, 256; d = 4, 12, 48, 64, 128; strided
tables and views of interleaved [N, 3, d] tables; duplicate candidates (and candidates equal to the positive); zero rows (the
1e-8 path); tau = 0.02 and others."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import ssm_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'ssm_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'ssm_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _table(rng, n, d, extra, view):
    """(block, offset, stride): n rows of width d; ``view``: view 1 of an interleaved [n, 3, d + extra] block."""
    rs = 3 * (d + extra) if view else d + extra
    off = d + extra if view else 0
    block = (rng.standard_normal((n - 1) * rs + off + d) * rng.choice([0.25, 1.0, 4.0])).astype(np.float32)
    return block, off, rs


def _rows(block, off, rs, ids, d):
    return np.stack([block[off + i * rs: off + i * rs + d] for i in ids.ravel()]).reshape(ids.shape + (d,))


CASES = [  # (B, M, d, extra, view, tau, dup, zero)
    (1, 1, 4, 0, 0, 0.02, False, False), (5, 2, 12, 4, 0, 0.2, True, False), (31, 31, 48, 0, 1, 0.02, False, True),
    (33, 32, 64, 0, 0, 1.0, True, False), (70, 33, 128, 4, 1, 0.02, True, True), (9, 256, 64, 8, 0, 0.02, True, False),
    (37, 256, 4, 0, 1, 0.5, False, True), (65, 1, 128, 0, 0, 0.02, False, False), (257, 2, 12, 0, 1, 0.02, True, True),
    (3, 256, 128, 4, 0, 0.07, True, True), (40, 31, 4, 4, 0, 3, True, False), (17, 33, 48, 8, 1, 0.02, True, True),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'B%d-M%d-d%d-x%d-view%d-tau%g-dup%d-zero%d' % c)
def test_ssm_kernels_match_their_sequential_restatement_on_the_host(emulator, case, tmp_path):
    B, M, d, extra, view, tau, dup, zero = case
    rng = np.random.default_rng(sum(int(v) for v in case[:5]) + 11)
    n_user, n_item = 29, 41 + M
    ub, uo, us = _table(rng, n_user, d, extra, view)
    ib, io, is_ = _table(rng, n_item, d, extra, view)
    if zero:                                         # user 0 and items 0 .. 2 are zero rows: n = sqrt(1e-8)
        for blk, off, rs, n in ((ub, uo, us, 1), (ib, io, is_, 3)):
            for r in range(n):
                blk[off + r * rs: off + r * rs + d] = 0.0
    ancs = rng.integers(0, n_user, B)
    poss = rng.integers(0, n_item, B)
    cands = rng.integers(0, n_item, (B, M))
    if dup:                                          # repeated users, positives and candidates; candidates equal to the positive
        ancs[::2] %= 3
        poss[::3] %= 4
        cands[:, ::2] %= 5
        cands[::4, -1] = poss[::4]
    if zero:
        ancs[::5] = 0
        cands[:, 0] = rng.integers(0, 3, B)
    scale, gscale = np.float32(1 / 3), np.float32(0.75)
    fin, fout = str(tmp_path / 'in.bin'), str(tmp_path / 'out.bin')
    with open(fin, 'wb') as f:
        np.array([B, M, d, ub.size, ib.size, uo, io, us, is_], np.int64).tofile(f)
        np.array([tau, scale, gscale], np.float32).tofile(f)
        ub.tofile(f)
        ib.tofile(f)
        for a in (ancs, poss, cands):
            a.astype(np.int64).tofile(f)
    r = subprocess.run([emulator, fin, fout], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    out = np.fromfile(fout, np.float32)
    Q = M + 1
    sizes = [B, B * Q, B * Q, B * (Q + 1), B * d, B * Q * d, ub.size, ib.size]
    assert out.size == sum(sizes)
    loss, s, w, nrm, su, si, gu, gi = np.split(out, np.cumsum(sizes)[:-1])

    u = _rows(ub, uo, us, ancs, d)
    c = _rows(ib, io, is_, np.concatenate([poss[:, None], cands], 1), d)
    w_loss, w_s, w_w, w_nrm = S.forward32(u, c, tau)
    for name, got, want in (('loss_b', loss, w_loss), ('s', s, w_s), ('w', w, w_w), ('nrm', nrm, w_nrm)):
        assert np.array_equal(got.view(np.uint32), want.ravel().view(np.uint32)), name
    g_u, g_c = S.backward32(u, c, tau, w_s, w_w, w_nrm, scale * gscale)
    # stage positions: users 0 .. B-1; items 0 .. B-1 the positives, then B + b M + j candidate j of pair b
    want_si = np.concatenate([g_c[:, 0], g_c[:, 1:].reshape(B * M, d)])
    assert np.array_equal(su.view(np.uint32), g_u.ravel().view(np.uint32)), 'user stage'
    assert np.array_equal(si.view(np.uint32), want_si.ravel().view(np.uint32)), 'item stage'
    # the atomic backward on the tables: every row's contributions, summed in any order
    sink_u, sink_i = np.zeros(ub.size, np.float64), np.zeros(ib.size, np.float64)
    for b in range(B):
        sink_u[uo + ancs[b] * us + np.arange(d)] += g_u[b]
        for q, item in enumerate([poss[b]] + list(cands[b])):
            sink_i[io + item * is_ + np.arange(d)] += g_c[b, q]
    for name, got, want in (('user sink', gu, sink_u), ('item sink', gi, sink_i)):
        assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), name
    assert np.isfinite(loss).all() and (loss >= -1e-4).all()
