"""Kernel sources executed ON THE HOST.  The tiled score kernel (sslrec_b200/csrc/predict_tile.cuh): the same source the library compiles for
sm_90a, run thread by thread (tests/emu/cuda_emu.h: one pthread per CUDA thread, __syncthreads = barrier) under
AddressSanitizer, against a float64 restatement of lightgcn.py:64 + base_model.py:35-36 and bit for bit against the sequential
fp32 FMA chain the kernel documents.  Every global / shared-memory index the kernel forms is checked at ragged sizes (tiles cut
by n_b and n_item, inner dimensions that are not a multiple of the staging depth, strided tables, repeated users), for the
three mask modes.  The k-means assignment kernel (csrc/kmeans_assign.cuh; warp shuffles and __syncwarp are pthread barriers around an
exchange buffer): the 4-rows-per-round instantiation against the 1-row one BIT FOR BIT (assignments, per-CTA partial sums and counts,
change counter) and against a plain restatement of the Lloyd assignment pass (aug_utils.py:150-155).  No GPU involved."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

#        n_b  n_item dim u_stride i_stride mode(0 none, 1 dense, 2 CSR) seed
CASES = [(1, 1, 4, 4, 4, 0, 1), (1, 1, 4, 4, 4, 2, 1), (130, 300, 64, 64, 64, 1, 3), (130, 300, 64, 64, 64, 2, 4),
         (128, 128, 32, 32, 32, 2, 5), (257, 129, 48, 144, 48, 2, 6), (5, 1000, 128, 128, 128, 1, 7), (129, 257, 36, 36, 108, 2, 8)]


@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'predict_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'predict_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and 'asan' in (r.stderr or '').lower():
        cmd = [c for c in cmd if not c.startswith('-fsanitize')]          # no sanitizer runtime on this box: still check the values
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'b%d_i%d_d%d_m%d' % (c[0], c[1], c[2], c[5]))
def test_predict_tile_kernel_on_the_host(emulator, case):
    r = subprocess.run([emulator] + [str(v) for v in case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'bad=0' in r.stdout, r.stdout[-500:] + '\n' + r.stderr[-2000:]


def _build(tmp_path_factory, src, name):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / name)
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'), os.path.join(ROOT, 'tests', 'emu', src), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and 'asan' in (r.stderr or '').lower():
        r = subprocess.run([c for c in cmd if not c.startswith('-fsanitize')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return exe


@pytest.fixture(scope='module')
def kmeans_emulator(tmp_path_factory):
    return _build(tmp_path_factory, 'kmeans_emu.cpp', 'kmeans_emu')


#              n   dim  K  ctas warps seed
KMEANS_CASES = [(40, 16, 3, 2, 4, 1), (700, 32, 7, 5, 8, 2), (1000, 64, 50, 4, 8, 3), (333, 48, 50, 3, 8, 4), (65, 128, 50, 2, 4, 5), (9, 8, 2, 3, 2, 6)]


@pytest.mark.parametrize('case', KMEANS_CASES, ids=lambda c: 'n%d_d%d_k%d' % c[:3])
def test_kmeans_assign_rows_per_round_is_bit_identical_on_the_host(kmeans_emulator, case):
    r = subprocess.run([kmeans_emulator] + [str(v) for v in case], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'bad=0' in r.stdout, r.stdout[-500:] + '\n' + r.stderr[-2000:]


SEQ_C = r"""
#include <math.h>
void seq_scores(const float *a, const float *b, float *c, int m, int n, int k) {
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j) {
            float s = 0.f;
            for (int q = 0; q < k; ++q) s = fmaf(a[i * k + q], b[j * k + q], s);
            c[i * n + j] = s;
        }
}
"""


def test_reference_score_gemm_is_the_sequential_fma_chain_bit_for_bit(tmp_path):
    """The reference scores with ``pck_user_embeds @ item_embeds.T`` on the CPU (lightgcn.py:64).  For the inner dimensions of this path
    (d <= 128) torch's fp32 GEMM evaluates every score as ONE sequential FMA chain over k -- exactly the order predict_tile_kernel documents
    and the emulator checks bit for bit above.  Hence, on the same embeddings, the tiled kernel's unmasked scores are bit-identical to the
    reference operator's (so is every top-k built from them); the GPU test checks the same equality on the device."""
    import ctypes
    import numpy as np
    import torch
    if shutil.which('gcc') is None:
        pytest.skip('needs gcc')
    src, lib = tmp_path / 'seq.c', tmp_path / 'libseq.so'
    src.write_text(SEQ_C)
    r = subprocess.run(['gcc', '-O2', '-mfma', '-shared', '-fPIC', str(src), '-o', str(lib), '-lm'], capture_output=True, text=True)
    if r.returncode != 0:
        r = subprocess.run(['gcc', '-O2', '-shared', '-fPIC', str(src), '-o', str(lib), '-lm'], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-1000:]
    seq = ctypes.CDLL(str(lib)).seq_scores
    for m, n, k in [(256, 5000, 64), (128, 3000, 32), (64, 1000, 128), (33, 777, 48)]:
        g = torch.Generator().manual_seed(m)
        a = (torch.randn(m, k, generator=g) * 0.1).contiguous()
        b = (torch.randn(n, k, generator=g) * 0.1).contiguous()
        c = np.empty((m, n), np.float32)
        seq(ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr()), ctypes.c_void_p(c.ctypes.data), m, n, k)
        before = torch.get_num_threads()
        try:
            for threads in (1, 4):
                torch.set_num_threads(threads)
                got = (a @ b.T).numpy()
                assert np.array_equal(got.view(np.uint32), c.view(np.uint32)), (m, n, k, threads)
        finally:
            torch.set_num_threads(before)


SPMM_C = r"""
#include <math.h>
void seq_spmm(const int *rowptr, const int *col, const float *val, const float *x, float *y, int n, int d) {
    for (int r = 0; r < n; ++r)
        for (int j = 0; j < d; ++j) {
            float acc = 0.f;
            for (int e = rowptr[r]; e < rowptr[r + 1]; ++e) acc = fmaf(val[e], x[(long)col[e] * d + j], acc);
            y[(long)r * d + j] = acc;
        }
}
"""


def test_reference_spmm_is_a_sequential_fma_chain_in_column_order(tmp_path):
    """``t.spmm(adj, embeds)`` (lightgcn.py:29) on the reference's uncoalesced, column-sorted COO adjacency accumulates an output element as
    ONE sequential FMA chain over the row's entries in ascending column order -- bit for bit.  That is the order of prop_kernel's accumulator
    for a row that is not split (<= 128 entries: acc = fma(w, x, acc) over the CSR row); split rows add segment partials and agree to rounding
    (the GPU tests compare against float64 with tolerances; this test pins what the reference computes)."""
    import ctypes
    import numpy as np
    import torch
    from oracle import cf_oracle as O
    from oracle import inputs
    if shutil.which('gcc') is None:
        pytest.skip('needs gcc')
    src, lib = tmp_path / 'spmm.c', tmp_path / 'libspmm.so'
    src.write_text(SPMM_C)
    r = subprocess.run(['gcc', '-O2', '-mfma', '-shared', '-fPIC', str(src), '-o', str(lib), '-lm'], capture_output=True, text=True)
    if r.returncode != 0:
        r = subprocess.run(['gcc', '-O2', '-shared', '-fPIC', str(src), '-o', str(lib), '-lm'], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-1000:]
    seq = ctypes.CDLL(str(lib)).seq_spmm
    rows, cols = inputs.bipartite_edges(900, 700, 8000, 5)
    adj = O.normalized_adjacency(rows, cols, 900, 700)
    n, d = adj.n, 64
    x = (torch.randn(n, d, generator=torch.Generator().manual_seed(1)) * 0.1).contiguous()
    want = torch.spmm(adj.torch_coo(), x).numpy()
    order = np.lexsort((adj.cols, adj.rows))
    c, v = adj.cols[order].astype(np.int32), adj.vals[order].astype(np.float32)
    rowptr = np.zeros(n + 1, np.int32)
    rowptr[1:] = np.cumsum(np.bincount(adj.rows[order], minlength=n))
    y = np.empty((n, d), np.float32)
    seq(ctypes.c_void_p(rowptr.ctypes.data), ctypes.c_void_p(c.ctypes.data), ctypes.c_void_p(v.ctypes.data), ctypes.c_void_p(x.data_ptr()),
        ctypes.c_void_p(y.ctypes.data), n, d)
    assert np.array_equal(y.view(np.uint32), want.view(np.uint32))


@pytest.fixture(scope='module')
def spmm_exact_emulator(tmp_path_factory):
    return _build(tmp_path_factory, 'spmm_exact_emu.cpp', 'spmm_exact_emu')


#                     rows cols dim x_stride y_stride max_deg seed
SPMM_EXACT_CASES = [(1, 1, 4, 4, 4, 1, 1), (50, 40, 64, 64, 64, 10, 2), (33, 70, 48, 144, 50, 300, 3), (9, 9, 128, 128, 130, 5, 4), (100, 100, 36, 36, 36, 20, 5)]


@pytest.mark.parametrize('case', SPMM_EXACT_CASES, ids=lambda c: 'r%d_d%d' % (c[0], c[2]))
def test_spmm_exact_kernel_on_the_host(spmm_exact_emulator, case):
    """csrc/spmm_exact.cuh (opt-in test.exact_order) against the sequential FMA chain over each CSR row, bit for bit, under ASan: isolated rows, a
    hub row, strided tables, a dim that is not a multiple of the warp."""
    r = subprocess.run([spmm_exact_emulator] + [str(v) for v in case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'bad=0' in r.stdout, r.stdout[-500:] + '\n' + r.stderr[-2000:]
