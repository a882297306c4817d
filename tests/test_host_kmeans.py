"""The k-means checks of tests/test_gpu_kmeans.py, on the host: ssl_kmeans_workspace's launch shape (warps per CTA, CTA cap,
rejection) against the shared-memory table, and the bounds of ``kmeans_pass_check``.  A float32 restatement of one Lloyd
pass, with the kernels' row partition and summation order, meets every bound (so they are achievable); four slightly
wrong restatements each miss at least one case (so they are tight enough): the highest id on exact ties, one member
dropped from a cluster, no 1e-6 guard (empty clusters become NaN), and a change counter that counts every row."""
import ctypes as C

import numpy as np
import pytest
import torch

import ssl_test_helpers as H

# (d, the largest K at W = 8, 4, 2, 1): from csrc/kmeans_assign.cuh smem_floats at 4 rows per round and 200 KB
TABLE = [(32, (168, 307, 514, 773)), (64, (84, 154, 259, 391)), (128, (40, 76, 129, 196))]

# (n, d, K): a few CTAs of 8 warps, ragged 4-row tails, one CTA, and the shipped NCL shape at the golden size
CASES = [(333, 20, 33), (1000, 36, 50), (61, 32, 5), (700, 64, 50), (2113, 4, 40), (97, 100, 31)]


def _workspace(n, d, K):
    from sslrec_b200._lib import lib
    n_cta, W = C.c_int32(), C.c_int32()
    rc = lib.ssl_kmeans_workspace(n, d, K, C.byref(n_cta), C.byref(W))
    return rc, n_cta.value, W.value


@pytest.mark.parametrize('d,limits', TABLE)
def test_workspace_warps_follow_the_shared_memory_table(d, limits):
    for W, k_max in zip((8, 4, 2, 1), limits):
        assert H.kmeans_k_limit(d, W) == k_max
        for K in (k_max, k_max + 1):
            rc, n_cta, got_w = _workspace(83761, d, K)
            want = H.kmeans_launch(83761, d, K)
            if K == k_max or W > 1:
                assert rc == 0 and (n_cta, got_w) == want[:2] == (132, W if K == k_max else W // 2), (d, K, rc, n_cta, got_w)
            else:
                assert rc == -1 and want is None, (d, K, rc)          # SSL_E_ARG


@pytest.mark.parametrize('W', [8, 4, 2, 1])
def test_workspace_caps_the_grid_at_one_cta_per_sm(W):
    d = 32
    K = H.kmeans_k_limit(d, W)
    edge = 132 * W * 8
    for n in (1, 31, 33, W * 8, W * 8 + 1, edge - 1, edge, edge + 1, 83761):
        rc, n_cta, got_w = _workspace(n, d, K)
        want = H.kmeans_launch(n, d, K)
        assert rc == 0 and (n_cta, got_w) == want[:2], (n, rc, n_cta, got_w, want)
        n_cta, W_, rpc, rpw = want
        assert n_cta == min(-(-n // (W * 8)), 132) and rpc * n_cta >= n and rpw * W >= rpc
    for n, d, K in [(0, 32, 5), (10, 0, 5), (10, 32, 0), (-1, 32, 5)]:
        assert _workspace(n, d, K)[0] == -1


def lloyd_pass_f32(x, c0, a0, ch0, tie='low', drop=False, eps=True, count_all=False):
    """One Lloyd pass in float32 numpy with the kernels' arithmetic: distances as the chain d2 = fma(t, t, d2), t = x - c (a
    product of floats is exact in double; one rounding per step up to a rare double rounding); the warp slabs summed in row
    order, the CTA partials in warp order, the centroids in CTA order; centroid = sum / (count + 1e-6).  The mutations:
    tie='high' takes the highest id among equal distances, drop=True leaves one member out of its cluster's sum and count,
    eps=False divides by the bare count, count_all=True counts every row as changed."""
    x, c0, a0 = x.numpy(), c0.numpy(), a0.numpy()
    n, d = x.shape
    K = c0.shape[0]
    t = (x[:, None, :] - c0[None]).astype(np.float32)
    d2 = np.zeros((n, K), np.float32)
    for j in range(d):
        d2 = (t[:, :, j].astype(np.float64) ** 2 + d2).astype(np.float32)
    a = d2.argmin(1) if tie == 'low' else K - 1 - d2[:, ::-1].argmin(1)
    n_cta, W, rpc, rpw = H.kmeans_launch(n, d, K)
    cents = np.zeros((K, d), np.float32)
    cnt = np.zeros(K, np.float32)
    dropped = int(np.flatnonzero(np.bincount(a, minlength=K) >= 2)[0]) if drop else -1
    for b in range(n_cta):
        ps, pc = np.zeros((K, d), np.float32), np.zeros(K, np.float32)
        for w in range(W):
            slab, sc = np.zeros((K, d), np.float32), np.zeros(K, np.float32)
            r0 = b * rpc + w * rpw
            for r in range(r0, min(r0 + rpw, (b + 1) * rpc, n)):
                if a[r] == dropped:
                    dropped = -1
                    continue
                slab[a[r]] += x[r]
                sc[a[r]] += 1
            ps += slab
            pc += sc
        cents += ps
        cnt += pc
    with np.errstate(invalid='ignore'):
        cents = cents / (cnt[:, None] + (np.float32(1e-6) if eps else np.float32(0)))
    changed = ch0 + (n if count_all else int((a != a0).sum()))
    return dict(assign=torch.from_numpy(a.astype(np.int64)), cents=torch.from_numpy(cents), counts=torch.from_numpy(cnt),
                changed=changed)


def _check(case, **mutation):
    n, d, K = case
    x, c0, a0 = H.kmeans_case(n, d, K, seed=n + d + K)
    n_cta, W, _, rpw = H.kmeans_launch(n, d, K)
    out = lloyd_pass_f32(x, c0, a0, 11, **mutation)
    return H.kmeans_pass_check(x, c0, a0, 11, out, W, n_cta, rpw)


@pytest.mark.parametrize('case', CASES)
def test_float32_restatement_meets_the_bounds(case):
    n, d, K = case
    x, c0, _ = H.kmeans_case(n, d, K, seed=n + d + K)
    assert len(torch.unique(c0, dim=0)) < K                   # exact ties planted
    r = _check(case)
    assert r['assign'] <= 1.0 and r['cents'] <= 1.0, r


@pytest.mark.parametrize('mutation', [dict(tie='high'), dict(drop=True), dict(eps=False), dict(count_all=True)],
                         ids=['highest-id-on-ties', 'member-dropped', 'no-1e-6-guard', 'counts-every-row'])
def test_wrong_restatements_miss_the_bounds(mutation):
    failed = []
    for case in CASES:
        try:
            _check(case, **mutation)
        except AssertionError as e:
            failed.append((case, str(e).splitlines()[0]))
    assert failed, f'{mutation} passes every case'
