"""NCL's k-means on the GPU (csrc/kmeans_assign.cuh kmeans_assign_kernel<R>, csrc/cluster_sample.cu kmeans_update_kernel and
its C entry points, sslrec_b200/kmeans.py KMeansClustering) against float64 on the device and the reference's clusterings:

A. One Lloyd pass, ssl_kmeans_iter, at every dim class (4, 20, 32, 36, 64, 100, 124, 128: the j += 32 loops with and without a
   partial last step), K = 1, 31, 32, 33, 50 and the largest K of each warp count W = 8, 4, 2, 1, and n = 1, 31, 33, one row
   either side of the 132-CTA cap (132 W 8 +- 1) and 83 761 (amazon's item side: ~80 rows per warp, ragged 4-row rounds),
   with contiguous and row-strided x.  The centroids carry exact ties (duplicated rows across and within a lane, all-zero
   rows).  ``ssl_test_helpers.kmeans_pass_check`` holds the pass to float64: assignments, lowest id on ties, counts,
   centroids, empty clusters exactly 0, the change counter.  Every output buffer has a NaN / sentinel guard tail; both
   rows-per-round instantiations and a second launch must agree bit for bit; the counter is incremented, from three
   starting assignments (a given one, all -1, the result itself).
B. Rejected arguments return SSL_E_ARG and leave every output untouched (the workspace table is tests/test_host_kmeans.py).
C. The Lloyd loop: KMeansClustering from the reference's initial draws reproduces the golden clusterings; the early stop is
   bit-identical to 1000 iterations; the per-iteration counters equal the changes between assignment snapshots; NCL
   clustering for itself matches the golden loss and gradients.

The worst err / bound of each group is printed when the module finishes (visible with pytest -s)."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
from oracle import inputs, replay
import ssl_test_helpers as H

pytestmark = pytest.mark.gpu

NAN = float('nan')
DIMS = (4, 20, 32, 36, 64, 100, 124, 128)
AMAZON_ROWS = 83761
GUARD = 64                       # guard elements after every output buffer
SENT64, SENT32 = -7, -123456     # assign and changed guard values

_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report_worst():
    yield
    if _WORST:
        print('\nworst: ' + ', '.join(f'{k} {v:.3e}' for k, v in sorted(_WORST.items())))


def _note(key, v, lo=False):
    _WORST[key] = (min if lo else max)(_WORST.get(key, v), v)


def _L():
    from sslrec_b200._lib import check, lib
    return lib, check


def _set_rows(rows):
    lib, check = _L()
    check(lib.ssl_set_option(b'kmeans_rows_per_round', rows), 'ssl_set_option')


def _workspace(n, d, K):
    lib, check = _L()
    n_cta, W = C.c_int32(), C.c_int32()
    check(lib.ssl_kmeans_workspace(n, d, K, C.byref(n_cta), C.byref(W)), 'ssl_kmeans_workspace')
    return n_cta.value, W.value


def _x_layout(x, layout):
    """x as passed to the kernel: contiguous, or a row-strided view (stride d + 3) whose gap columns hold NaN."""
    if layout == 'contig':
        return x.contiguous()
    base = torch.full((x.shape[0], x.shape[1] + 3), NAN, device='cuda')
    v = base[:, :x.shape[1]]
    v.copy_(x)
    return v


def _nan(m):
    return torch.full((m,), NAN, device='cuda')


def _iter(x, c0, a_in, ch0, rows=4):
    """One ssl_kmeans_iter on fresh buffers with guard tails -> its outputs; asserts that every guard survived and that
    every partial was written."""
    lib, check = _L()
    n, d = x.shape
    K = c0.shape[0]
    n_cta, _ = _workspace(n, d, K)
    cents = _nan(K * d + GUARD)
    cents[:K * d] = c0.reshape(-1)
    assign = torch.full((n + GUARD,), SENT64, dtype=torch.int64, device='cuda')
    assign[:n] = a_in
    ps, pc, counts = _nan(n_cta * K * d + GUARD), _nan(n_cta * K + GUARD), _nan(K + GUARD)
    changed = torch.full((1 + GUARD,), SENT32, dtype=torch.int32, device='cuda')
    changed[0] = ch0
    _set_rows(rows)
    try:
        rc = lib.ssl_kmeans_iter(x.data_ptr(), x.stride(0), n, d, K, cents.data_ptr(), assign.data_ptr(), ps.data_ptr(),
                                 pc.data_ptr(), counts.data_ptr(), changed.data_ptr(), torch.cuda.current_stream().cuda_stream)
    finally:
        _set_rows(4)
    check(rc, 'ssl_kmeans_iter')
    torch.cuda.synchronize()
    for name, t in (('centroids', cents), ('part_sum', ps), ('part_cnt', pc), ('counts', counts)):
        assert bool(torch.isnan(t[-GUARD:]).all()), f'{name} written past its end'
    assert bool((assign[-GUARD:] == SENT64).all()) and bool((changed[1:] == SENT32).all()), 'assign / changed written past the end'
    assert bool(torch.isfinite(ps[:-GUARD]).all()) and bool(torch.isfinite(pc[:-GUARD]).all()), 'a partial left unwritten'
    return dict(assign=assign[:n], cents=cents[:K * d].view(K, d), counts=counts[:K], changed=int(changed[0]),
                part_sum=ps[:-GUARD], part_cnt=pc[:-GUARD])


def _same(a, b, what, keys=('assign', 'cents', 'counts', 'part_sum', 'part_cnt')):
    for k in keys:
        assert torch.equal(a[k].view(torch.int32) if a[k].dtype == torch.float32 else a[k],
                           b[k].view(torch.int32) if b[k].dtype == torch.float32 else b[k]), f'{what}: {k} differs'


# =====================================================================================================================
# A. one Lloyd pass
# =====================================================================================================================

def _ks(d):
    return sorted({1, 31, 32, 33, 50} | {H.kmeans_k_limit(d, W) for W in (8, 4, 2, 1)})


def _ns(W):
    edge = H.KMEANS_MAX_CTAS * W * 8
    return (1, 31, 33, edge - 1, edge + 1, AMAZON_ROWS)


def _pass_cases():
    out = []
    for d in DIMS:
        for i, K in enumerate(_ks(d)):
            W = H.kmeans_launch(1, d, K)[1]
            for j, n in enumerate(_ns(W)):
                out.append((d, K, n, 'strided' if (i + j) % 2 else 'contig'))
    return out


PASS_CASES = _pass_cases()


def test_pass_matrix_reaches_every_launch_shape():
    """Every warp count with fewer CTAs than SMs, exactly one per SM, and the grid capped (more rows per warp than 8)."""
    def shape(d, K, n):
        W = H.kmeans_launch(n, d, K)[1]
        return W, (-(-n // (W * 8)) > H.KMEANS_MAX_CTAS) - (-(-n // (W * 8)) < H.KMEANS_MAX_CTAS)
    shapes = {shape(d, K, n) for d, K, n, _ in PASS_CASES}
    assert shapes == {(W, grid) for W in (8, 4, 2, 1) for grid in (-1, 0, 1)}
    assert {lay for *_, lay in PASS_CASES} == {'contig', 'strided'}
    for d in DIMS:
        assert {H.kmeans_launch(1, d, K)[1] for K in _ks(d)} == {8, 4, 2, 1}
        assert H.kmeans_launch(1, d, H.kmeans_k_limit(d, 1) + 1) is None


@pytest.mark.parametrize('d,K,n,layout', PASS_CASES, ids=[f'd{d}-K{K}-n{n}-{lay}' for d, K, n, lay in PASS_CASES])
def test_one_lloyd_pass_matches_float64(d, K, n, layout):
    x, c0, given = H.kmeans_case(n, d, K, zlib.crc32(repr((d, K, n)).encode()), 'cuda')
    x = _x_layout(x, layout)
    n_cta, W, _, rpw = H.kmeans_launch(n, d, K)
    assert _workspace(n, d, K) == (n_cta, W)
    out = _iter(x, c0, given, 1000)
    r = H.kmeans_pass_check(x, c0, given, 1000, out, W, n_cta, rpw)
    _note(f'A assign W={W}', r['assign'])
    _note(f'A cents W={W}', r['cents'])
    _same(_iter(x, c0, given, 1000, rows=1), out, 'kmeans_rows_per_round 1 against 4')
    fresh = _iter(x, c0, torch.full((n,), -1, dtype=torch.int64, device='cuda'), 7)
    _same(fresh, out, 'a second launch')
    assert fresh['changed'] == 7 + n, fresh['changed']
    again = _iter(x, c0, out['assign'], 5)
    _same(again, out, 'a launch from its own result')
    assert again['changed'] == 5, again['changed']


# =====================================================================================================================
# B. rejected arguments
# =====================================================================================================================

def test_rejected_arguments_leave_the_outputs_untouched():
    lib, _ = _L()
    n, d = 100, 64
    K_big = H.kmeans_k_limit(d, 1) + 1
    K = 50
    x, c0, given = H.kmeans_case(n, d, K, 3, 'cuda')
    # every buffer sized for the largest K tried, so nothing could be written out of bounds even if a call were accepted
    bufs = dict(cents=torch.rand(K_big * d, device='cuda'), assign=torch.zeros(n, dtype=torch.int64, device='cuda'),
                ps=_nan(H.KMEANS_MAX_CTAS * K_big * d), pc=_nan(H.KMEANS_MAX_CTAS * K_big), counts=_nan(K_big),
                changed=torch.full((1,), 17, dtype=torch.int32, device='cuda'))
    bufs['assign'][:] = given
    before = {k: v.clone() for k, v in bufs.items()}
    ptr = {k: v.data_ptr() for k, v in bufs.items()}
    good = dict(x=x.data_ptr(), stride=d, n=n, d=d, K=K, **ptr)
    calls = {f'null {k}': {k: None} for k in ('x', 'cents', 'assign', 'ps', 'pc', 'counts', 'changed')}
    calls.update({'stride < dim': dict(stride=d - 1), 'n = 0': dict(n=0), 'n < 0': dict(n=-5), 'K = 0': dict(K=0),
                  'dim = 0': dict(d=0, stride=0), f'K = {K_big} at d = {d}': dict(K=K_big)})
    for what, change in calls.items():
        a = dict(good, **change)
        rc = lib.ssl_kmeans_iter(a['x'], a['stride'], a['n'], a['d'], a['K'], a['cents'], a['assign'], a['ps'], a['pc'],
                                 a['counts'], a['changed'], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc == -1 and lib.ssl_last_error(), f'{what}: rc {rc}'           # SSL_E_ARG
        for k, v in bufs.items():
            b = before[k]
            assert torch.equal(v.view(torch.int32) if v.dtype == torch.float32 else v,
                               b.view(torch.int32) if b.dtype == torch.float32 else b), f'{what}: {k} changed'
    n_cta, W = C.c_int32(), C.c_int32()
    assert lib.ssl_kmeans_workspace(n, d, K_big, C.byref(n_cta), C.byref(W)) == -1


# =====================================================================================================================
# C. the Lloyd loop
# =====================================================================================================================

GOLDEN = [(key, size, side) for key, size in (('ncl', 'tiny'), ('ncl_k50', 'small')) for side in ('user', 'item')]


def _golden(key, size):
    g = replay.load_golden(key, size)
    case = inputs.make_case(size)
    adj = O.normalized_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
    return g, case, replay.draws(key, case, g['hp'], adj)


def _drive(x, init, iters):
    """Lloyd iterations through the C ABI as KMeansClustering runs them (one buffer set, one counter per iteration), with a
    snapshot of the centroids and assignment after each -> (list of (centroids, assign) after iteration t, counters)."""
    lib, check = _L()
    n, d = x.shape
    K = init.shape[0]
    n_cta, _ = _workspace(n, d, K)
    cents = init.to('cuda', torch.float32).contiguous().clone()
    ps, pc, counts = torch.empty(n_cta, K, d, device='cuda'), torch.empty(n_cta, K, device='cuda'), torch.zeros(K, 1, device='cuda')
    idx = torch.full((n,), -1, dtype=torch.int64, device='cuda')
    changed = torch.zeros(iters, dtype=torch.int32, device='cuda')
    snaps = []
    s = torch.cuda.current_stream().cuda_stream
    for it in range(iters):
        check(lib.ssl_kmeans_iter(x.data_ptr(), x.stride(0), n, d, K, cents.data_ptr(), idx.data_ptr(), ps.data_ptr(),
                                  pc.data_ptr(), counts.data_ptr(), changed.data_ptr() + 4 * it, s), 'ssl_kmeans_iter')
        snaps.append((cents.clone(), idx.clone(), counts.clone()))
    return snaps, changed


@pytest.mark.parametrize('key,size,side', GOLDEN)
def test_kmeans_reproduces_the_reference_clustering(key, size, side):
    """KMeansClustering (1000 iterations, early stop every 16) from the reference's t.rand draw: the reference's 1000-iteration
    assignment exactly; at the fixed point the centroids are the float64 means of their members within the section-A bound,
    and within that bound plus the reference's own (a sum of count members) of the reference's centroids."""
    from sslrec_b200.kmeans import KMeansClustering
    g, case, dr = _golden(key, size)
    K, d = g['hp']['cluster_num'], case['dim']
    x = case[f'{side}_e'].cuda()
    n = x.shape[0]
    km = KMeansClustering(K, d)
    km.init_centroids = dr[f'init_{side}_centroids']
    cents, idx, cnt = km(x)
    assert km.last_iters < 1000
    want = torch.from_numpy(g[f'{side}2cluster']).cuda()
    assert torch.equal(idx, want), f'{int((idx != want).sum())} of {n} assignments differ from the reference after {km.last_iters} iterations'
    n_cta, W, _, rpw = H.kmeans_launch(n, d, K)
    r = H.kmeans_pass_check(x, cents, idx, 0, dict(assign=idx, cents=cents, counts=cnt, changed=0), W, n_cta, rpw)
    _note('C golden cents', r['cents'])
    more = _iter(x, cents, idx, 0)
    _same(more, dict(assign=idx, cents=cents, counts=cnt.reshape(-1)), 'one more pass', ('assign', 'cents', 'counts'))
    assert more['changed'] == 0
    cnt64 = torch.bincount(idx, minlength=K).double()[:, None]
    A = torch.zeros(K, d, dtype=torch.float64, device='cuda').index_add_(0, idx, x.double().abs())
    den = cnt64 + H.KMEANS_EPS
    bound = (H.gamma(rpw + W + n_cta + 2) + H.gamma(cnt64 + 2)) * A / den
    err = (cents.double() - torch.from_numpy(g[f'{side}_centroids']).cuda().double()).abs()
    assert bool((err <= bound).all()), f'centroids against the reference: max err / bound {(err / bound.clamp_min(1e-300)).max().item():.3e}'
    _note('C golden cents vs reference', float((err / bound.clamp_min(1e-300)).max()))
    empty = cnt64[:, 0] == 0
    print(f'{key}-{size} {side}: {km.last_iters} iterations, {int(empty.sum())} of {K} clusters empty, '
          f'smallest best / second-best gap at the fixed point {r["tie_gap"]:.3e} x its bound')


def _ncl_like(n, d, K, seed):
    """NCL's situation: embeddings of xavier scale around 0, initial centroids t.rand in [0, 1)^d (aug_utils.py:147), so most
    clusters empty in the first pass and the zero centroids they become tie exactly."""
    g = torch.Generator().manual_seed(seed)
    a = float(np.sqrt(6.0 / (n + d)))
    x = (torch.rand(n, d, generator=g) * 2 - 1) * a
    return x.cuda(), torch.rand(K, d, generator=g).cuda()


SEEDED = [(5000, 64, 50, 1), (AMAZON_ROWS, 64, 50, 2), (3001, 20, 33, 3), (1500, 128, 40, 4)]


@pytest.mark.parametrize('n,d,K,seed', SEEDED)
def test_early_stop_is_bit_identical_to_1000_iterations(n, d, K, seed):
    from sslrec_b200.kmeans import KMeansClustering
    x, init = _ncl_like(n, d, K, seed)
    out = {}
    for every in (16, 1001):
        km = KMeansClustering(K, d, iters=1000, check_every=every)
        km.init_centroids = init
        out[every] = [t.clone() for t in km(x)] + [km.last_iters]
    assert 16 < out[16][3] < 1000 and out[1001][3] == 1000, (out[16][3], out[1001][3])
    for a, b, what in zip(out[16][:3], out[1001][:3], ('centroids', 'assignment', 'counts')):
        assert torch.equal(a, b), f'{what} after the early stop at {out[16][3]} differ from 1000 iterations'


@pytest.mark.parametrize('src', [f'{k}-{s}-{side}' for k, s, side in GOLDEN] + [f'seeded-{i}' for i in range(len(SEEDED))])
def test_change_counters_equal_the_snapshot_differences(src):
    """Each iteration's counter equals the rows whose assignment differs from the previous snapshot (all -1 before the first),
    every iteration is a Lloyd pass within the section-A bounds of its incoming centroids, and KMeansClustering stopped at
    the same iteration count gives the same bits."""
    from sslrec_b200.kmeans import KMeansClustering
    kind, *rest = src.split('-')
    if kind == 'seeded':
        n, d, K, seed = SEEDED[int(rest[0])]
        x, init = _ncl_like(min(n, 5000), d, K, seed)
    else:
        key, size, side = kind, rest[0], rest[1]
        g, case, dr = _golden(key, size)
        x, init = case[f'{side}_e'].cuda(), dr[f'init_{side}_centroids'].cuda()
    n, d = x.shape
    K = init.shape[0]
    iters = 40
    snaps, changed = _drive(x, init, iters)
    changed = changed.tolist()
    n_cta, W, _, rpw = H.kmeans_launch(n, d, K)
    prev_c, prev_a = init.float(), torch.full((n,), -1, dtype=torch.int64, device='cuda')
    gaps = []
    for t, (c, a, cnt) in enumerate(snaps):
        assert changed[t] == int((a != prev_a).sum()), (t, changed[t], int((a != prev_a).sum()))
        r = H.kmeans_pass_check(x, prev_c, prev_a, 0, dict(assign=a, cents=c, counts=cnt, changed=changed[t]), W, n_cta, rpw)
        _note('C trajectory assign', r['assign'])
        _note('C trajectory cents', r['cents'])
        gaps.append(r['tie_gap'])
        prev_c, prev_a = c, a
    assert changed[0] == n
    last = next((t + 1 for t in range(iters) if changed[t] == 0), iters)
    km = KMeansClustering(K, d, iters=last, check_every=10 ** 9)
    km.init_centroids = init
    got = km(x)
    for a, b, what in zip(got, snaps[last - 1], ('centroids', 'assignment', 'counts')):
        assert torch.equal(a, b), f'KMeansClustering {what} after {last} iterations differ from the C ABI loop'
    _note('C smallest tie gap / bound', min(gaps), lo=True)
    print(f'{src}: changes per iteration {changed[:last]}; smallest best / second-best gap {min(gaps):.3e} x its bound '
          f'(iteration {int(np.argmin(gaps)) + 1})')


class _PerSide:
    """model.kmeans replaced: the real KMeansClustering, given the reference's initial draw of the side it clusters (user
    first, then item: ncl.py:26-28)."""

    def __init__(self, km, inits):
        self.km, self.inits, self.calls = km, list(inits), 0

    def __call__(self, embeds):
        self.km.init_centroids = self.inits[self.calls]
        self.calls += 1
        return self.km(embeds)


@pytest.mark.parametrize('key,size', [('ncl', 'tiny'), ('ncl_k50', 'small')])
def test_ncl_clusters_for_itself_and_matches_the_reference(key, size):
    g, case, dr = _golden(key, size)
    model, _ = H.make_model(key, case, g['hp'], inject={})
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    model.kmeans = _PerSide(model.kmeans, (dr['init_user_centroids'], dr['init_item_centroids']))
    assert not hasattr(model, 'user2cluster')
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')] + [torch.zeros(case['batch'], dtype=torch.int64).cuda()]
    loss, parts = model.cal_loss(batch)
    assert model.kmeans.calls == 2
    for side in ('user', 'item'):
        assert torch.equal(getattr(model, f'{side}2cluster'), torch.from_numpy(g[f'{side}2cluster']).cuda()), side
    loss.backward()
    H.golden_loss_grads_close(g, loss, parts, model.named_parameters(), f'{key}-{size} ')
