"""train.deterministic at the kernel level: ssl_scatter_rows_ordered through the C ABI against a sequential float32 restatement of
its contract (bit for bit) and float64, and the four routed loss backwards (BPR, InfoNCE rows, alignment, uniformity):
  * on all-distinct ids the routed launch equals the atomic launch bit for bit, so the per-position contribution c_p is unchanged
    (an InfoNCE term whose e1 and e2 share a sink excepted: there every row takes two contributions, one scatter of [e1; e2]);
  * on a duplicate-heavy batch it equals  sink[r] + (((c_p1 + c_p2) + c_p3) + ...)  built from the c_p of a replay of the batch on
    a table whose rows are the gathered rows (every id distinct, so the atomic launch there is exact);
  * the count-bounded InfoNCE form leaves the rows of dead positions bit-unchanged."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def _L():
    from sslrec_b200._lib import check, lib
    return check, lib


def _s():
    return torch.cuda.current_stream().cuda_stream


def _rand(*shape, gen):
    # several binades and both signs: the order of the adds shows in the last bits
    x = torch.rand(*shape, device='cuda', generator=gen) - 0.5
    return x * torch.pow(2.0, torch.randint(0, 12, shape, device='cuda', generator=gen).float())


def restate(prior: torch.Tensor, ids: torch.Tensor, c: torch.Tensor) -> np.ndarray:
    """sink[r] = sink[r] + (((c_p1 + c_p2) + c_p3) + ...) in float32, sequentially in position order (np.add.at applies its
    updates one after the other; -0.0 is the exact additive identity, so the running sum starts at c_p1 itself)."""
    prior, ids, c = prior.cpu().numpy(), ids.cpu().numpy(), c.cpu().numpy()
    live = ids >= 0
    acc = np.full(prior.shape, -0.0, np.float32)
    np.add.at(acc, ids[live], c[live])
    hit = np.zeros(prior.shape[0], bool)
    hit[ids[live]] = True
    out = prior.copy()
    out[hit] = prior[hit] + acc[hit]
    return out


def f64_bound_ok(got: torch.Tensor, prior: torch.Tensor, ids: torch.Tensor, c: torch.Tensor) -> bool:
    """|got - exact| <= n gamma (|prior| + sum |c_p|) per element, n = the row's positions + 1."""
    prior64, c64, ids = prior.double().cpu(), c.double().cpu(), ids.cpu()
    live = ids >= 0
    exact, mag, cnt = prior64.clone(), prior64.abs(), torch.ones(prior.shape[0], dtype=torch.float64)
    exact.index_add_(0, ids[live], c64[live])
    mag.index_add_(0, ids[live], c64[live].abs())
    cnt.index_add_(0, ids[live], torch.ones(int(live.sum()), dtype=torch.float64))
    return bool(((got.double().cpu() - exact).abs() <= cnt[:, None] * U32 * mag * 1.01).all())


def _ids(pattern, P, N, gen):
    if pattern == 'distinct':
        return torch.randperm(N, device='cuda', generator=gen)[:P]
    if pattern == 'one_id':
        return torch.full((P,), N // 2, dtype=torch.int64, device='cuda')
    if pattern == 'ends':
        return torch.where(torch.rand(P, device='cuda', generator=gen) < 0.5, 0, N - 1).long()
    if pattern == 'dead':
        ids = torch.randint(0, max(1, P // 4), (P,), device='cuda', generator=gen)
        return torch.where(torch.rand(P, device='cuda', generator=gen) < 0.25, -1, ids)
    return torch.randint(0, max(1, P // 8), (P,), device='cuda', generator=gen)


def scatter(stage, ids, sink, stride, order=None):
    check, lib = _L()
    order = torch.argsort(ids, stable=True) if order is None else order
    check(lib.ssl_scatter_rows_ordered(stage.data_ptr(), ids.data_ptr(), order.data_ptr(), ids.numel(), stage.shape[1], sink.data_ptr(),
                                       stride, _s()), 'ssl_scatter_rows_ordered')


# ---- 1. ssl_scatter_rows_ordered through the C ABI ---------------------------------------------------------------

def _abi_cases():
    pats = ('random', 'distinct', 'one_id', 'ends', 'dead')
    out = []
    for i, P in enumerate((0, 1, 31, 33, 4096, 3 * 4096 + 5)):
        for j, d in enumerate((4, 36, 64, 128)):
            k = 4 * i + j
            out.append((P, d, (0, 3, d, 64)[k % 4], k % 2 == 1, pats[k % 5]))
    out += [(4096, 128, 0, True, 'one_id'), (3 * 4096 + 5, 64, 64, True, 'one_id'), (3 * 4096 + 5, 128, 5, False, 'distinct'),
            (33, 4, 0, True, 'ends'), (3 * 4096 + 5, 36, 0, True, 'dead')]
    return out


@pytest.mark.parametrize('P,d,extra,prior,pattern', _abi_cases())
def test_scatter_rows_ordered_matches_sequential_restatement(P, d, extra, prior, pattern):
    gen = torch.Generator(device='cuda').manual_seed(P * 131 + d)
    N, stride = P + 3, d + extra
    ids = _ids(pattern, P, N, gen)
    stage = _rand(P, d, gen=gen)
    sink = _rand(N, stride, gen=gen) if prior else torch.zeros(N, stride, device='cuda')
    before = sink.clone()
    scatter(stage, ids, sink, stride)
    torch.cuda.synchronize()
    want = restate(before[:, :d].contiguous(), ids, stage)
    got = sink[:, :d].cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (np.argwhere(got != want)[:5])
    assert torch.equal(sink[:, d:], before[:, d:])                      # the padding of a strided sink is never touched
    assert f64_bound_ok(sink[:, :d], before[:, :d], ids, stage)


def test_scatter_rows_ordered_rejects_bad_arguments():
    check, lib = _L()
    stage, sink = torch.zeros(8, 32, device='cuda'), torch.zeros(8, 64, device='cuda')
    ids = torch.arange(8, device='cuda')
    p = (stage.data_ptr(), ids.data_ptr(), ids.data_ptr(), sink.data_ptr())
    ok = lambda st, i, o, n, d, sk, stride: lib.ssl_scatter_rows_ordered(st, i, o, n, d, sk, stride, _s())
    assert ok(*p[:3], 8, 32, p[3], 64) == 0
    bad = [(None, p[1], p[2], 8, 32, p[3], 64), (p[0], None, p[2], 8, 32, p[3], 64), (p[0], p[1], None, 8, 32, p[3], 64),
           (p[0], p[1], p[2], 8, 32, None, 64), (p[0], p[1], p[2], 8, 0, p[3], 64), (p[0], p[1], p[2], 8, 129, p[3], 200),
           (p[0], p[1], p[2], 8, 32, p[3], 31), (p[0], p[1], p[2], -1, 32, p[3], 64)]
    for a in bad:
        assert ok(*a) != 0, a
        assert lib.ssl_last_error()
    before = sink.clone()
    assert ok(*p[:3], 0, 32, p[3], 64) == 0                              # no positions: a no-op
    torch.cuda.synchronize()
    assert torch.equal(sink, before)


# ---- 2. the routed loss backwards ---------------------------------------------------------------------------------

@pytest.fixture
def E():
    from sslrec_b200 import engine
    yield engine
    engine.DETERMINISTIC = None


def _rows(E, base, v, n_views, sink, grad_views=None):
    return E.Rows(base, v, n_views, 0, base.shape[0], base.shape[-1], (lambda: sink) if sink is not None else None, grad_views=grad_views)


def _bpr(E, det, U, I, ancs, poss, negs, su, si, g):
    E.DETERMINISTIC = det
    su, si = su.clone(), si.clone()
    users, items = _rows(E, U, 0, 1, su), _rows(E, I, 0, 1, si)
    _, coef = E._bpr_fwd(users, items, ancs, poss, negs)
    E._bpr_bwd(users, items, ancs, poss, negs, coef, g)
    torch.cuda.synchronize()
    return su, si


def _nce(E, det, T, sink, idx, alias, g, live=None):
    """e1 = view 0, e2 = view 1 of T [N, 2, d] (the table, view 1, has no sink); ``alias``: one [N, 1, d] sink for both views."""
    E.DETERMINISTIC = det
    sink = sink.clone()
    gv = 1 if alias else 2
    e1, e2 = _rows(E, T, 0, 2, sink, gv), _rows(E, T, 1, 2, sink, gv)
    table = _rows(E, T, 1, 2, None)
    mean = live is not None
    _, saved = E._nce_fwd(e1, e2, table, idx, idx, 0.2, 1 if mean else 0, mean, 1e-8 if mean else 0.0, live)
    E._nce_bwd(saved, g)
    torch.cuda.synchronize()
    return sink


def _align(E, det, X, Y, ix, iy, sx, sy, g):
    E.DETERMINISTIC = det
    sx, sy = sx.clone(), sy.clone()
    x, y = _rows(E, X, 0, 1, sx), _rows(E, Y, 0, 1, sy)
    _, pack = E._align_fwd(x, y, ix, iy)
    E._align_bwd(pack, g)
    torch.cuda.synchronize()
    return sx, sy


def _uniform(E, det, X, ix, sx, g):
    E.DETERMINISTIC = det
    sx = sx.clone()
    _, pack = E._uniform_fwd(_rows(E, X, 0, 1, sx), ix)
    E._uniform_bwd(pack, g)
    torch.cuda.synchronize()
    return sx


def _setup(d, seed):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    return gen, (lambda *s: torch.randn(*s, device='cuda', generator=gen)), torch.full((), 0.7, device='cuda')


def _dup(B, pool, gen, N):
    """ids of a duplicate-heavy batch: half from a pool of ``pool`` ids, half anywhere in [0, N)"""
    ids = torch.randint(0, N, (B,), device='cuda', generator=gen)
    hot = torch.randint(0, pool, (B,), device='cuda', generator=gen) * 7 % N
    return torch.where(torch.rand(B, device='cuda', generator=gen) < 0.5, hot, ids)


def _eqbits(a, b, what):
    assert torch.equal(a, b), (what, (a - b).abs().max().item())


@pytest.mark.parametrize('d', [32, 64, 128])
def test_routed_bpr(E, d):
    gen, rn, g = _setup(d, d)
    Nu, Ni, B = 5000, 7000, 1024
    U, I, su, si = rn(Nu, d), rn(Ni, d), rn(Nu, d), rn(Ni, d)
    # all-distinct ids: the routed launch is the atomic launch
    ancs = torch.randperm(Nu, device='cuda', generator=gen)[:B]
    it = torch.randperm(Ni, device='cuda', generator=gen)[:2 * B]
    a = _bpr(E, False, U, I, ancs, it[:B], it[B:], su, si, g)
    b = _bpr(E, True, U, I, ancs, it[:B], it[B:], su, si, g)
    _eqbits(a[0], b[0], 'users')
    _eqbits(a[1], b[1], 'items')
    # duplicate-heavy: the restatement from the c_p of the replay on the gathered rows
    ancs, poss, negs = _dup(B, 5, gen, Nu), _dup(B, 5, gen, Ni), _dup(B, 3, gen, Ni)
    got_u, got_i = _bpr(E, True, U, I, ancs, poss, negs, su, si, g)
    ar = torch.arange(B, device='cuda')
    item_ids = torch.cat([poss, negs])
    cu, ci = _bpr(E, False, U[ancs], I[item_ids], ar, ar, ar + B, torch.zeros(B, d, device='cuda'), torch.zeros(2 * B, d, device='cuda'), g)
    assert np.array_equal(got_u.cpu().numpy(), restate(su, ancs, cu))
    assert np.array_equal(got_i.cpu().numpy(), restate(si, item_ids, ci))
    assert f64_bound_ok(got_i, si, item_ids, ci)


@pytest.mark.parametrize('alias', [True, False])
@pytest.mark.parametrize('d', [32, 64])
def test_routed_infonce_rows(E, d, alias):
    gen, rn, g = _setup(d, d + alias)
    N, B = 6000, 1024
    T = rn(N, 2, d)
    sink = rn(N, 1 if alias else 2, d)
    distinct = torch.randperm(N, device='cuda', generator=gen)[:B]
    if not alias:         # aliased sinks take two contributions per row even then: the atomic kernel adds them in its own order
        _eqbits(_nce(E, False, T, sink, distinct, alias, g), _nce(E, True, T, sink, distinct, alias, g), 'distinct')
    for idx in (distinct, _dup(B, 4, gen, N)):
        got = _nce(E, True, T, sink, idx, alias, g)
        # replay: the anchors' rows gathered into a table of B distinct rows, separate sinks for e1 and e2
        Tg = torch.cat([T[idx], T], 0)             # rows 0..B: the gathered anchors (both views); the table rows follow unchanged
        c = _replay_nce(E, Tg, idx.numel(), g, N)
        if alias:
            want = restate(sink[:, 0], torch.cat([idx, idx]), torch.cat([c[:, 0], c[:, 1]]))
            assert np.array_equal(got[:, 0].cpu().numpy(), want)
        else:
            for v in (0, 1):
                assert np.array_equal(got[:, v].cpu().numpy(), restate(sink[:, v].contiguous(), idx, c[:, v].contiguous()))


def _replay_nce(E, Tg, B, g, N, live=None):
    """c_p of both views: the term on anchors = rows [0, B) of Tg (distinct ids) against the same table rows [B, B + N)."""
    E.DETERMINISTIC = False
    sink = torch.zeros(B, 2, Tg.shape[-1], device='cuda')
    base = Tg
    e1 = E.Rows(base, 0, 2, 0, B, Tg.shape[-1], lambda: sink, grad_views=2)
    e2 = E.Rows(base, 1, 2, 0, B, Tg.shape[-1], lambda: sink, grad_views=2)
    table = E.Rows(base, 1, 2, B, N, Tg.shape[-1])
    ar = torch.arange(B, device='cuda')
    mean = live is not None
    _, saved = E._nce_fwd(e1, e2, table, ar, ar, 0.2, 1 if mean else 0, mean, 1e-8 if mean else 0.0, live)
    E._nce_bwd(saved, g)
    torch.cuda.synchronize()
    return sink


@pytest.mark.parametrize('alias', [True, False])
def test_routed_infonce_rows_live_leaves_dead_rows_unchanged(E, alias):
    d, B, N = 64, 1000, 5000
    gen, rn, g = _setup(d, 7 + alias)
    T = rn(N, 2, d)
    sink = rn(N, 1 if alias else 2, d)
    live_n = 613
    idx = _dup(B, 6, gen, N - 1)
    idx[live_n:] = N - 1                      # dead positions: a row no live position addresses (as ssl_unique_ids pads)
    live = torch.full((), live_n, dtype=torch.int64, device='cuda')
    got = _nce(E, True, T, sink, idx, alias, g, live)
    _eqbits(got[N - 1], sink[N - 1], 'dead row')
    c = _replay_nce(E, torch.cat([T[idx], T], 0), B, g, N, live)
    ids = torch.where(torch.arange(B, device='cuda') < live_n, idx, -1)
    if alias:
        want = restate(sink[:, 0], torch.cat([ids, ids]), torch.cat([c[:, 0], c[:, 1]]))
        assert np.array_equal(got[:, 0].cpu().numpy(), want)
    else:
        for v in (0, 1):
            assert np.array_equal(got[:, v].cpu().numpy(), restate(sink[:, v].contiguous(), ids, c[:, v].contiguous()))


@pytest.mark.parametrize('B', [100, 1024])
def test_routed_alignment_and_uniformity(E, B):
    d = 64
    gen, rn, g = _setup(d, B)
    Nu, Ni = 3000, 4000
    X, Y, sx, sy = rn(Nu, d), rn(Ni, d), rn(Nu, d), rn(Ni, d)
    ix, iy = torch.randperm(Nu, device='cuda', generator=gen)[:B], torch.randperm(Ni, device='cuda', generator=gen)[:B]
    for a, b in zip(_align(E, False, X, Y, ix, iy, sx, sy, g), _align(E, True, X, Y, ix, iy, sx, sy, g)):
        _eqbits(a, b, 'align distinct')
    _eqbits(_uniform(E, False, X, ix, sx, g), _uniform(E, True, X, ix, sx, g), 'uniform distinct')
    ix, iy = _dup(B, 4, gen, Nu), _dup(B, 4, gen, Ni)
    gx, gy = _align(E, True, X, Y, ix, iy, sx, sy, g)
    ar = torch.arange(B, device='cuda')
    z = torch.zeros(B, d, device='cuda')
    cx, cy = _align(E, False, X[ix], Y[iy], ar, ar, z, z, g)
    assert np.array_equal(gx.cpu().numpy(), restate(sx, ix, cx))
    assert np.array_equal(gy.cpu().numpy(), restate(sy, iy, cy))
    gu = _uniform(E, True, X, ix, sx, g)
    cu = _uniform(E, False, X[ix], ar, z, g)
    assert np.array_equal(gu.cpu().numpy(), restate(sx, ix, cu))
    # x and y rows of one sink: one scatter over [x positions; y positions]
    XY = torch.cat([X, Y])
    sxy = torch.cat([sx, sy])
    E.DETERMINISTIC = True
    s = sxy.clone()
    x, y = _rows(E, XY, 0, 1, s), _rows(E, XY, 0, 1, s)
    _, pack = E._align_fwd(x, y, ix, iy + Nu)
    E._align_bwd(pack, g)
    torch.cuda.synchronize()
    assert np.array_equal(s.cpu().numpy(), restate(sxy, torch.cat([ix, iy + Nu]), torch.cat([cx, cy])))


def test_rows_at_backward_is_the_ordered_scatter(E):
    d, N, B = 64, 3000, 2048
    gen, rn, _ = _setup(d, 5)
    T = rn(N, d).requires_grad_(True)
    ids = _dup(B, 5, gen, N)
    up = rn(B, d)
    E.DETERMINISTIC = True
    out = E.rows_at(T, ids)
    assert torch.equal(out, T.detach()[ids])
    out.backward(up)
    assert np.array_equal(T.grad.cpu().numpy(), restate(torch.zeros(N, d), ids, up))
