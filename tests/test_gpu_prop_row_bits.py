"""Row-restricted views of the last summed layer (``ssl_prop_args.row_bits``, ``ViewSpec.row_bits``, ``engine.row_bitmap``).

A view the losses read at batch rows only (SimGCL's views 0 and 2, SGL's view 0) is gathered and written at the rows its
bitmap marks.  At marked rows every output is bit-identical to an unrestricted launch, and unrestricted views are
bit-identical everywhere; unmarked rows of a restricted view are never stored.  The graph has split rows on both sides of
``side_split``, marked and unmarked; index lists repeat ids and may be empty.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
from oracle import inputs

pytestmark = pytest.mark.gpu

N_USER, N_ITEM = 3000, 1200


def _graph():
    rows, cols = inputs.bipartite_edges(N_USER, N_ITEM, 30000, 12)
    # split rows: two item hubs (900 and 300 entries) and one user hub (600 entries)
    rows = np.concatenate([rows, np.arange(900) % N_USER, np.arange(300) % N_USER + 5, np.full(600, N_USER - 1)])
    cols = np.concatenate([cols, np.full(900, N_ITEM - 1), np.full(300, N_ITEM - 2), np.arange(600) % N_ITEM])
    return O.normalized_adjacency(rows, cols, N_USER, N_ITEM)


@pytest.fixture(scope='module')
def setup():
    from sslrec_b200.graph import GraphPlan
    adj = _graph()
    plan = GraphPlan(adj.rows, adj.cols, adj.vals, adj.n, torch.device('cuda'), side_split=N_USER)
    assert plan.stats()['split_rows'] >= 3
    e0 = (torch.randn(adj.n, 64, generator=torch.Generator().manual_seed(2)) * 0.1).cuda()
    return adj, plan, e0


def _views(kind, bits):
    from sslrec_b200 import engine as E
    if kind == 'simgcl':
        vs = [E.ViewSpec(noise_mode=1, seed=101), E.ViewSpec(noise_mode=1, seed=102), E.ViewSpec()]
        restrict = (0, 2)
    else:        # SGL-like: per-view edge masks (MODE 2), view 0 restricted
        vs = [E.ViewSpec(edge_mode=1, keep=0.8, scale=1.25, seed=201), E.ViewSpec(edge_mode=1, keep=0.8, scale=1.25, seed=202), E.ViewSpec()]
        restrict = (0,)
    if bits is not None:
        for i in restrict:
            vs[i].row_bits = bits
    return vs, restrict


def _marked(bits, n):
    rows = torch.arange(n, device=bits.device)
    return ((bits.to(torch.int64)[rows >> 5] >> (rows & 31)) & 1).bool()


BATCHES = {
    'hubs': (torch.tensor([N_USER - 1, 7, 7, 7]), torch.tensor([N_ITEM - 1, 3, 3]), torch.tensor([0])),      # marked split rows, duplicates
    'no_hubs': (torch.tensor([10, 11]), torch.tensor([4]), torch.tensor([], dtype=torch.int64)),            # every split row unmarked, empty list
    'items_only': (torch.tensor([], dtype=torch.int64), torch.tensor([N_ITEM - 2, 0]), torch.tensor([N_ITEM - 2])),
    'random': None,
}


def _batch(name):
    if BATCHES[name] is not None:
        return BATCHES[name]
    g = torch.Generator().manual_seed(5)
    return torch.randint(0, N_USER, (512,), generator=g), torch.randint(0, N_ITEM, (512,), generator=g), torch.randint(0, N_ITEM, (512,), generator=g)


@pytest.mark.parametrize('kind', ['simgcl', 'sgl'])
@pytest.mark.parametrize('batch', list(BATCHES))
def test_restricted_views_are_bit_equal_at_marked_rows(setup, kind, batch):
    from sslrec_b200 import engine as E
    adj, plan, e0 = setup
    ancs, poss, negs = _batch(batch)
    bits = E.row_bitmap(adj.n, 'cuda', (ancs, 0), (poss, N_USER), (negs, N_USER))
    marked = _marked(bits, adj.n)
    want = torch.zeros(adj.n, dtype=torch.bool)
    want[ancs] = True
    want[N_USER + poss] = True
    want[N_USER + negs] = True
    assert torch.equal(marked.cpu(), want)
    views, restrict = _views(kind, bits)
    full = E.Propagation(plan, _views(kind, None)[0], 3, noise_eps=0.1).forward(e0, N_USER)
    E.TIMER = E.KernelTimer()
    try:
        st = E.Propagation(plan, views, 3, noise_eps=0.1).forward(e0, N_USER)
        torch.cuda.synchronize()
        meta = [m for name, m, _ in E.TIMER.launches() if name == 'prop_fwd']
    finally:
        E.TIMER = None
    assert st.restricted_views == set(restrict)
    for v in range(3):
        if v in restrict:
            assert torch.equal(st.E[marked, v], full.E[marked, v]), f'view {v} at marked rows'
        else:
            assert torch.equal(st.E[:, v], full.E[:, v]), f'view {v}'
    assert meta[-1]['restricted_views'] == len(restrict) and meta[-1]['gather_views'] < 3
    assert all(m['restricted_views'] == 0 for m in meta[:-1])
    for v in restrict:                        # a restricted view is gathered by index, never read whole
        with pytest.raises(RuntimeError, match='row_bits'):
            st.users(v).dense()
        with pytest.raises(RuntimeError, match='row_bits'):
            E.infonce_loss_sum(st.users(1), st.users(1), st.items(v), torch.zeros(1, dtype=torch.int64, device='cuda'), 0.2)


def _launch_last(plan, views, e0, x_in, out, x_out=None, reduce=False):
    """The last summed layer through the C ABI: sum_out = layer + E0 (a 1-view sum source); returns the status."""
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import lib
    prop = E.Propagation(plan, views, 1, noise_eps=0.1)
    a = prop._args(64, 1, False)
    a.in_views, a.x_in, a.sum_out = 3, x_in.data_ptr(), out.data_ptr()
    a.n_sum_src, a.sum_src[0], a.sum_src_views[0] = 1, e0.data_ptr(), 1
    for i, v in enumerate(views):
        if v.row_bits is not None:
            a.row_bits[i] = v.row_bits.data_ptr()
    if x_out is not None:
        a.x_out = x_out.data_ptr()
    if reduce:
        a.reduce_views = 1
    rc = lib.ssl_propagate_layer(plan.handle, C.byref(a), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def test_unmarked_rows_are_not_stored_and_forbidden_launches_are_rejected(setup):
    from sslrec_b200 import engine as E
    adj, plan, e0 = setup
    ancs, poss, negs = _batch('hubs')
    bits = E.row_bitmap(adj.n, 'cuda', (ancs, 0), (poss, N_USER), (negs, N_USER))
    marked = _marked(bits, adj.n)
    x_in = (torch.randn(adj.n, 3, 64, generator=torch.Generator().manual_seed(3)) * 0.1).cuda()
    views, restrict = _views('simgcl', bits)
    ref = torch.full((adj.n, 3, 64), float('nan'), device='cuda')
    assert _launch_last(plan, _views('simgcl', None)[0], e0, x_in, ref) == 0
    out = torch.full((adj.n, 3, 64), float('nan'), device='cuda')
    assert _launch_last(plan, views, e0, x_in, out) == 0
    for v in range(3):
        if v in restrict:
            assert torch.equal(out[marked, v], ref[marked, v])
            assert torch.isnan(out[~marked, v]).all(), f'view {v} stored at unmarked rows'
        else:
            assert torch.equal(out[:, v], ref[:, v])
    # a restriction with x_out (a layer the next layer reads) or with reduce_views is rejected, nothing is written
    for kw in (dict(x_out=torch.full((adj.n, 3, 64), float('nan'), device='cuda')), dict(reduce=True)):
        out = torch.full((adj.n, 3, 64), float('nan'), device='cuda')
        assert _launch_last(plan, views, e0, x_in, out, **kw) != 0
        assert torch.isnan(out).all()
        if 'x_out' in kw:
            assert torch.isnan(kw['x_out']).all()


def test_graph_replay_with_two_batches_equals_eager(setup):
    from sslrec_b200 import engine as E
    adj, plan, e0 = setup
    batches = [_batch('random'), _batch('hubs')]
    static = [t.clone().cuda() for t in batches[0]]

    def step():
        bits = E.row_bitmap(adj.n, 'cuda', (static[0], 0), (static[1], N_USER), (static[2], N_USER))
        return bits, E.Propagation(plan, _views('simgcl', bits)[0], 3, noise_eps=0.1).forward(e0, N_USER)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        bits_g, st_g = step()
    for b in batches:
        # same shape, new ids: pad the hubs batch to the capture's lengths by repeating its first id
        for dst, src in zip(static, b):
            src = src.cuda() if src.numel() else torch.zeros(1, dtype=torch.int64, device='cuda')
            dst.copy_(src[torch.arange(dst.numel(), device='cuda') % src.numel()])
        g.replay()
        torch.cuda.synchronize()
        bits_e, st_e = step()
        assert torch.equal(bits_g, bits_e)
        marked = _marked(bits_e, adj.n)
        for v in range(3):
            rows = marked if v in (0, 2) else torch.ones_like(marked)
            assert torch.equal(st_g.E[rows, v], st_e.E[rows, v])
