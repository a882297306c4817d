"""The view-linear backward of the propagation (``engine.Propagation.view_linear``).

When no view masks edges or drops nodes, every view's layers are the same linear map Â and the views differ only by the
SimGCL perturbation eps sign(x) û, whose derivative is zero.  The losses then add every view's gradient into one [N, 1, d]
sink and the transposed recursion D_{k-1} = Â^T D_k + sum_v G^v_{k-1} runs as one view.  Checked here:

- dE0 against a float64 per-view recursion (the multi-view form), with keep_layers sinks, the regulariser fold with and
  without a G_e0 sink, split rows, and at the amazon bench shape; the bound is derived from sum |terms|;
- the loss kernels address the shared sink (its row stride is d) -- the gradients of a SimGCL-style loss with BPR, InfoNCE,
  alignment and uniformity terms equal those of the per-view sinks within rounding;
- views with edge masks or node drop keep per-view sinks and V-view backward launches.
"""
import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
from oracle import inputs
import ssl_test_helpers as H

pytestmark = pytest.mark.gpu

TAU, TAU_ABS = 1e-5, 1e-7    # |got - ref| <= TAU * sum |terms| + TAU_ABS
EPS = 0.1                    # noise_eps


def _graph(n_user, n_item, n_edge, seed, hub=0):
    rows, cols = inputs.bipartite_edges(n_user, n_item, n_edge, seed)
    if hub:      # one item connected to `hub` users: a split row (> 128 entries)
        rows = np.concatenate([rows, np.arange(hub) % n_user])
        cols = np.concatenate([cols, np.full(hub, n_item - 1)])
    return O.normalized_adjacency(rows, cols, n_user, n_item)


def _plan(adj, side_split=0, need_rev=False):
    from sslrec_b200.graph import GraphPlan
    return GraphPlan(adj.rows, adj.cols, adj.vals, adj.n, torch.device('cuda'), need_rev=need_rev, side_split=side_split)


def _noise_views():
    from sslrec_b200 import engine as E
    return [E.ViewSpec(noise_mode=1, seed=0x1234_5678_9ABC_DEF1), E.ViewSpec(noise_mode=1, seed=0x0BAD_CAFE_0000_0002), E.ViewSpec()]


def _adj_t(adj):
    """Â^T in float64 on the device."""
    return torch.sparse_coo_tensor(torch.from_numpy(np.stack([adj.cols, adj.rows])), torch.from_numpy(adj.vals.astype(np.float64)),
                                   (adj.n, adj.n)).coalesce().cuda()


def _ref_de0(adj, L, S, w_sum, w_layers, e0, reg_g, g_e0):
    """float64 per view: D^v_L = G^v_L, D^v_{k-1} = Â^T D^v_k + G^v_{k-1} (G^v_k = [k <= S] W_sum^v + W_k^v), summed over the
    views at k = 0 with 2 g E0 + G_e0.  Returns (dE0, the same recursion over |Â|, |W|: the scale of the rounding)."""
    V, at = w_sum.shape[1], _adj_t(adj)
    out, scale = torch.zeros_like(e0, dtype=torch.float64), torch.zeros_like(e0, dtype=torch.float64)
    for absval in (False, True):
        f = (lambda t: t.abs()) if absval else (lambda t: t)
        acc = scale if absval else out
        for v in range(V):
            def g(k):
                t = torch.zeros_like(acc)
                if k <= S:
                    t = t + f(w_sum[:, v].double())
                if k in w_layers:
                    t = t + f(w_layers[k][:, v].double())
                return t
            D = g(L)
            for k in range(L, 0, -1):
                D = torch.sparse.mm(at, D) + g(k - 1)     # Â >= 0, so Â^T |D| is the abs recursion
            acc += D
        if reg_g is not None:
            acc += f(2.0 * reg_g * e0.double())
        if g_e0 is not None:
            acc += f(g_e0.double())
    return out, scale


def _run(adj, plan, n_user, dim, L, S, keep, reg, with_g_e0, seed=3):
    from sslrec_b200 import engine as E
    gen = torch.Generator().manual_seed(seed)
    N = adj.n
    e0 = (torch.randn(N, dim, generator=gen) * 0.1).cuda()
    prop = E.Propagation(plan, _noise_views(), L, sum_layers=S, keep_layers=keep, noise_eps=EPS)
    assert prop.view_linear
    st = prop.forward(e0, n_user)
    V = st.n_views
    w_sum = torch.randn(N, V, dim, generator=gen).cuda()
    w_layers = {k: torch.randn(N, V, dim, generator=gen).cuda() for k in keep}
    # every view's rows address the same sink row, with the sink's own stride
    for v in range(V):
        r = st.all_nodes(v)
        assert r.grad_ptr() == st.g_sum().data_ptr() and r.grad_stride == dim and r.stride == V * dim
        r.grad_dense().add_(w_sum[:, v])
        for k in keep:
            rk = st.all_nodes(v, which=k)
            assert rk.grad_ptr() == st.g_layer(k).data_ptr() and rk.grad_stride == dim
            rk.grad_dense().add_(w_layers[k][:, v])
    assert st.g_sum().shape == (N, 1, dim) and all(st.g_layer(k).shape == (N, 1, dim) for k in keep)
    reg_g = g_e0 = None
    if reg:
        reg_g = 0.37
        st.reg_pending = torch.tensor(reg_g, device='cuda')
    if with_g_e0:
        g_e0 = torch.randn(N, dim, generator=gen).cuda()
        st.g_e0().copy_(g_e0)
    E.TIMER = E.KernelTimer()
    try:
        de0 = prop.backward(st)
        torch.cuda.synchronize()
        bwd = [m for name, m, _ in E.TIMER.launches() if name == 'prop_bwd']
    finally:
        E.TIMER = None
    assert len(bwd) == L and all(m['views'] == 1 and m['gather_views'] == 1 for m in bwd), bwd
    ref, scale = _ref_de0(adj, L, S, w_sum, w_layers, e0, reg_g, g_e0)
    err = (de0.double() - ref).abs()
    bad = err > TAU * scale + TAU_ABS
    assert not bad.any(), f'{int(bad.sum())} of {bad.numel()} off, worst ratio {(err / (scale + 1e-30)).max().item():.3e}'
    return de0


@pytest.mark.parametrize('dim', [64, 32])
@pytest.mark.parametrize('layers', [(3, 3, ()), (3, 2, (1, 3)), (2, 2, (2,))])
@pytest.mark.parametrize('reg', ['none', 'reg', 'reg+g_e0'])
def test_one_view_backward_matches_per_view_recursion(dim, layers, reg):
    adj = _graph(900, 700, 8000, 5, 700)
    plan = _plan(adj)
    assert plan.stats()['split_rows'] >= 1
    L, S, keep = layers
    _run(adj, plan, 900, dim, L, S, keep, reg != 'none', reg == 'reg+g_e0')


def test_one_view_backward_at_the_bench_shape():
    from synth_graphs import named_graph
    rows, cols, U, I = named_graph('amazon', seed=2023)
    adj = O.normalized_adjacency(rows, cols, U, I)
    _run(adj, _plan(adj, side_split=U), U, 64, 3, 3, (), True, False)


def _simgcl_style_grads(plan, adj, n_user, view_linear):
    """Gradients of BPR (view 2) + InfoNCE (views 0 / 1, users and items) + alignment / uniformity (views 0 / 1) + reg, with
    the sinks the propagation picks, or -- ``view_linear`` False -- forced per-view sinks and launches."""
    from sslrec_b200 import engine as E
    gen = torch.Generator().manual_seed(9)
    N, d, B = adj.n, 64, 512
    flat = (torch.randn(N, d, generator=gen) * 0.1).cuda().requires_grad_(True)
    ue, ie = flat[:n_user], flat[n_user:]
    prop = E.Propagation(plan, _noise_views(), 3, noise_eps=EPS)
    assert prop.view_linear
    prop.view_linear = view_linear
    st = E.propagate(prop, ue, ie)
    ancs = torch.randint(0, n_user, (B,), generator=gen).cuda()
    poss = torch.randint(0, N - n_user, (B,), generator=gen).cuda()
    negs = torch.randint(0, N - n_user, (B,), generator=gen).cuda()
    loss = E.bpr_loss_sum(st.users(2), st.items(2), ancs, poss, negs) / B
    loss = loss + E.infonce_loss_sum(st.users(0), st.users(1), st.users(1), ancs, 0.2) / B
    loss = loss + E.infonce_loss_sum(st.items(0), st.items(1), st.items(1), poss, 0.2) / B
    loss = loss + E.alignment_mean(st.users(0), st.users(1), ancs, ancs) + E.uniformity_log_mean(st.items(1), poss)
    loss = loss + 1e-4 * E.table_sumsq(st)
    loss.backward()
    assert st.grad_views == (1 if view_linear else 3)
    return loss.item(), flat.grad.clone()


def test_loss_kernels_write_the_shared_sink():
    adj = _graph(3000, 2000, 30000, 8, 900)
    plan = _plan(adj)
    l1, g1 = _simgcl_style_grads(plan, adj, 3000, True)
    l3, g3 = _simgcl_style_grads(plan, adj, 3000, False)
    assert abs(l1 - l3) <= 1e-6 * abs(l3)             # the forward is the same code
    H.close(g1, g3, 1e-4, 1e-5 * g3.abs().max().item(), 'dE0: shared sink vs per-view sinks')


@pytest.mark.parametrize('kind', ['edge_rng', 'edge_mask', 'node_drop', 'single'])
def test_masked_or_node_dropped_views_keep_per_view_sinks(kind):
    from sslrec_b200 import engine as E
    adj = _graph(900, 700, 8000, 5, 700)
    plan = _plan(adj, need_rev=True)          # an injected mask is read through the rev permutation in the backward
    gen = torch.Generator().manual_seed(4)
    aug = {
        'edge_rng': E.ViewSpec(edge_mode=1, keep=0.5, scale=2.0, seed=77),
        'edge_mask': E.ViewSpec(edge_mode=2, keep=0.5, scale=2.0, edge_masks=(torch.rand(len(adj.vals), generator=gen) < 0.5).to(torch.uint8).cuda()),
        'node_drop': E.ViewSpec(node_mode=2, node_keep=0.5, node_mask=(torch.rand(adj.n, generator=gen) < 0.5).to(torch.uint8).cuda()),
        'single': None,
    }[kind]
    views = [E.ViewSpec()] if aug is None else [aug, E.ViewSpec(), E.ViewSpec()]
    V = len(views)
    prop = E.Propagation(plan, views, 2)
    assert prop.view_linear == (kind == 'single')
    st = prop.forward((torch.randn(adj.n, 32, generator=gen) * 0.1).cuda(), 900)
    assert st.g_sum().shape == (adj.n, V, 32)
    assert st.all_nodes(V - 1).grad_stride == V * 32
    st.g_sum().copy_(torch.randn(adj.n, V, 32, generator=gen).cuda())
    E.TIMER = E.KernelTimer()
    try:
        prop.backward(st)
        torch.cuda.synchronize()
        bwd = [m for name, m, _ in E.TIMER.launches() if name == 'prop_bwd']
    finally:
        E.TIMER = None
    assert bwd and all(m['views'] == V for m in bwd), bwd
