"""Kernel-level parity on the GPU, through the C ABI (ctypes): each kernel against the oracle /
a float64 torch restatement of the same formula on seeded inputs, plus size-independent
properties (adjointness of the masked SpMM, keep fractions, noise norms, determinism)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
from oracle import inputs
import ssl_test_helpers as H

pytestmark = pytest.mark.gpu


def _graph(n_user, n_item, n_edge, seed, hub=0):
    rows, cols = inputs.bipartite_edges(n_user, n_item, n_edge, seed)
    if hub:      # one item connected to `hub` users: exercises the split-row path (> 128 entries)
        extra_u = np.arange(hub) % n_user
        rows = np.concatenate([rows, extra_u])
        cols = np.concatenate([cols, np.full(hub, n_item - 1)])
    return O.normalized_adjacency(rows, cols, n_user, n_item)


def _plan(adj, need_rev=False):
    from sslrec_b200.graph import GraphPlan
    return GraphPlan(adj.rows, adj.cols, adj.vals, adj.n, torch.device('cuda'), need_rev=need_rev)


@pytest.mark.parametrize('dim', [16, 32, 64, 128, 48, 4, 20, 68, 124])
@pytest.mark.parametrize('hub', [0, 700])
def test_propagation_matches_oracle(dim, hub):
    from sslrec_b200 import engine as E
    adj = _graph(900, 700, 8000, 5, hub)
    plan = _plan(adj)
    if hub:
        assert plan.stats()['split_rows'] >= 1
    g = torch.Generator().manual_seed(1)
    e0 = torch.randn(adj.n, dim, generator=g) * 0.1
    for L in (1, 3):
        prop = E.Propagation(plan, [E.ViewSpec()], L)
        st = prop.forward(e0.cuda(), 900)
        ref = O.lightgcn_embeds(adj.torch_coo(torch.float64), e0.double(), L)
        H.close(st.E.view(adj.n, dim), ref, 1e-5, 1e-6, f'E L={L}')
        again = prop.forward(e0.cuda(), 900)
        assert torch.equal(st.E, again.E)              # fixed summation order -> bit-reproducible


def test_three_views_share_layer_one_and_match_single_views():
    """A V-view propagation (3 layers, layer sum) equals V one-view propagations of its views, bit for bit: the three SimGCL
    views (two noisy, one clean) and in general V = 2..4 views at every lane-group dim, with per-view noise (MODE 0 at layer 1,
    MODE 1 after) or mixed per-view edge modes (MODE 2), through the interleaved and the view-major kernel.  The hub row has
    4097 entries: 256-entry segments."""
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import check, lib
    adj = _graph(5000, 400, 20000, 6, 4097)
    plan = _plan(adj)
    assert plan.stats()['max_row_nnz'] == 4097
    g = torch.Generator().manual_seed(2)
    mask = (torch.rand(adj.nnz, generator=g) < 0.5).to(torch.uint8).cuda()
    for dim in (4, 12, 16, 20, 32, 36, 48, 64, 68, 124, 128):
        e0 = (torch.randn(adj.n, dim, generator=g) * 0.1).cuda()
        u = [torch.rand(adj.n, dim, generator=g).cuda() for _ in range(3)]
        noisy = [E.ViewSpec(noise_mode=1, seed=11), E.ViewSpec(noise_mode=1, seed=12), E.ViewSpec(), E.ViewSpec(noise_mode=2, noise_u=u)]
        masked = [E.ViewSpec(edge_mode=1, keep=0.5, scale=2.0, seed=13), E.ViewSpec(noise_mode=1, seed=14),
                  E.ViewSpec(edge_mode=2, keep=0.5, scale=2.0, edge_masks=mask), E.ViewSpec(edge_mode=1, keep=0.8, scale=1.25, seed=15)]
        run = lambda views: E.Propagation(plan, views, 3, noise_eps=0.2).forward(e0, 5000).E
        for views in (noisy, masked):
            for V in (2, 3, 4):
                packed = run(views[:V])
                check(lib.ssl_set_option(b'prop_view_major', 1), 'ssl_set_option')
                try:
                    vm = run(views[:V])
                finally:
                    check(lib.ssl_set_option(b'prop_view_major', 0), 'ssl_set_option')
                assert torch.equal(vm, packed), (dim, V, 'view-major')
                for v in range(V):
                    assert torch.equal(run([views[v]])[:, 0], packed[:, v]), (dim, V, v)


def test_injected_noise_matches_oracle_and_rng_noise_has_norm_eps():
    from sslrec_b200 import engine as E
    adj = _graph(300, 200, 3000, 7)
    plan = _plan(adj)
    g = torch.Generator().manual_seed(3)
    e0 = torch.randn(adj.n, 32, generator=g) * 0.1
    us = [torch.rand(adj.n, 32, generator=g) for _ in range(2)]
    st = E.Propagation(plan, [E.ViewSpec(noise_mode=2, noise_u=[u.cuda() for u in us])], 2, noise_eps=0.9).forward(e0.cuda(), 300)
    ref = O.simgcl_embeds(adj.torch_coo(torch.float64), e0.double(), 2, 0.9, [u.double() for u in us])
    H.close(st.E.view(adj.n, 32), ref, 1e-5, 1e-6, 'perturbed E')
    # RNG noise: x_out - A x has row norm eps wherever no entry of the clean output is exactly 0
    clean = E.Propagation(plan, [E.ViewSpec()], 1, sum_layers=1, keep_layers=(1,)).forward(e0.cuda(), 300).layers[1]
    noisy = E.Propagation(plan, [E.ViewSpec(noise_mode=1, seed=99)], 1, sum_layers=1, keep_layers=(1,), noise_eps=0.9).forward(e0.cuda(), 300).layers[1]
    diff = (noisy - clean).view(adj.n, 32)
    full = (clean.view(adj.n, 32) != 0).all(1)
    norms = diff[full].norm(dim=1)
    assert full.sum() > 100 and torch.allclose(norms, torch.full_like(norms, 0.9), rtol=1e-4)
    assert (torch.sign(diff[full]) == torch.sign(clean.view(adj.n, 32)[full])).all()       # noise follows sign(X)
    assert (diff[~full][clean.view(adj.n, 32)[~full] == 0] == 0).all()


@pytest.mark.parametrize('mode', ['rng', 'injected'])
def test_masked_spmm_is_adjoint_of_its_transpose(mode):
    """<A_m x, y> == <x, A_m^T y> with the edge mask evaluated in-kernel: the backward kernel
    (transpose = 1, key swapped / rev-indexed) is the exact transpose of the forward one."""
    from sslrec_b200 import engine as E
    adj = _graph(800, 600, 9000, 8, 400)
    plan = _plan(adj, need_rev=True)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(adj.n, 64, generator=g).cuda()
    y = torch.randn(adj.n, 64, generator=g).cuda()
    keep = 0.5
    if mode == 'rng':
        view = E.ViewSpec(edge_mode=1, keep=keep, scale=2.0, seed=1234)
    else:
        m = (torch.rand(adj.nnz, generator=g) < keep).to(torch.uint8).cuda()
        view = E.ViewSpec(edge_mode=2, keep=keep, scale=2.0, edge_masks=m)
    prop = E.Propagation(plan, [view], 1)

    def apply(v, transpose):
        a = prop._args(64, 1, transpose)
        out = torch.empty(adj.n, 1, 64, device='cuda')
        a.in_views, a.x_in, a.x_out = 1, v.data_ptr(), out.data_ptr()
        prop._launch(a, v)
        return out.view(adj.n, 64)
    ax, aty = apply(x, False), apply(y, True)
    lhs, rhs = (ax.double() * y.double()).sum().item(), (x.double() * aty.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-6 * max(abs(lhs), 1.0)
    # keep fraction of the RNG mask ~ keep, and it is asymmetric (each directed entry drawn independently)
    ones = torch.ones(adj.n, 64, device='cuda')
    kept = apply(ones, False)[:, 0].double().sum().item() / (2.0 * float(adj.vals.astype(np.float64).sum()))
    assert abs(kept - keep) < 0.02
    if mode == 'injected':
        ref = torch.spmm(O.edge_dropped(adj, m.cpu().numpy().astype(bool), keep, True, torch.float64), x.cpu().double())
        H.close(ax, ref, 1e-5, 1e-6, 'injected-mask SpMM')


def test_node_drop_forward_backward():
    from sslrec_b200 import engine as E
    adj = _graph(300, 200, 3000, 9)
    plan = _plan(adj)
    g = torch.Generator().manual_seed(5)
    e0 = torch.randn(adj.n, 32, generator=g) * 0.1
    mask = (torch.rand(adj.n, generator=g) < 0.5)
    view = E.ViewSpec(node_mode=2, node_keep=0.5, node_mask=mask.to(torch.uint8).cuda())
    prop = E.Propagation(plan, [view, E.ViewSpec()], 2)
    st = prop.forward(e0.cuda(), 300)
    a_t = adj.torch_coo(torch.float64)
    ref0 = O.lightgcn_embeds(a_t, O.node_dropped(e0.double(), mask), 2)
    ref1 = O.lightgcn_embeds(a_t, e0.double(), 2)
    H.close(st.E[:, 0, :], ref0, 1e-5, 1e-6, 'node-dropped view')
    H.close(st.E[:, 1, :], ref1, 1e-5, 1e-6, 'clean view')
    # backward: d/dE0 of sum(E * W)
    w = torch.randn(adj.n, 2, 32, generator=g)
    st.g_sum().copy_(w.cuda())
    de0 = prop.backward(st)
    e0r = e0.double().clone().requires_grad_(True)
    tot = (O.lightgcn_embeds(a_t, O.node_dropped(e0r, mask), 2) * w[:, 0].double()).sum() + (O.lightgcn_embeds(a_t, e0r, 2) * w[:, 1].double()).sum()
    tot.backward()
    H.close(de0, e0r.grad, 1e-5, 1e-5, 'dE0 with node drop')


@pytest.mark.parametrize('use_tc', [True, False])
@pytest.mark.parametrize('dim,B,n', [(64, 4096, 9000), (32, 100, 777), (128, 300, 2000), (48, 257, 1000), (64, 64, 50), (64, 130, 64 * 9 + 1)])
def test_infonce_term_forward_backward(dim, B, n, use_tc, monkeypatch):
    """use_tc: the tensor-core contraction at dims 32 / 64 (3xFP16 at tau = 0.2, offset 7.2) vs the FP32-FMA kernel -- same
    tolerances."""
    from sslrec_b200 import engine
    from sslrec_b200 import loss_utils as LU
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', use_tc)
    g = torch.Generator().manual_seed(6)
    e1 = torch.randn(B, dim, generator=g)
    e2 = torch.randn(B, dim, generator=g)
    tab = torch.randn(n, dim, generator=g)
    tau = 0.2
    ins = [t.clone().cuda().requires_grad_(True) for t in (e1, e2, tab)]
    loss = LU.cal_infonce_loss(*ins, tau)
    loss.backward()
    ref_in = [t.double().clone().requires_grad_(True) for t in (e1, e2, tab)]
    ref = O.infonce_loss_sum(*ref_in, tau)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 2e-6 * abs(ref.item())
    # absolute term relative to the largest gradient entry: 2e-6 for the FP32-FMA kernel; 1e-5 for the tensor-core
    # 3xTF32 kernel, whose tensor-core accumulators do not round to nearest over up to ~10^3 accumulations per output
    rel_atol = 1e-5 if (use_tc and dim in (32, 64)) else 2e-6
    for a, b, name in zip(ins, ref_in, ('e1', 'e2', 'table')):
        H.close(a.grad, b.grad, 2e-4, rel_atol * b.grad.abs().max().item(), 'grad ' + name)


def test_spec_nodes_infonce_and_bpr_dense():
    from sslrec_b200 import loss_utils as LU
    g = torch.Generator().manual_seed(7)
    e1, e2 = torch.randn(500, 32, generator=g), torch.randn(500, 32, generator=g)
    nodes = torch.unique(torch.randint(0, 500, (200,), generator=g))
    a = e2.clone().cuda().requires_grad_(True)
    loss = LU.cal_infonce_loss_spec_nodes(e1.cuda(), a, nodes.cuda(), 0.1)
    loss.backward()
    b = e2.double().clone().requires_grad_(True)
    ref = O.infonce_spec_nodes_mean(e1.double(), b, nodes, 0.1)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 2e-6 * abs(ref.item()) + 1e-6
    H.close(a.grad, b.grad, 2e-4, 2e-6 * b.grad.abs().max().item(), 'spec-nodes grad')
    anc, pos, neg = (torch.randn(300, 64, generator=g) for _ in range(3))
    ins = [t.clone().cuda().requires_grad_(True) for t in (anc, pos, neg)]
    l = LU.cal_bpr_loss(*ins)
    l.backward()
    rin = [t.double().clone().requires_grad_(True) for t in (anc, pos, neg)]
    r = O.bpr_loss_sum(*rin)
    r.backward()
    assert abs(l.item() - r.item()) <= 2e-6 * abs(r.item())
    for x, y in zip(ins, rin):
        H.close(x.grad, y.grad, 1e-5, 1e-6, 'bpr grad')


def _predict_case(n_b, n_item, dim, view, mode, dev):
    """Seeded inputs of one ssl_predict_mask call: (user table view, item table, users, dense mask | None, rowptr | None, cols | None,
    float64 scores, bool positions that must read -1e8)."""
    g = torch.Generator().manual_seed(11)
    n_user = n_b // 2 + 3                                      # users repeat inside the batch
    V = 3 if view else 1
    ubase = (torch.randn(n_user, V, dim, generator=g) * 0.2).to(dev)
    ibase = (torch.randn(n_item, dim, generator=g) * 0.2).to(dev)
    ut = ubase[:, V - 1, :]                                    # view: the last view of an interleaved [n, 3, d] table (row stride 3 d)
    users = torch.randint(0, n_user, (n_b,), generator=g)
    keep = torch.rand(n_user, n_item, generator=g) < 0.2       # the users' training positives
    mask = rowptr = cols = None
    if mode == 'dense':
        mask = keep[users].long().contiguous().to(dev)
    elif mode == 'csr':
        rowptr = torch.cat([torch.zeros(1, dtype=torch.long), keep.sum(1).cumsum(0)]).int().to(dev)
        cols = keep.nonzero()[:, 1].int()                      # row-major: ascending inside a row
        cols = (cols if cols.numel() else torch.zeros(1, dtype=torch.int32)).to(dev)
    ref = ut.cpu().double()[users] @ ibase.cpu().double().T
    masked = keep[users] if mode != 'none' else torch.zeros(n_b, n_item, dtype=torch.bool)
    return ut, ibase, users.to(dev), mask, rowptr, cols, ref, masked


@pytest.mark.parametrize('n_b,n_item,dim,view', [(1, 1, 4, False), (130, 300, 64, False), (257, 1029, 48, True), (1024, 5003, 128, False)])
@pytest.mark.parametrize('mode', ['none', 'dense', 'csr'])
def test_predict_tiled_kernel_matches_float64_and_the_warp_kernel(n_b, n_item, dim, view, mode):
    """ssl_predict_mask through both of its kernels (the 128 x 128 tiled product, default, and the round-1 warp-per-item kernel,
    ssl_set_option("predict_tiled", 0)): scores against float64, masked positions exactly -1e8, ragged tiles, strided table view."""
    from sslrec_b200._lib import check, lib
    dev = torch.device('cuda')
    ut, ibase, users, mask, rowptr, cols, ref, masked = _predict_case(n_b, n_item, dim, view, mode, dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def run(tiled):
        preds = torch.full((n_b, n_item), -7.0, device=dev)
        check(lib.ssl_set_option(b'predict_tiled', int(tiled)), 'ssl_set_option')
        try:
            check(lib.ssl_predict_mask(ut.data_ptr(), ut.stride(0), ibase.data_ptr(), ibase.stride(0), users.data_ptr(), n_b, n_item, dim,
                                       None if mask is None else mask.data_ptr(), None if rowptr is None else rowptr.data_ptr(),
                                       None if cols is None else cols.data_ptr(), preds.data_ptr(), stream), 'ssl_predict_mask')
        finally:
            check(lib.ssl_set_option(b'predict_tiled', 1), 'ssl_set_option')
        torch.cuda.synchronize()
        return preds.cpu()

    tiled = run(True)
    for name, got in (('tiled', tiled), ('warp', run(False))):
        assert torch.equal(got[masked], torch.full_like(got[masked], -1e8)), name
        err = (got[~masked].double() - ref[~masked]).abs().max().item() if (~masked).any() else 0.0
        assert err <= 5e-6, (name, err)
    if n_b <= 300 and mode == 'none':
        # the tiled kernel's documented order: one sequential fp32 FMA chain over k -- which is also how the reference's CPU GEMM evaluates a
        # score (tests/test_host_emulation.py).  Restated here in float64 (a * b is exact, one extra rounding to double per step: a handful of
        # last-bit differences in a million scores at most); printed next to it: equality with this box's own torch CPU matmul.
        a, b = ut.cpu()[users.cpu()], ibase.cpu()
        s = torch.zeros(n_b, n_item, dtype=torch.float64)
        for q in range(dim):
            s = (a[:, q:q + 1].double() * b[:, q].double().unsqueeze(0) + s).float().double()
        chain = (tiled == s.float()).float().mean().item()
        gemm = (tiled == (a @ b.T)).float().mean().item()
        print(f'tiled scores bit-equal to the sequential FMA chain: {chain:.6f}; to torch CPU matmul on this host: {gemm:.6f}')
        assert chain >= 0.9999, chain


def test_topk_exact_with_ties():
    from sslrec_b200.trainer import topk
    g = torch.Generator().manual_seed(8)
    p = torch.randn(37, 5003, generator=g)
    p[:, 100:140] = 0.5                      # a run of ties
    p[3, :] = -1e8                           # fully masked row
    p[5, 17] = float('inf')
    idx, val = topk(p.cuda(), 40, return_values=True)
    tv, _ = torch.topk(p, 40)
    assert torch.equal(val.cpu(), tv)
    # ties resolve to the lower index, and every returned index carries the returned value
    assert torch.equal(p.gather(1, idx.cpu()), val.cpu())
    srt = torch.sort(torch.stack([-p[0], torch.arange(5003).float()], 1)[:, 0], stable=True).indices[:40]
    assert torch.equal(idx[0].cpu(), srt)


def test_adam_matches_torch():
    from sslrec_b200.optim import FusedAdam
    g = torch.Generator().manual_seed(9)
    w = torch.randn(1003, 33, generator=g)
    a = torch.nn.Parameter(w.clone().cuda())
    b = torch.nn.Parameter(w.clone())
    oa, ob = FusedAdam([a], lr=1e-3, weight_decay=1e-4), torch.optim.Adam([b], lr=1e-3, weight_decay=1e-4)
    for _ in range(4):
        gr = torch.randn(1003, 33, generator=g)
        a.grad, b.grad = gr.cuda(), gr.clone()
        oa.step(); ob.step()
    H.close(a, b, 1e-6, 1e-7, 'adam params')
    H.close(oa.state[a]['exp_avg_sq'], ob.state[b]['exp_avg_sq'], 1e-6, 1e-12, 'adam v')


def test_c_abi_rejects_bad_arguments():
    from sslrec_b200 import _lib
    rc = _lib.lib.ssl_sumsq(None, 4, None, None)
    assert rc == -1 and b'null' in _lib.lib.ssl_last_error()
    x = torch.zeros(8, device='cuda')
    rc = _lib.lib.ssl_rows_normalize(x.data_ptr(), 6, None, 1, 6, 0, 1.0, x.data_ptr(), None, None, None, None, None, None, 0, None)
    assert rc == -1                                               # dim must be a multiple of 4


# ---------------------------------------------------------------------------------------------------
# in-kernel counter-based draws, bit for bit against their numpy restatement (oracle/philox.py)
# ---------------------------------------------------------------------------------------------------

def _apply_layer(prop, plan_n, dim, v, transpose, layer=1):
    a = prop._args(dim, layer, transpose)
    out = torch.empty(plan_n, 1, dim, device='cuda')
    a.in_views, a.x_in, a.x_out = 1, v.data_ptr(), out.data_ptr()
    prop._launch(a, v)
    return out.view(plan_n, dim)


@pytest.mark.parametrize('keep', [0.5, 0.9])
def test_rng_edge_mask_equals_numpy_philox_mask(keep):
    """edge_mode 1 (keep test evaluated in-kernel from Philox(seed; row, col, stream)) gives exactly the SpMM of
    edge_mode 2 with the mask computed on the host from the same generator, forward and transposed."""
    from oracle import philox as P
    from sslrec_b200 import engine as E
    adj = _graph(800, 600, 9000, 18, 400)
    plan = _plan(adj, need_rev=True)
    seed = 0x1234_5678_9ABC_DEF1
    mask = P.edge_keep(seed, 0, adj.rows, adj.cols, keep)
    assert abs(mask.mean() - keep) < 0.02
    x = torch.randn(adj.n, 64, generator=torch.Generator().manual_seed(14)).cuda()
    rng = E.Propagation(plan, [E.ViewSpec(edge_mode=1, keep=keep, scale=1.0 / keep, seed=seed)], 1)
    inj = E.Propagation(plan, [E.ViewSpec(edge_mode=2, keep=keep, scale=1.0 / keep,
                                          edge_masks=torch.from_numpy(mask.astype(np.uint8)).cuda())], 1)
    for transpose in (False, True):
        assert torch.equal(_apply_layer(rng, adj.n, 64, x, transpose), _apply_layer(inj, adj.n, 64, x, transpose)), transpose
    # per-layer masks (HCCF) are keyed by the layer number
    mask2 = P.edge_keep(seed, 2, adj.rows, adj.cols, keep)
    rng2 = E.Propagation(plan, [E.ViewSpec(edge_mode=1, keep=keep, scale=1.0, seed=seed, per_layer_edges=True)], 2)
    inj2 = E.Propagation(plan, [E.ViewSpec(edge_mode=2, keep=keep, scale=1.0, edge_masks=[None, torch.from_numpy(mask2.astype(np.uint8)).cuda()])], 2)
    assert torch.equal(_apply_layer(rng2, adj.n, 64, x, False, layer=2), _apply_layer(inj2, adj.n, 64, x, False, layer=2))


def test_rng_noise_and_node_masks_equal_numpy_philox():
    from oracle import philox as P
    from sslrec_b200 import engine as E
    adj = _graph(300, 200, 3000, 19)
    plan = _plan(adj)
    seed, dim, L = 987654321012345, 48, 2
    e0 = (torch.randn(adj.n, dim, generator=torch.Generator().manual_seed(15)) * 0.1).cuda()
    us = [torch.from_numpy(P.noise_uniform(seed, layer, adj.n, dim)).cuda() for layer in range(1, L + 1)]
    assert 0.45 < float(us[0].mean()) < 0.55 and float(us[0].max()) < 1.0
    rng = E.Propagation(plan, [E.ViewSpec(noise_mode=1, seed=seed)], L, noise_eps=0.3).forward(e0, 300)
    inj = E.Propagation(plan, [E.ViewSpec(noise_mode=2, noise_u=us)], L, noise_eps=0.3).forward(e0, 300)
    assert torch.equal(rng.E, inj.E)
    nm = P.node_keep(seed, np.arange(adj.n), 0.7)
    assert abs(nm.mean() - 0.7) < 0.06
    rng = E.Propagation(plan, [E.ViewSpec(node_mode=1, node_keep=0.7, seed=seed)], L).forward(e0, 300)
    inj = E.Propagation(plan, [E.ViewSpec(node_mode=2, node_keep=0.7, node_mask=torch.from_numpy(nm.astype(np.uint8)).cuda())], L).forward(e0, 300)
    assert torch.equal(rng.E, inj.E)


@pytest.mark.parametrize('n_user,n_item,n_edge', [(300, 200, 3000), (50, 12, 400), (2000, 3000, 60000)])
def test_negative_sampler_bit_exact_and_valid(n_user, n_item, n_edge):
    """ssl_sample_negs == the numpy restatement on the same Philox draws; no negative is a training positive;
    different epochs redraw; the draw is uniform over the items."""
    import scipy.sparse as sp
    from oracle import philox as P
    from sslrec_b200.data_handler import DeviceLoader, DeviceTrnData
    rows, cols = inputs.bipartite_edges(n_user, n_item, n_edge, 21)
    mat = sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    ds = DeviceTrnData(mat, 'cuda', seed=77)
    csr = sp.csr_matrix(mat)
    csr.sort_indices()
    pos = set(zip(rows.tolist(), cols.tolist()))
    got = []
    for epoch in range(2):
        ds.sample_negs()
        negs = ds.negs.cpu().numpy()
        want = P.sample_negs(mat.row, csr.indptr, csr.indices, n_item, 77, epoch)
        assert np.array_equal(negs, want), epoch
        assert negs.min() >= 0 and negs.max() < n_item
        assert not any((int(u), int(j)) in pos for u, j in zip(mat.row, negs))
        got.append(negs)
    assert (got[0] != got[1]).mean() > 0.5
    if n_edge >= 60000:            # uniform over the items the user has NOT interacted with: chi-square against the exact expectation
        deg = np.diff(csr.indptr).astype(np.float64)
        w = deg / (n_item - deg)                                   # pairs of user u x probability of each admissible item
        exp = w.sum() - np.bincount(csr.indices, weights=np.repeat(w, np.diff(csr.indptr)), minlength=n_item)
        cnt = np.bincount(got[0], minlength=n_item).astype(np.float64)
        ok = exp >= 5
        chi2, dof = ((cnt[ok] - exp[ok]) ** 2 / exp[ok]).sum(), int(ok.sum())
        assert dof > 1000 and chi2 < dof + 6 * math.sqrt(2 * dof), (chi2, dof)
    # one epoch of the device loader serves every pair exactly once, with its negative
    loader = DeviceLoader(ds, 256, seed=5)
    seen = torch.cat([torch.stack(b[:3], 1) for b in loader]).cpu().numpy()
    assert len(loader) == (len(rows) + 255) // 256 and seen.shape == (len(rows), 3)
    order = np.lexsort((seen[:, 1], seen[:, 0]))
    ref = np.stack([mat.row, mat.col, got[1]], 1)
    assert np.array_equal(seen[order], ref[np.lexsort((ref[:, 1], ref[:, 0]))])
    # NCL's epoch flag (datasets_general_cf.py:35-44): the very first sample served, then pair 0 every epoch_period visits
    fl = DeviceTrnData(mat, 'cuda', seed=77, epoch_period=2)
    fl_loader = DeviceLoader(fl, 256, seed=6)
    sums = []
    for epoch in range(4):
        fl.sample_negs()
        batches = list(fl_loader)
        assert all(len(b) == 4 for b in batches)
        flags, pairs = torch.cat([b[3] for b in batches]), torch.cat([torch.stack(b[:2], 1) for b in batches])
        sums.append(int(flags.sum()))
        if epoch == 1:
            assert pairs[flags.bool()].cpu().tolist() == [[int(mat.row[0]), int(mat.col[0])]]
    assert sums == [1, 1, 0, 1]
    # two data-parallel ranks split the same permutation without overlap
    parts = [torch.cat([torch.stack(b[:2], 1) for b in DeviceLoader(ds, 256, rank=r, world=2, seed=9)]) for r in range(2)]
    both = torch.cat(parts).cpu().numpy()
    assert len(np.unique(both[:, 0] * n_item + both[:, 1])) == len(rows) and abs(len(parts[0]) - len(parts[1])) == 0


@pytest.mark.parametrize('n,dim,K', [(5000, 64, 50), (701, 32, 7), (3001, 128, 50), (41, 16, 3)])
def test_kmeans_rows_per_round_is_bit_identical(n, dim, K):
    """kmeans_assign_kernel<4> (default) and <1> (ssl_set_option("kmeans_rows_per_round", 1)): same centroids, assignments and counts, bit for bit."""
    from sslrec_b200._lib import check, lib
    from sslrec_b200.kmeans import KMeansClustering
    g = torch.Generator().manual_seed(31)
    x = torch.rand(n, dim, generator=g).cuda()
    init = torch.rand(K, dim, generator=g)
    out = {}
    for rows in (4, 1):
        check(lib.ssl_set_option(b'kmeans_rows_per_round', rows), 'ssl_set_option')
        try:
            km = KMeansClustering(K, dim, iters=12, check_every=100)
            km.init_centroids = init
            out[rows] = [t.clone() for t in km(x)]
        finally:
            check(lib.ssl_set_option(b'kmeans_rows_per_round', 4), 'ssl_set_option')
    for a, b in zip(out[4], out[1]):
        assert torch.equal(a, b)


@pytest.mark.parametrize('n,dim,K', [(5000, 64, 50), (700, 32, 7), (3000, 128, 50), (40, 16, 3)])
def test_kmeans_matches_oracle_and_is_deterministic(n, dim, K):
    from sslrec_b200.kmeans import KMeansClustering
    g = torch.Generator().manual_seed(23)
    centers = torch.randn(K, dim, generator=g)
    x = centers[torch.randint(0, K, (n,), generator=g)] * 0.5 + 0.1 * torch.randn(n, dim, generator=g)
    init = torch.rand(K, dim, generator=g)
    km = KMeansClustering(K, dim, iters=64, check_every=4)
    km.init_centroids = init
    cents, idx, cnt = km(x.cuda())
    ref_c, ref_i, ref_n = O.kmeans(x.double(), init.double(), iters=km.last_iters)
    agree = (idx.cpu() == ref_i).double().mean().item()
    assert agree >= 0.999, agree                       # fp32 vs fp64 distances may flip a near-tie
    if agree == 1.0:
        H.close(cents, ref_c, 1e-5, 1e-6, 'centroids')
        assert torch.equal(cnt.cpu().double(), ref_n)
    assert int(cnt.sum().item()) == n and cnt.shape == (K, 1) and idx.dtype == torch.int64
    c2, i2, n2 = km(x.cuda())
    assert torch.equal(c2, cents) and torch.equal(i2, idx) and torch.equal(n2, cnt)     # no floating-point atomics
    # a single iteration against the formula: assignment to the nearest initial centroid, mean of the members
    km1 = KMeansClustering(K, dim, iters=1)
    km1.init_centroids = init
    c1, i1, n1 = km1(x.cuda())
    d2 = (x.double().unsqueeze(1) - init.double().unsqueeze(0)).square().sum(-1)
    near = d2.argmin(1)
    margin = d2.topk(2, dim=1, largest=False).values
    safe = (margin[:, 1] - margin[:, 0]) > 1e-4 * margin[:, 1] if K > 1 else torch.ones(n, dtype=torch.bool)
    assert torch.equal(i1.cpu()[safe], near[safe])


@pytest.mark.parametrize('use_tc', [True, False])
@pytest.mark.parametrize('dim,B', [(64, 4096), (32, 100), (128, 300), (48, 257), (64, 2)])
def test_alignment_uniformity_forward_backward(dim, B, use_tc, monkeypatch):
    """DirectAU's losses (loss_utils.py:75-86) with the reference's dense signatures against the float64 oracle;
    the uniformity pair sum runs on the InfoNCE contraction (tensor-core 3xTF32 at dims 32 / 64, FP32 FMA otherwise)."""
    from sslrec_b200 import engine
    from sslrec_b200 import loss_utils as LU
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', use_tc)
    g = torch.Generator().manual_seed(31)
    x = torch.randn(B, dim, generator=g) * 0.3
    y = x * 0.5 + torch.randn(B, dim, generator=g) * 0.2
    if B > 10:
        x[7] = x[3]                                           # duplicated rows (the same user twice in a batch): pair distance 0
    xs = [t.clone().cuda().requires_grad_(True) for t in (x, y)]
    loss = LU.alignment(xs[0], xs[1]) + 2.0 * (LU.uniformity(xs[0]) + LU.uniformity(xs[1])) / 2
    loss.backward()
    ref = [t.double().clone().requires_grad_(True) for t in (x, y)]
    want = O.alignment(ref[0], ref[1]) + 2.0 * (O.uniformity(ref[0]) + O.uniformity(ref[1])) / 2
    want.backward()
    assert abs(loss.item() - want.item()) <= 1e-5 * max(1.0, abs(want.item())), (loss.item(), want.item())
    for a, b, name in zip(xs, ref, 'xy'):
        H.close(a.grad, b.grad, 2e-4, 2e-5 * b.grad.abs().max().item(), 'grad_' + name)
    # the single terms, and the fp32 reference formula (pdist) for the record
    assert abs(LU.uniformity(xs[0].detach()).item() - O.uniformity(x.double()).item()) <= 1e-5
    assert abs(LU.alignment(xs[0].detach(), xs[1].detach()).item() - O.alignment(x.double(), y.double()).item()) <= 1e-5


@pytest.mark.parametrize('use_tc', [True, False])
@pytest.mark.parametrize('dim,B,n', [(64, 1024, 5000), (32, 100, 777), (128, 130, 900), (64, 3, 70)])
def test_dense_logsumexp_mean_forward_backward(dim, B, n, use_tc, monkeypatch):
    """LightGCL's mean_b log(sum_j exp(a_b . t_j / temp) + 1e-8) on raw rows (lightgcl.py:112-113) against float64 torch."""
    from sslrec_b200 import engine
    monkeypatch.setattr(engine, 'USE_TENSOR_CORES', use_tc)
    g = torch.Generator().manual_seed(41)
    a = torch.randn(B, dim, generator=g) * 0.15
    t = torch.randn(n, dim, generator=g) * 0.15
    temp = 0.1
    ins = [x.clone().cuda().requires_grad_(True) for x in (a, t)]
    out = engine.dense_logsumexp_mean(ins[0], ins[1], temp, 1e-8)
    (out * 1.7).backward()
    ref = [x.double().clone().requires_grad_(True) for x in (a, t)]
    want = torch.log(torch.exp(ref[0] @ ref[1].T / temp).sum(1) + 1e-8).mean()
    (want * 1.7).backward()
    assert abs(out.item() - want.item()) <= 1e-5 * max(1.0, abs(want.item())), (out.item(), want.item())
    for x, r, name in zip(ins, ref, ('anchors', 'table')):
        H.close(x.grad, r.grad, 2e-4, 2e-5 * r.grad.abs().max().item(), 'grad_' + name)
    # the anchors may be a gathered, non-leaf slice and the table a slice of a larger tensor, as in the model
    big = torch.randn(n + 50, dim, generator=g).cuda().requires_grad_(True)
    idx = torch.randint(0, n, (B,), generator=g).cuda()
    o2 = engine.dense_logsumexp_mean((big * 0.1)[:n][idx], (big * 0.1)[:n], temp)
    o2.backward()
    b64 = big.detach().double().cpu().requires_grad_(True)
    w2 = torch.log(torch.exp((b64 * 0.1)[:n][idx.cpu()] @ (b64 * 0.1)[:n].T / temp).sum(1) + 1e-8).mean()
    w2.backward()
    assert abs(o2.item() - w2.item()) <= 1e-5 * max(1.0, abs(w2.item()))
    H.close(big.grad, b64.grad, 2e-4, 2e-5 * b64.grad.abs().max().item(), 'grad through slices')


@pytest.mark.parametrize('nu,ni,d,h,slope,keep', [(700, 500, 64, 128, 0.5, 0.5), (130, 65, 32, 16, 0.2, 1.0), (1000, 3, 48, 40, 1.0, 0.7),
                                                  (64, 64, 128, 128, 0.5, 0.5), (300, 200, 32, 128, 0.5, 0.5),
                                                  (25500, 130, 64, 128, 1.0, 0.5)])
def test_hyper_branch_forward_backward(nu, ni, d, h, slope, keep):
    """HCCF's hyper-graph layer (hccf.py:43-49, :100-108) on ssl_rowgemm / ssl_colgemm / ssl_hyper_dropout against torch
    autograd in float64, with the dropout keeps injected.  d = 32, H = 128 is hccf.yml's shape (colgemm <8, 2> and <2, 8>);
    25 500 user rows are more than 397 tiles of 64, so colgemm's CTAs sum two tiles each and the trailing ones are empty --
    there at slope 1, where no LeakyReLU kink can flip a derivative and the tight tolerance holds."""
    from sslrec_b200 import engine as E
    g = torch.Generator().manual_seed(nu + d + h)
    eu, ei = torch.randn(nu, d, generator=g) * 0.3, torch.randn(ni, d, generator=g) * 0.3
    wu, wi = torch.randn(d, h, generator=g) * 0.2, torch.randn(d, h, generator=g) * 0.2
    x = torch.randn(nu + ni, d, generator=g) * 0.5
    ku, ki = (torch.rand(nu, h, generator=g) + keep).floor(), (torch.rand(ni, h, generator=g) + keep).floor()
    gy = torch.randn(nu + ni, d, generator=g)
    mult = 1.3

    def run(dtype, dev, native):
        leaves = [t.to(dev, dtype).clone().requires_grad_(True) for t in (eu, ei, wu, wi, x)]
        e_u, e_i, w_u, w_i, xx = leaves
        if native:
            a_u, a_i = E.hyper_incidence(e_u, w_u, mult), E.hyper_incidence(e_i, w_i, mult)
            du = E.HyperDrop(keep=keep, mask=ku.to(dev)) if keep != 1.0 else E.HyperDrop()
            di = E.HyperDrop(keep=keep, mask=ki.to(dev)) if keep != 1.0 else E.HyperDrop()
            y = E.hyper_layer(xx, a_u, a_i, slope, du, di)
        else:
            outs = []
            for e_, w_, k_, xs in ((e_u, w_u, ku, xx[:nu]), (e_i, w_i, ki, xx[nu:])):
                hk = e_ @ w_ * mult * k_.to(dev, dtype) / keep
                outs.append(F.leaky_relu(hk @ F.leaky_relu(hk.T @ xs, slope), slope))
            y = torch.cat(outs)
        y.backward(gy.to(dev, dtype))
        return [y.detach()] + [t.grad for t in leaves]
    import torch.nn.functional as F
    got = run(torch.float32, 'cuda', True)
    want = run(torch.float64, 'cpu', False)
    for name, a, b in zip(('y', 'dE_u', 'dE_i', 'dW_u', 'dW_i', 'dX'), got, want):
        H.close(a, b, 2e-4, 2e-5 * b.abs().max().item() + 1e-9, f'hyper {name} ({nu},{ni},{d},{h})')


def test_hyper_dropout_rng_keep_fraction_and_determinism():
    from sslrec_b200 import engine as E
    a = torch.ones(5000, 128, device='cuda')
    d = E.HyperDrop(keep=0.3, seed=1234, stream=3)
    o1, o2 = E._drop(a, d), E._drop(a, d)
    assert torch.equal(o1, o2)                                                     # counter-based: same (seed, stream) -> same mask
    kept = (o1 != 0).float().mean().item()
    assert abs(kept - 0.3) < 0.005 and torch.allclose(o1[o1 != 0], torch.tensor(1 / 0.3, device='cuda'))
    o3 = E._drop(a, E.HyperDrop(keep=0.3, seed=1234, stream=4))
    assert (o3 != o1).float().mean().item() > 0.3                                   # another (layer, side) stream: another mask
    # backward = the same mask applied to the gradient
    gacc = torch.zeros_like(a)
    E._drop(torch.full_like(a, 2.0), d, out=gacc, accumulate=True)
    assert torch.equal(gacc, 2.0 * o1)


def test_hgnn_layer_one_side_forward_backward():
    """HGNNLayer(leaky)(adj, embeds) = act(adj @ act(adj.T @ embeds)) (hccf.py:100-108) on its own: one side through
    engine.hyper_layer, whose second side is empty (null row pointers), against torch autograd in float64."""
    import torch.nn.functional as F
    from sslrec_b200.general_cf.hccf import HGNNLayer
    g = torch.Generator().manual_seed(17)
    n, h, d, slope = 300, 40, 32, 0.5
    adj, embeds, gy = torch.randn(n, h, generator=g) * 0.3, torch.randn(n, d, generator=g) * 0.5, torch.randn(n, d, generator=g)
    a, e = adj.cuda().requires_grad_(True), embeds.cuda().requires_grad_(True)
    y = HGNNLayer(slope)(a, e)
    y.backward(gy.cuda())
    a64, e64 = adj.double().requires_grad_(True), embeds.double().requires_grad_(True)
    want = F.leaky_relu(a64 @ F.leaky_relu(a64.T @ e64, slope), slope)
    want.backward(gy.double())
    for name, got, ref in (('y', y.detach(), want.detach()), ('d adj', a.grad, a64.grad), ('d embeds', e.grad, e64.grad)):
        H.close(got, ref, 2e-4, 2e-5 * ref.abs().max().item(), f'HGNNLayer {name}')


def test_hyper_layer_rejects_a_negative_slope():
    """The backward takes LeakyReLU's derivative from the saved output, which is right only while the activation keeps the
    sign (slope >= 0); a negative slope is refused rather than trained with the wrong gradient."""
    from sslrec_b200 import engine as E
    from sslrec_b200.general_cf.hccf import HGNNLayer
    g = torch.Generator().manual_seed(18)
    x, a_u, a_i = torch.randn(50, 16, generator=g).cuda(), torch.randn(30, 8, generator=g).cuda(), torch.randn(20, 8, generator=g).cuda()
    with pytest.raises(ValueError, match='slope'):
        E.hyper_layer(x, a_u, a_i, -0.2, E.HyperDrop(), E.HyperDrop())
    with pytest.raises(ValueError, match='slope'):
        HGNNLayer(-0.2)(a_u, x[:30])
    E.hyper_layer(x, a_u, a_i, 0.0, E.HyperDrop(), E.HyperDrop())          # slope 0 (ReLU) is fine


@pytest.mark.parametrize('dim,V', [(64, 3), (128, 1)])
def test_row_sharded_plan_and_peer_stores_on_one_gpu(dim, V):
    """The kernel side of the fused all-gather without a second GPU: two plans that own complementary (user range, item
    range) pairs write their rows into one table and into two stand-in "peer" tables (ssl_prop_args.x_out_peers /
    sum_out_peers) -- together they must reproduce the full plan's layer bit for bit, and rows a plan does not own stay
    untouched.  Also the view-reduced last backward layer with the folded regulariser and the sharded Adam's peer stores."""
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import check, lib
    from sslrec_b200.graph import GraphPlan
    adj = _graph(300, 260, 5000, 3, hub=400)
    nu, n = adj.n_user, adj.n
    full = _plan(adj)
    x = torch.randn(n, V, dim, device='cuda')
    res = torch.randn(n, V, dim, device='cuda')
    views = [E.ViewSpec(edge_mode=1, keep=0.7, seed=5 + v) for v in range(V)]

    def launch(plan, out_tabs, peers=(), transpose=False, reduce=False, reg=None):
        prop = E.Propagation(plan, views, 1)
        a = prop._args(dim, 1, transpose)
        a.in_views, a.x_in, a.residual = V, x.data_ptr(), res.data_ptr()
        field, pf = ('sum_out', 'sum_out_peers') if reduce else ('x_out', 'x_out_peers')
        setattr(a, field, out_tabs.data_ptr())
        a.reduce_views = int(reduce)
        if reg is not None:
            a.reg_src, a.reg_coef, a.reg_coef_dev, a.reg_src2 = reg[0].data_ptr(), 2.0, reg[1].data_ptr(), reg[2].data_ptr()
        a.n_peers = len(peers)
        for q, p in enumerate(peers):
            getattr(a, pf)[q] = p.data_ptr()
        prop._launch(a, x)

    cuts = ((0, 120), (nu, nu + 100)), ((120, nu), (nu + 100, n))
    plans = [GraphPlan(adj.rows, adj.cols, adj.vals, n, torch.device('cuda'), row_ranges=c, side_split=nu) for c in cuts]
    assert sum(p.nnz for p in plans) == full.nnz and sum(p.n_rows for p in plans) == n
    for transpose in (False, True):
        want = torch.empty(n, V, dim, device='cuda')
        launch(full, want, transpose=transpose)
        own = torch.full((n, V, dim), -7.0, device='cuda')
        peers = [torch.full((n, V, dim), -7.0, device='cuda') for _ in range(2)]
        launch(plans[0], own, peers, transpose=transpose)
        (a0, a1), (b0, b1) = cuts[0]
        mine = torch.zeros(n, dtype=torch.bool, device='cuda')
        mine[a0:a1] = True
        mine[b0:b1] = True
        for t in [own] + peers:
            assert torch.equal(t[mine], want[mine]) and (t[~mine] == -7.0).all()
        launch(plans[1], own, peers, transpose=transpose)
        for t in [own] + peers:
            assert torch.equal(t, want)                      # every "GPU" now holds the whole layer, bit-identical to the unsharded launch
    # last backward layer: reduce over views + 2 g E0 read from the table + a second row source, stored to the peers as well
    e0, g, src2 = torch.randn(n, dim, device='cuda'), torch.tensor(0.37, device='cuda'), torch.randn(n, dim, device='cuda')
    want = torch.empty(n, dim, device='cuda')
    launch(full, want, transpose=True, reduce=True, reg=(e0, g, src2))
    own, peer = torch.zeros(n, dim, device='cuda'), torch.zeros(n, dim, device='cuda')
    for p in plans:
        launch(p, own, [peer], transpose=True, reduce=True, reg=(e0, g, src2))
    assert torch.equal(own, want) and torch.equal(peer, want)
    ref = torch.empty(n, dim, device='cuda')
    launch(full, ref, transpose=True, reduce=True)
    H.close(want, ref.double() + 2.0 * 0.37 * e0.double() + src2.double(), 1e-5, 1e-5, 'folded regulariser gradient')
    # sharded Adam: the owned range is updated and stored into the stand-in replicas
    p = torch.randn(1000, dim, device='cuda')
    reps, p_old = [p.clone(), p.clone()], p.clone()
    gr, m, v = torch.randn_like(p), torch.zeros_like(p), torch.zeros_like(p)
    p_ref, m_ref, v_ref = p.clone(), m.clone(), v.clone()
    lo, hi = 200, 650
    off = 4 * lo * dim
    arr = (C.c_void_p * 2)(*[r.data_ptr() + off for r in reps])
    s = torch.cuda.current_stream().cuda_stream
    check(lib.ssl_adam_step_peers(p.data_ptr() + off, arr, 2, gr.data_ptr() + off, m.data_ptr() + off, v.data_ptr() + off, (hi - lo) * dim, 1,
                                  1e-2, 0.9, 0.999, 1e-8, 0.0, s))
    check(lib.ssl_adam_step(p_ref.data_ptr(), gr.data_ptr(), m_ref.data_ptr(), v_ref.data_ptr(), p_ref.numel(), 1, 1e-2, 0.9, 0.999, 1e-8, 0.0, s))
    for t in [p] + reps:
        assert torch.equal(t[lo:hi], p_ref[lo:hi])                                        # the owned rows: updated everywhere
        assert torch.equal(t[:lo], p_old[:lo]) and torch.equal(t[hi:], p_old[hi:])         # the others: untouched
