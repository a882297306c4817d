"""Parity at BASELINE.json's full sizes (synthetic graphs with the bundled datasets' shapes): the CUDA path against the
oracle run live on the host cores with the same weights, batch and injected noise / masks."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import cf_oracle as O
import ssl_test_helpers as H

pytestmark = pytest.mark.gpu


def _setup(model_name, graph, hp, seed=7):
    from synth_graphs import named_graph
    rows, cols, U, I = named_graph(graph, seed=2023)
    case = dict(rows=rows, cols=cols, n_user=U, n_item=I, dim=hp['embedding_size'], batch=4096)
    g = torch.Generator().manual_seed(seed)
    d = hp['embedding_size']
    case['user_e'] = (torch.rand(U, d, generator=g) * 2 - 1) * float(np.sqrt(6.0 / (U + d)))
    case['item_e'] = (torch.rand(I, d, generator=g) * 2 - 1) * float(np.sqrt(6.0 / (I + d)))
    rs = np.random.RandomState(seed)
    pick = rs.randint(0, len(rows), size=4096)
    case['ancs'], case['poss'], case['negs'] = rows[pick], cols[pick], rs.randint(0, I, size=4096).astype(np.int64)
    adj = O.normalized_adjacency(rows, cols, U, I)
    return case, adj, g


def test_simgcl_amazon_shape_step_matches_oracle():
    hp = dict(layer_num=3, embedding_size=64, temperature=0.2, eps=0.9, cl_weight=1.0e-2, reg_weight=1.0e-6, keep_rate=1.0)
    case, adj, g = _setup('simgcl', 'amazon', hp)
    uniforms = [[torch.rand(adj.n, 64, generator=g) for _ in range(3)] for _ in range(2)]
    inj = {'noise_u': [[u.cuda() for u in view] for view in uniforms]}
    model, _ = H.make_model('simgcl', case, hp, inject=inj)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    ue, ie = case['user_e'].clone().requires_grad_(True), case['item_e'].clone().requires_grad_(True)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref, rparts = O.simgcl_loss(adj, ue, ie, tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 3, hp['reg_weight'],
                                hp['cl_weight'], hp['temperature'], hp['eps'], uniforms[0], uniforms[1])
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5, (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k]) - float(rparts[k])) <= 1e-5, k
    bad_rows = []
    for got, want in ((model.user_embeds.grad, ue.grad), (model.item_embeds.grad, ie.grad)):
        # 10.2 M gradient entries.  EmbedPerturb adds eps * sign(x) * noise: where a propagated value sits within fp32
        # reassociation noise of zero (expected for a handful of the 41 M perturbed elements) the CPU and CUDA summation
        # orders can disagree on sign(x), which moves that element by ~0.1 and its neighbourhood's gradient by ~1e-2
        # relative.  So: every entry within 5e-4 / 5e-5 of the largest, except at most 2e-5 of them, and those within 2e-2
        # of the largest entry (measured: 29 of 4.9 M item-gradient entries, worst 2.8e-3 of the largest).
        got64, want64 = got.double().cpu(), want.double()
        err = (got64 - want64).abs()
        tol = 5e-4 * want64.abs() + 5e-5 * want64.abs().max()
        bad = err > tol
        assert bad.float().mean().item() <= 2e-5, f'{int(bad.sum())} of {bad.numel()} gradient entries off'
        assert err.max().item() <= 2e-2 * want64.abs().max().item(), (err.max().item(), want64.abs().max().item())
        bad_rows.append(torch.nonzero(bad.any(1)).flatten())
    # pin the explanation: the off entries must sit inside the L-hop neighbourhoods of the nodes that own a "fragile"
    # element -- a pre-perturbation value within reassociation noise of zero in some layer of a perturbed view, where
    # sign(x) (aug_utils.py:131) is not decidable in fp32.  Counted on the oracle side in float64.
    a64 = adj.torch_coo(torch.float64)
    fragile = torch.zeros(adj.n, dtype=torch.bool)
    n_fragile = 0
    for view in uniforms:
        x = torch.cat([case['user_e'], case['item_e']], 0).double()
        for k in range(3):
            pre = O.propagate(a64, x)
            scale = O.propagate(a64, x.abs())                        # sum of |terms|: the reassociation error is ~1e-7 of it
            fr = pre.abs() <= 4e-7 * scale
            n_fragile += int(fr.sum())
            fragile |= fr.any(1)
            x = O.perturbed(pre, view[k].double(), hp['eps'])
    reach = fragile.clone().double().unsqueeze(1)
    hood = fragile.clone()
    for _ in range(3):
        reach = (O.propagate(a64, reach) > 0).double()
        hood |= reach.squeeze(1).bool()
    off = torch.cat([bad_rows[0], bad_rows[1] + adj.n_user]) if bad_rows else torch.empty(0, dtype=torch.long)
    inside = hood[off].float().mean().item() if off.numel() else 1.0
    print(f'simgcl/amazon gradient: {n_fragile} fragile sign(x) elements on {int(fragile.sum())} nodes; {off.numel()} gradient rows beyond the tight '
          f'tolerance, {inside:.3f} of them inside the 3-hop neighbourhoods ({hood.float().mean().item():.4f} of all nodes)')
    assert off.numel() == 0 or n_fragile > 0, 'gradient rows off without any undecidable sign(x)'
    assert inside >= 0.999, 'gradient rows off outside the neighbourhoods of the undecidable sign(x) elements' 
    # evaluation on the same weights: top-40 of 1024 users against torch.topk of the oracle's scores
    from sslrec_b200.trainer import topk
    model.eval()
    users = torch.arange(1024)
    with torch.no_grad():
        preds = model.full_predict([users.cuda(), None])
        e = O.lightgcn_embeds(adj.torch_coo(), torch.cat([case['user_e'], case['item_e']], 0), 3)
        want = e[:1024] @ e[adj.n_user:].T
    idx, val = topk(preds, 40, return_values=True)
    wv, wi = torch.topk(want, 40)
    H.close(val, wv, 1e-5, 1e-7, 'top-40 scores')
    gap = (wv[:, :-1] - wv[:, 1:]).abs()
    near = gap <= 2e-6 * wv[:, :-1].abs().clamp(min=1e-3)
    ok = torch.ones_like(wi, dtype=torch.bool)
    ok[:, :-1] &= ~near
    ok[:, 1:] &= ~near
    ok[:, -1] = False
    _assert_topk(idx, wi, ok, 'simgcl/amazon')


def _assert_topk(idx, wi, decidable, what):
    """Top-k index parity: identical wherever the reference's own score gap is not a near-tie, and the EXACT match
    fraction over all positions is printed and must be >= 0.99."""
    same = idx.cpu() == wi
    frac = same.float().mean().item()
    print(f'top-k {what}: exact index match {frac:.5f} of {same.numel()} positions; decidable {decidable.float().mean().item():.5f}')
    assert same[decidable].all(), f'{what}: index differs at a position whose score gap is not a tie'
    assert frac >= 0.99, f'{what}: only {frac:.4f} of the top-k positions match exactly'


def _compare_grads(model, ue, ie, what, rtol=2e-4, atol_rel=5e-6, kink_frac=0.0, kink_rel=0.0):
    """Every gradient entry within rtol * |want| + atol_rel * max|want|.  Models with a kink in the forward pass (LeakyReLU at 0
    in HCCF's hyper branch, like sign(x) in SimGCL) may have a fraction ``kink_frac`` of entries outside it -- an element whose
    pre-activation lies within fp32 reassociation noise of zero takes the other branch's derivative on one of the two sides --
    and those must still be within ``kink_rel`` of the largest entry."""
    for name, got, want in (('user', model.user_embeds.grad, ue.grad), ('item', model.item_embeds.grad, ie.grad)):
        got64, want64 = got.double().cpu(), want.double()
        err = (got64 - want64).abs()
        tol = rtol * want64.abs() + atol_rel * want64.abs().max()
        bad = err > tol
        msg = f'{what} {name} gradient: {int(bad.sum())} of {bad.numel()} entries off, max err {err.max().item():.3e} (largest entry {want64.abs().max().item():.3e})'
        if bad.any():
            print(msg)
        assert bad.float().mean().item() <= kink_frac, msg
        assert (not bad.any()) or err.max().item() <= kink_rel * want64.abs().max().item(), msg


def _topk_check(model, adj, e_final, what, n_users=1024):
    from sslrec_b200.trainer import topk
    model.eval()
    users = torch.arange(n_users)
    with torch.no_grad():
        preds = model.full_predict([users.cuda(), None])
    want = e_final[:n_users] @ e_final[adj.n_user:].T
    idx, val = topk(preds, 40, return_values=True)
    wv, wi = torch.topk(want, 40)
    H.close(val, wv, 1e-5, 1e-7, what + ' top-40 scores')
    gap = (wv[:, :-1] - wv[:, 1:]).abs()
    near = gap <= 2e-6 * wv[:, :-1].abs().clamp(min=1e-3)
    ok = torch.ones_like(wi, dtype=torch.bool)
    ok[:, :-1] &= ~near
    ok[:, 1:] &= ~near
    ok[:, -1] = False
    _assert_topk(idx, wi, ok, what)
    model.train()


def test_lightgcn_gowalla_shape_injected_edge_mask_matches_oracle():
    """BASELINE config 1: LightGCN, gowalla shape, d = 64, L = 3, keep_rate 0.5 with the SAME edge mask on both sides."""
    hp = dict(layer_num=3, embedding_size=64, reg_weight=1.0e-8, keep_rate=0.5)
    case, adj, g = _setup('lightgcn', 'gowalla', hp)
    keep = (torch.rand(adj.nnz, generator=g) + 0.5).floor().bool().numpy()            # floor(U + keep), aug_utils.py:28
    inj = {'edge_masks': [torch.from_numpy(keep.astype(np.uint8)).cuda(), None, None, None]}
    model, _ = H.make_model('lightgcn', case, hp, inject=inj)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    ue, ie = case['user_e'].clone().requires_grad_(True), case['item_e'].clone().requires_grad_(True)
    ref, rparts = O.lightgcn_loss(adj, ue, ie, tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 3, hp['reg_weight'], 0.5, keep)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5, (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k].detach()) - float(rparts[k].detach())) <= 1e-5, k
    _compare_grads(model, ue, ie, 'lightgcn/gowalla')
    with torch.no_grad():
        e = O.lightgcn_embeds(adj.torch_coo(), torch.cat([case['user_e'], case['item_e']], 0), 3)     # evaluation: no edge drop
    model.final_embeds = None
    model.is_training = False
    _topk_check(model, adj, e, 'lightgcn/gowalla')


def test_sgl_yelp_shape_injected_masks_match_oracle():
    """BASELINE config 3: SGL edge_drop, yelp shape, d = 64, L = 3, keep 0.5 -- VALUES against the oracle with both views'
    edge masks injected on both sides."""
    hp = dict(layer_num=3, embedding_size=64, temperature=0.2, cl_weight=1.0, reg_weight=1.0e-5, keep_rate=0.5, augmentation='edge_drop')
    case, adj, g = _setup('sgl', 'yelp', hp)
    keeps = [(torch.rand(adj.nnz, generator=g) + 0.5).floor().bool().numpy() for _ in range(2)]
    inj = {'edge_masks': [torch.from_numpy(m.astype(np.uint8)).cuda() for m in keeps] + [None, None], 'node_masks': [None, None]}
    model, _ = H.make_model('sgl', case, hp, inject=inj)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    ue, ie = case['user_e'].clone().requires_grad_(True), case['item_e'].clone().requires_grad_(True)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref, rparts = O.sgl_loss(adj, ue, ie, tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 3, hp['reg_weight'], hp['cl_weight'],
                             hp['temperature'], 'edge_drop', 0.5, edge_keeps=keeps)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(1.0, abs(ref.item())), (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k].detach()) - float(rparts[k].detach())) <= 1e-5 * max(1.0, abs(float(rparts[k].detach()))), k
    _compare_grads(model, ue, ie, 'sgl/yelp')


def test_ncl_amazon_shape_k50_matches_oracle():
    """BASELINE config 5 (NCL): amazon shape, d = 64, L = 3, high_order 2, cluster_num 50 (ncl.yml), k-means state injected."""
    hp = dict(layer_num=3, embedding_size=64, high_order=2, reg_weight=1.0e-7, proto_weight=1.0e-4, struct_weight=1.0e-3, temperature=0.1,
              epoch_period=3, cluster_num=50, keep_rate=1.0)
    case, adj, g = _setup('ncl', 'amazon', hp)
    U, I = case['n_user'], case['n_item']
    cents = [torch.randn(50, 64, generator=g) * 0.05 for _ in range(2)]
    assign = [torch.randint(0, 50, (U,), generator=g), torch.randint(0, 50, (I,), generator=g)]
    model, _ = H.make_model('ncl', case, hp)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    model.user_centroids, model.item_centroids = cents[0].cuda(), cents[1].cuda()
    model.user2cluster, model.item2cluster = assign[0].cuda(), assign[1].cuda()
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')] + [torch.zeros(4096, dtype=torch.int64).cuda()]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    ue, ie = case['user_e'].clone().requires_grad_(True), case['item_e'].clone().requires_grad_(True)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref, rparts = O.ncl_loss(adj, ue, ie, tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 3, 2, hp['reg_weight'], hp['proto_weight'],
                             hp['struct_weight'], hp['temperature'], cents[0], assign[0], cents[1], assign[1])
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5, (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k].detach()) - float(rparts[k].detach())) <= 1e-5, k
    _compare_grads(model, ue, ie, 'ncl/amazon')


def test_hccf_amazon_shape_h128_matches_oracle():
    """BASELINE config 5 (HCCF): amazon shape, d = 64, L = 2, hyper_num 128 (hccf.yml), keep 0.5; edge masks and the hyper
    dropout keeps injected on both sides."""
    hp = dict(layer_num=2, embedding_size=64, reg_weight=1.0e-7, cl_weight=1.0, temperature=0.1, keep_rate=0.5, mult=1.0, hyper_num=128, leaky=0.5)
    case, adj, g = _setup('hccf', 'amazon', hp)
    U, I = case['n_user'], case['n_item']
    a = float(np.sqrt(6.0 / (64 + 128)))
    uw, iw = ((torch.rand(64, 128, generator=g) * 2 - 1) * a for _ in range(2))
    edge_keeps = [(torch.rand(adj.nnz, generator=g) + 0.5).floor().bool().numpy() for _ in range(2)]
    hyper_keeps = [((torch.rand(U, 128, generator=g) + 0.5).floor(), (torch.rand(I, 128, generator=g) + 0.5).floor()) for _ in range(2)]
    inj = {'edge_masks_per_layer': [torch.from_numpy(m.astype(np.uint8)).cuda() for m in edge_keeps],
           'hyper_keeps': [(ku.cuda(), ki.cuda()) for ku, ki in hyper_keeps]}
    model, _ = H.make_model('hccf', case, hp, inject=inj)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e'], 'user_hyper_embeds': uw, 'item_hyper_embeds': iw})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    ps = [t.clone().requires_grad_(True) for t in (case['user_e'], case['item_e'], uw, iw)]
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref, rparts = O.hccf_loss(adj, ps[0], ps[1], ps[2], ps[3], tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 2, hp['reg_weight'],
                              hp['cl_weight'], hp['temperature'], 0.5, 1.0, 0.5, edge_keeps=edge_keeps, hyper_keeps=hyper_keeps)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(1.0, abs(ref.item())), (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k].detach()) - float(rparts[k].detach())) <= 1e-5 * max(1.0, abs(float(rparts[k].detach()))), k
    _compare_grads(model, ps[0], ps[1], 'hccf/amazon', rtol=5e-4, atol_rel=2e-5, kink_frac=2e-5, kink_rel=2e-2)
    for name, got, want in (('user_hyper', model.user_hyper_embeds.grad, ps[2].grad), ('item_hyper', model.item_hyper_embeds.grad, ps[3].grad)):
        H.close(got, want, 1e-3, 2e-5 * want.abs().max().item(), 'hccf/amazon grad ' + name)


def test_lightgcn_config4_slice_d128_matches_oracle():
    """The d = 128 path of BASELINE config 4 on a 1/8 slice of its graph family (625 k x 125 k nodes, 18.75 M edges: the
    384 MB table is 8x the 50 MB L2): propagation + BPR + reg forward and backward against the oracle."""
    import synth_graphs as S
    U, I, E = 625_000, 125_000, 18_750_000
    keys = S.bipartite_keys_device(U, I, E, 2023, 1.0, 'cuda')
    rows, cols = (keys // I).cpu().numpy(), (keys % I).cpu().numpy()
    hp = dict(layer_num=3, embedding_size=128, reg_weight=1.0e-8, keep_rate=1.0)
    g = torch.Generator().manual_seed(11)
    case = dict(rows=rows, cols=cols, n_user=U, n_item=I, dim=128, batch=4096)
    case['user_e'] = (torch.rand(U, 128, generator=g) * 2 - 1) * float(np.sqrt(6.0 / (U + 128)))
    case['item_e'] = (torch.rand(I, 128, generator=g) * 2 - 1) * float(np.sqrt(6.0 / (I + 128)))
    rs = np.random.RandomState(5)
    pick = rs.randint(0, E, size=4096)
    case['ancs'], case['poss'], case['negs'] = rows[pick], cols[pick], rs.randint(0, I, size=4096).astype(np.int64)
    # the device generator's CSR values against the host formula (bit-identical) -- and through the plan the model uses
    adj = O.normalized_adjacency(rows, cols, U, I)
    rowptr, colidx, vals = S.normalized_csr_device(keys, U, I)
    assert np.array_equal(colidx.cpu().numpy(), adj.cols.astype(np.int32))
    assert (vals.cpu().numpy().view(np.uint32) != adj.vals.view(np.uint32)).mean() <= 1e-6      # float64 pow on the device: last-ulp ties at most
    model, _ = H.make_model('lightgcn', case, hp)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    loss, parts = model.cal_loss(batch)
    loss.backward()
    assert model._plan().stats()['max_row_nnz'] > 10_000                # the Zipf head: split rows are exercised
    ue, ie = case['user_e'].clone().requires_grad_(True), case['item_e'].clone().requires_grad_(True)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref, rparts = O.lightgcn_loss(adj, ue, ie, tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')), 3, hp['reg_weight'])
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5, (loss.item(), ref.item())
    for k in rparts:
        assert abs(float(parts[k].detach()) - float(rparts[k].detach())) <= 1e-5, k
    _compare_grads(model, ue, ie, 'lightgcn/config-4 slice')


def test_sgl_yelp_shape_rng_augmentation_statistics():
    """In-kernel RNG edge drop at keep 0.5 on the yelp-shaped graph: the kept fraction and the step's determinism."""
    hp = dict(layer_num=3, embedding_size=64, temperature=0.2, cl_weight=1.0, reg_weight=1.0e-5, keep_rate=0.5, augmentation='edge_drop')
    case, adj, g = _setup('sgl', 'yelp', hp)
    model, _ = H.make_model('sgl', case, hp)
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']})
    batch = [torch.from_numpy(case[k]).cuda() for k in ('ancs', 'poss', 'negs')]
    from sslrec_b200 import engine as E
    losses = []
    for _ in range(2):
        model._seeds = E.SeedStream(2023)
        loss, _ = model.cal_loss(batch)
        losses.append(loss.item())
    assert losses[0] == losses[1]                       # same seeds -> bit-identical loss (fixed summation order, counter-based RNG)
    ones = torch.ones(adj.n, 64, device='cuda')
    view = model.edge_dropper.view(0.5, 99)
    kept = E.spmm(model._plan(), ones, view)[:, 0].double().sum().item() / float(adj.vals.astype(np.float64).sum())
    assert abs(kept - 0.5) < 0.01
