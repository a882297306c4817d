"""Dynamic negative sampling (optional key train.dns_candidates) on the GPU.

Kernels, through the C ABI: ``ssl_neg_candidates`` equals tests/dns_oracle.neg_candidates bit for bit, column 0 is the loader's
negative, no candidate is a training positive (a user with every item but one gets that item, a user with every item the
capped draw), and the seed read from the device gives the host seed's candidates.  ``ssl_neg_select`` is bit-identical across
launches, plain tables and views of an interleaved table give the same ids, the chosen candidate's float64 score is within the
fp32 FMA-chain budget of the float64 maximum and is the exact argmax wherever the gap exceeds that budget; ties, NaN scores
and rejected arguments.

Models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL) under train.deterministic: M = 1 is the plain step bit for bit; an M = 8
step equals the plain step on the batch whose negatives are the selected ones (``dns_negs``), from the same seed-stream state;
two runs are identical and a CUDA-graph replay equals the eager loop; SimGCL and SGL mark every candidate row in the restricted
views; SimGCL and NCL resumed from a mid-run checkpoint end bit-identical to an uninterrupted run."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import dns_oracle as D
from oracle import inputs
from oracle import philox as P
from test_host_resume import make_run

pytestmark = pytest.mark.gpu

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def _graph(n_user, n_item, n_edge, seed):
    """A random graph in which user 0 has every item but n_item // 2 and user 1 every item (its candidates are the capped draw)."""
    rows, cols = inputs.bipartite_edges(n_user, n_item, n_edge, seed)
    keep = rows > 1
    free = n_item // 2
    rows = np.concatenate([rows[keep], np.zeros(n_item - 1, np.int64), np.ones(n_item, np.int64)])
    cols = np.concatenate([cols[keep], np.delete(np.arange(n_item), free), np.arange(n_item)])
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    m.sort_indices()
    dev = lambda a: torch.from_numpy(a.astype(np.int32)).cuda()
    return m, dev(m.indptr), dev(m.indices), free


@pytest.mark.parametrize('B,M,n_user,n_item', [(1, 2, 50, 12), (333, 8, 300, 200), (4096, 32, 2000, 3000), (77, 256, 400, 900)])
def test_candidates_match_the_oracle_and_avoid_positives(B, M, n_user, n_item):
    from sslrec_b200 import engine as E
    m, rowptr, cols, free = _graph(n_user, n_item, 10 * n_user, 21)
    rs = np.random.RandomState(B + M)
    users = rs.randint(0, n_user, size=B)
    users[: min(B, 3)] = [0, 1, 0][: min(B, 3)]
    negs = rs.randint(0, n_item, size=B)
    seed = 0x0123456789ABCDEF ^ B
    got = E.neg_candidates(torch.from_numpy(users).cuda(), torch.from_numpy(negs).cuda(), M, rowptr, cols, n_item, seed).cpu().numpy()
    want = D.neg_candidates(users, negs, M, m.indptr, m.indices, n_item, seed)
    assert np.array_equal(got, want)
    assert np.array_equal(got[:, 0], negs)
    assert got.min() >= 0 and got.max() < n_item
    dense = m.toarray() > 0
    drawn = got[:, 1:]
    rest = users > 1
    assert not dense[users[rest, None], drawn[rest]].any()
    # users 0 and 1: the free item or, after 256 rejected draws, the last draw (user 1 always)
    capped = lambda b, j: (int(P.philox4x32_10(b, j, 63, D.TAG_DNSC, seed)[3]) * n_item) >> 32
    for b in np.flatnonzero(~rest):
        for j in range(1, M):
            assert drawn[b, j - 1] == capped(b, j) or (users[b] == 0 and drawn[b, j - 1] == free), (b, j)
    assert (drawn[users == 0] == free).any()
    # the seed read from a device word (CUDA-graph replay) gives the same candidates
    word = torch.tensor([seed - (1 << 64) if seed >= 1 << 63 else seed], dtype=torch.int64, device='cuda')
    dseed = E.DevSeed(seed ^ 0x5555)            # a wrong host value: the device word must win
    dseed.ptr = word.data_ptr()
    got_dev = E.neg_candidates(torch.from_numpy(users).cuda(), torch.from_numpy(negs).cuda(), M, rowptr, cols, n_item, dseed)
    assert np.array_equal(got_dev.cpu().numpy(), got)


def _fp32_budget(u, items, ancs, cands):
    """|fp32 FMA chain - exact dot| <= gamma_d sum_k |u_k c_k|, gamma_d = d u / (1 - d u), u = 2^-24 (inputs are exact in float64)."""
    d = u.shape[1]
    g = d * 2.0 ** -24 / (1 - d * 2.0 ** -24)
    return g * torch.einsum('bd,bmd->bm', u.double()[ancs].abs(), items.double()[cands].abs())


@pytest.mark.parametrize('B,M,d', [(37, 2, 4), (1000, 8, 32), (4096, 32, 64), (513, 256, 128), (300, 3, 60)])
def test_selection_is_stable_and_the_float64_argmax(B, M, d):
    from sslrec_b200 import engine as E
    g = torch.Generator().manual_seed(B * M + d)
    n_user, n_item = 500, 700
    users = torch.randn(n_user, d, generator=g)
    items = torch.randn(n_item, d, generator=g)
    items[7] = items[3]                                  # twins: exact ties between distinct ids
    ancs = torch.randint(0, n_user, (B,), generator=g)
    cands = torch.randint(0, n_item, (B, M), generator=g)
    cands[::5, M - 1] = 7
    cands[::5, 0] = 3                                   # pairs where 3 (j = 0) and 7 (j = M-1) tie
    uc, ic, ac, cc = users.cuda(), items.cuda(), ancs.cuda(), cands.cuda()
    a = E.hard_negatives(uc, ic, ac, cc)
    b = E.hard_negatives(uc, ic, ac, cc)
    assert torch.equal(a, b)
    got = a.cpu()
    s64 = D.scores(users, items, ancs, cands)
    budget = _fp32_budget(users, items, ancs, cands)
    j_got = (cands == got[:, None]).to(torch.int8).argmax(1)
    best = s64.max(1).values
    chosen = s64.gather(1, j_got[:, None]).squeeze(1)
    slack = 2 * budget.max(1).values
    assert (chosen >= best - slack).all()
    top2 = s64.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > slack
    ref = D.hard_negatives(users, items, ancs, cands)
    assert torch.equal(got[clear], ref[clear])
    assert clear.float().mean() > 0.5
    # 3 and 7 tie exactly: wherever they clearly beat every other candidate, the lower j (3 at j = 0) wins
    tie_rows = torch.arange(0, B, 5)
    others = s64[tie_rows, 1:M - 1].max(1).values if M > 2 else torch.full((len(tie_rows),), -float('inf'), dtype=torch.float64)
    won = s64[tie_rows, 0] - others > slack[tie_rows]
    assert won.any() and (got[tie_rows[won]] == 3).all()
    # the same rows as view 1 of an interleaved [N, 3, d] table: the same ids
    n = n_user + n_item
    blk = torch.randn(n, 3, d, device='cuda')
    blk[:n_user, 1] = uc
    blk[n_user:, 1] = ic
    ur, ir = E.Rows(blk, 1, 3, 0, n_user, d), E.Rows(blk, 1, 3, n_user, n_item, d)
    assert torch.equal(E.hard_negatives(ur, ir, ac, cc), a)


def test_nan_scores_never_win():
    from sslrec_b200 import engine as E
    users = torch.ones(2, 4, device='cuda')
    items = torch.tensor([[1.0, 0, 0, 0], [float('nan'), 0, 0, 0], [-5.0, 0, 0, 0], [float('nan'), 1, 1, 1]], device='cuda')
    cands = torch.tensor([[1, 2, 0], [1, 3, 1]], device='cuda')
    got = E.hard_negatives(users, items, torch.tensor([0, 1], device='cuda'), cands)
    assert got.tolist() == [0, 1]                       # the finite maximum; all NaN -> candidate 0


def test_bad_arguments_are_rejected_and_write_nothing():
    from sslrec_b200._lib import lib
    dev = 'cuda'
    users = torch.zeros(4, dtype=torch.int64, device=dev)
    rowptr = torch.zeros(2, dtype=torch.int32, device=dev)
    cols = torch.zeros(1, dtype=torch.int32, device=dev)
    cands = torch.full((4, 8), -7, dtype=torch.int64, device=dev)
    tbl = torch.zeros(10, 32, device=dev)
    out = torch.full((4,), -7, dtype=torch.int64, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()

    def cand(B=4, M=8, n_item=10, nulls=()):
        a = [p(users), p(users), B, M, p(rowptr), p(cols), n_item, 1, None, p(cands), s]
        for i in nulls:
            a[i] = None
        return lib.ssl_neg_candidates(*a)

    def sel(B=4, M=8, dim=32, us=32, is_=32, nulls=()):
        a = [p(tbl), us, p(tbl), is_, p(users), p(cands), B, M, dim, p(out), s]
        for i in nulls:
            a[i] = None
        return lib.ssl_neg_select(*a)

    for rc in (cand(M=1), cand(M=257), cand(B=-1), cand(B=1 << 31), cand(n_item=0), cand(n_item=1 << 31), cand(nulls=(0,)),
               cand(nulls=(1,)), cand(nulls=(4,)), cand(nulls=(5,)), cand(nulls=(9,)),
               sel(M=1), sel(M=257), sel(dim=0), sel(dim=129), sel(us=31), sel(is_=16), sel(B=-2), sel(nulls=(0,)), sel(nulls=(2,)),
               sel(nulls=(4,)), sel(nulls=(5,)), sel(nulls=(9,))):
        assert rc == -1
    assert cand(B=0) == 0 and sel(B=0) == 0
    torch.cuda.synchronize()
    assert (cands == -7).all() and (out == -7).all()


# ---- models ------------------------------------------------------------------------------------------------------------------

def _run(key, M, **train):
    m, tr, dh = make_run(key, device='cuda', train=dict(deterministic=True, dns_candidates=M, **train))
    return m, tr


def _batches(key, n=5, seed=5):
    """Batches of the tiny graph with repeated users and items (NCL: the re-cluster flag on the first and the fourth)."""
    case = inputs.make_case('tiny')
    rs = np.random.RandomState(seed)
    B, n_edges = 96, len(case['rows'])
    out = []
    for k in range(n):
        pick = np.where(rs.rand(B) < 0.5, rs.randint(0, 3, size=B), rs.randint(0, n_edges, size=B))
        negs = rs.randint(0, case['n_item'], size=B)
        b = [torch.from_numpy(np.asarray(a)).long().cuda() for a in (case['rows'][pick], case['cols'][pick], negs)]
        if key == 'ncl':
            f = torch.zeros(B, dtype=torch.int64)
            f[0] = int(k in (0, 3))
            b.append(f.cuda())
        out.append(b)
    return out


def _step(m, opt, batch):
    opt.zero_grad()
    torch.manual_seed(0)                      # NCL's k-means draws its initial centroids from torch's generator
    loss, parts = m.cal_loss(batch)
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}
    opt.step()
    torch.cuda.synchronize()
    return ({k: torch.as_tensor(v).detach().clone() for k, v in dict(parts, loss=loss).items()}, grads,
            {n: p.detach().clone() for n, p in m.named_parameters()})


def _assert_equal(a, b, what):
    for x, y, part in zip(a, b, ('terms', 'grads', 'params')):
        assert x.keys() == y.keys(), (what, part)
        for k in x:
            assert torch.equal(x[k], y[k]), (what, part, k)


@pytest.mark.parametrize('key', BPR_MODELS)
def test_m1_is_the_plain_step_bit_for_bit(key):
    from sslrec_b200.optim import FusedAdam
    runs = []
    for train in (dict(deterministic=True), dict(deterministic=True, dns_candidates=1)):
        m, _, _ = make_run(key, device='cuda', train=train)
        opt = FusedAdam(m.parameters(), lr=1e-2)
        runs.append(([_step(m, opt, b) for b in _batches(key, n=2)], m._seeds.count, m.dns_negs))
    (plain, n_plain, _), (one, n_one, dns_negs) = runs
    assert n_plain == n_one and dns_negs is None             # no extra seed, no selection
    for k, (a, b) in enumerate(zip(plain, one)):
        _assert_equal(a, b, (key, k))


@pytest.mark.parametrize('key', BPR_MODELS)
def test_dns_step_is_the_plain_step_on_the_selected_negatives(key):
    from sslrec_b200.optim import FusedAdam
    dns, _ = _run(key, 8)
    plain, _ = _run(key, 1)
    plain.load_state_dict(dns.state_dict())
    od, op = FusedAdam(dns.parameters(), lr=1e-2), FusedAdam(plain.parameters(), lr=1e-2)
    changed = 0
    for k, batch in enumerate(_batches(key)):
        plain._seeds.load_state_dict(dns._seeds.state_dict())
        a = _step(dns, od, batch)
        sel = dns.dns_negs.clone()
        changed += int((sel != batch[2]).sum())
        b = _step(plain, op, [batch[0], batch[1], sel] + batch[3:])
        _assert_equal(a, b, (key, k))
        assert dns._seeds.count == plain._seeds.count + 1            # the candidate seed, drawn last
    assert changed > 0


def _train(key, graphed, n=6):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    m, _ = _run(key, 8)
    opt = FusedAdam(m.parameters(), lr=1e-2)
    batches = _batches(key, n=n)
    ncl = key == 'ncl'
    out = []
    if graphed:
        torch.manual_seed(0)
        step = GraphedStep(m, opt, batches[0], warmup=2, recluster=ncl)
        for k, b in enumerate(batches[1:], start=1):
            loss, parts = step(b, recluster=ncl and k == 3)
            out.append((loss.clone(), m.dns_negs.clone()))
        step.close()
    else:
        m._graph_mode = key == 'hccf'             # the path GraphedStep takes
        torch.manual_seed(0)
        for k, b in enumerate([batches[0]] * 2 + batches[1:]):
            opt.zero_grad()
            loss, _ = m.cal_loss(b)
            loss.backward()
            opt.step()
            if k >= 2:
                out.append((loss.detach().clone(), m.dns_negs.clone()))
        m._graph_mode = False
    torch.cuda.synchronize()
    return out, {n_: p.detach().clone() for n_, p in m.named_parameters()}


@pytest.mark.parametrize('key', BPR_MODELS)
def test_two_runs_and_graph_replay_are_bit_identical(key):
    first, second, graphed = _train(key, False), _train(key, False), _train(key, True)
    for other, what in ((second, 'eager run 2'), (graphed, 'graph replay')):
        assert len(other[0]) == len(first[0]) == 5
        for k, ((la, na), (lb, nb)) in enumerate(zip(first[0], other[0])):
            assert torch.equal(la, lb) and torch.equal(na, nb), (key, what, k)
        for n_ in first[1]:
            assert torch.equal(first[1][n_], other[1][n_]), (key, what, n_)


@pytest.mark.parametrize('key,views', [('simgcl', (0, 2)), ('sgl', (0,))])
def test_restricted_views_mark_every_candidate(monkeypatch, key, views):
    from sslrec_b200 import engine as E
    m, _ = _run(key, 32)
    seen = {}
    neg_candidates = E.neg_candidates

    def keep(*a, **kw):
        seen['cands'] = neg_candidates(*a, **kw)
        return seen['cands']

    monkeypatch.setattr(E, 'neg_candidates', keep)
    m.cal_loss(_batches(key, n=1)[0])[0].backward()
    st = m._state
    rows = (seen['cands'].view(-1) + m.user_num).cpu()
    for v in views:
        assert v in st.restricted_views
        bits = st.prop.views[v].row_bits.cpu().to(torch.int64)
        assert (((bits[rows >> 5] >> (rows & 31)) & 1) == 1).all(), v
    assert (seen['cands'] == m.dns_negs[:, None]).any(1).all()


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('key,hp', [('simgcl', {}), ('ncl', {'epoch_period': 2})])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph):
    import test_gpu_resume as R
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, dns_candidates=8)
    ref = R._train(key, hp, dict(base, epoch=4))
    first = R._train(key, hp, dict(base, epoch=2, checkpoint_step=1))
    assert first['losses'] == {e: ref['losses'][e] for e in (0, 1)}
    R._scramble()
    res = R._train(key, hp, dict(base, epoch=4, resume_path=str(R._checkpoint(tmp_path, key))), seed_globals=False)
    assert sorted(res['losses']) == [2, 3]
    for e in (2, 3):
        assert res['losses'][e] == ref['losses'][e], (e, res['losses'][e], ref['losses'][e])
    R._assert_same_evals(ref['evals'][2:], res['evals'])
    R._assert_same_params_and_adam(ref, res)
    assert res['seeds'] == ref['seeds']
