"""Popularity-proportional candidates (optional key train.neg_popularity) on the GPU.

Kernels, through the C ABI: ``ssl_neg_candidates_pop`` equals tests/pop_oracle.neg_candidates and its bias bit for bit (several
B, M up to 256, n_item not a power of two, a user with every item), with the seed read from a device word and under CUDA-graph
replay; the draws of one user follow the table's distribution restricted to its non-positives (chi-square); the logQ-corrected
sum sum_q exp(s_q - bias_q) over one user repeated 64 k times estimates sum over its non-positives of exp(s_i) without bias.
``ssl_ssm_fwd_logq``: scores and norms bit-exact against the float32 restatement, loss and gradients within fp32 bounds of
float64, bias = 0 equals ``ssl_ssm_fwd``; rejected arguments write nothing.

Models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL): key null is the key absent bit for bit; with DNS, MixGCF and the sampled
softmax, two runs and a CUDA-graph replay are bit-identical under train.deterministic; SimGCL's and SGL's restricted views mark
every candidate; with beta = 0 every bias entry is ln M - ln(n_item - deg_u) and the loss is the uncorrected loss with the
negative scores shifted by it; two steps on different batches each apply the bias of their own candidates; SimGCL and NCL resumed
from a mid-run checkpoint end bit-identical to an uninterrupted run.  All six, on both gradient routes, at beta 0.75 on every
row of tests/test_gpu_mixgcf.whole_step_rows(ssm=True) and at beta 1 and 0 for LightGCN and HCCF: the step's candidates and
bias are tests/pop_oracle's for its own seed, pairs and training matrix bit for bit, the bias is within a few ulp of the float64
bias from its definition, and the whole step equals the float64 oracle with the logQ-corrected term (pop_oracle.term64_logq)
within the golden tolerances, for every parameter's gradient, while the uncorrected term is outside them;
tests/test_host_neg_popularity.py shows on the host that the float32 oracle meets these bounds and wrong corrections do not."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.stats
import torch

import pop_oracle as O
import ssl_test_helpers as H
import ssm_oracle as S
from test_gpu_hard_negatives import _assert_equal, _batches, _step
from test_gpu_mixgcf import whole_step, whole_step_rows
from test_host_resume import make_run

pytestmark = pytest.mark.gpu

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def _graph(n_user, n_item, n_edge, seed):
    """Zipf-skewed item degrees (the top fifth of the ids never occurs); user 0 has every item, user 1 every item but
    n_item // 2."""
    rs = np.random.RandomState(seed)
    rows = rs.randint(2, n_user, n_edge)
    cols = (rs.zipf(1.2, n_edge) - 1) % max(1, int(n_item * 0.8))
    free = n_item // 2
    rows = np.concatenate([rows, np.zeros(n_item, np.int64), np.ones(n_item - 1, np.int64)])
    cols = np.concatenate([cols, np.arange(n_item), np.delete(np.arange(n_item), free)])
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    m.sum_duplicates()
    m.data[:] = 1
    m.sort_indices()
    dev = lambda a: torch.from_numpy(a.astype(np.int32)).cuda()
    return m, dev(m.indptr), dev(m.indices), free


@pytest.mark.parametrize('B,M,n_user,n_item,beta', [(1, 2, 50, 12, 0.75), (333, 8, 300, 201, 1.0), (4096, 64, 2000, 3001, 0.5),
                                                    (77, 256, 400, 900, 0.25), (1000, 3, 100, 97, 0.0)])
def test_candidates_and_bias_match_the_oracle(B, M, n_user, n_item, beta):
    from sslrec_b200 import engine as E
    m, rowptr, cols, _ = _graph(n_user, n_item, 10 * n_user, 21 + M)
    pop = E.PopTables(m.indptr, m.indices, n_item, beta, 'cuda')
    host = E.pop_tables(m.indptr, m.indices, n_item, beta)
    rs = np.random.RandomState(B + M)
    users = rs.randint(0, n_user, size=B)
    users[: min(B, 3)] = [0, 1, 0][: min(B, 3)]
    negs = rs.randint(0, n_item, size=B)
    seed = 0x0123456789ABCDEF ^ B
    ut, nt = torch.from_numpy(users).cuda(), torch.from_numpy(negs).cuda()
    got, bias = E.neg_candidates(ut, nt, M, rowptr, cols, n_item, seed, pop=pop, want_bias=True)
    want = O.neg_candidates(users, negs, M, m.indptr, m.indices, n_item, host['table'], seed)
    assert np.array_equal(got.cpu().numpy(), want)
    want_bias = O.bias(users, want, host['lp'], host['lz_pop'], host['lz_uni'])
    assert np.array_equal(bias.cpu().numpy().view(np.uint32), want_bias.view(np.uint32))
    dense = m.toarray() > 0
    rest = users > 1
    assert not dense[users[rest, None], want[rest, 1:]].any()
    # without the bias: the same candidates; the seed read from a device word (graph replay) wins over the host value
    assert torch.equal(E.neg_candidates(ut, nt, M, rowptr, cols, n_item, seed, pop=pop), got)
    word = torch.tensor([seed - (1 << 64) if seed >= 1 << 63 else seed], dtype=torch.int64, device='cuda')
    dseed = E.DevSeed(seed ^ 0x5555)
    dseed.ptr = word.data_ptr()
    got_dev, bias_dev = E.neg_candidates(ut, nt, M, rowptr, cols, n_item, dseed, pop=pop, want_bias=True)
    assert torch.equal(got_dev, got) and torch.equal(bias_dev, bias)


def test_graph_replay_draws_with_the_seed_written_before_it():
    from sslrec_b200 import engine as E
    m, rowptr, cols, _ = _graph(300, 501, 3000, 5)
    pop = E.PopTables(m.indptr, m.indices, 501, 0.75, 'cuda')
    host = E.pop_tables(m.indptr, m.indices, 501, 0.75)
    users = np.random.RandomState(0).randint(0, 300, 700)
    negs = np.random.RandomState(1).randint(0, 501, 700)
    ut, nt = torch.from_numpy(users).cuda(), torch.from_numpy(negs).cuda()
    word = torch.zeros(1, dtype=torch.int64, device='cuda')
    dseed = E.DevSeed(0)
    dseed.ptr = word.data_ptr()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.neg_candidates(ut, nt, 16, rowptr, cols, 501, dseed, pop=pop, want_bias=True)          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cands, bias = E.neg_candidates(ut, nt, 16, rowptr, cols, 501, dseed, pop=pop, want_bias=True)
    for seed in (7, 0x7EEDBEEF01234567, 99):
        word.fill_(seed)
        g.replay()
        torch.cuda.synchronize()
        want = O.neg_candidates(users, negs, 16, m.indptr, m.indices, 501, host['table'], seed)
        assert np.array_equal(cands.cpu().numpy(), want), seed
        assert np.array_equal(bias.cpu().numpy(), O.bias(users, want, host['lp'], host['lz_pop'], host['lz_uni'])), seed


def _one_user(n_item=60, beta=1.0):
    """A graph whose user 0 has a few popular and a few unpopular items; its non-positives keep at least half of the table's
    mass (Z_u >= 0.5), so the 128-draw cap is never reached in practice."""
    from sslrec_b200 import engine as E
    rs = np.random.RandomState(3)
    rows = rs.randint(1, 200, 4000)
    cols = (rs.zipf(1.3, 4000) - 1) % n_item
    pos = np.array([0, 2, 5, 31, 47])
    rows = np.concatenate([rows, np.zeros(len(pos), np.int64)])
    cols = np.concatenate([cols, pos])
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(200, n_item))
    m.sum_duplicates()
    m.sort_indices()
    host = E.pop_tables(m.indptr, m.indices, n_item, beta)
    z = 1 - host['V'][pos].sum() / float(n_item << 32)
    assert z >= 0.5, z
    pop = E.PopTables(m.indptr, m.indices, n_item, beta, 'cuda')
    dev = lambda a: torch.from_numpy(a.astype(np.int32)).cuda()
    return m, dev(m.indptr), dev(m.indices), pos, host, pop


def test_draws_follow_the_table_restricted_to_non_positives():
    from sslrec_b200 import engine as E
    n_item = 60
    m, rowptr, cols, pos, host, pop = _one_user(n_item)
    B, M = 1 << 14, 9
    users = torch.zeros(B, dtype=torch.int64, device='cuda')
    negs = torch.ones(B, dtype=torch.int64, device='cuda')
    cands = E.neg_candidates(users, negs, M, rowptr, cols, n_item, 0xC0FFEE, pop=pop)[:, 1:].reshape(-1).cpu().numpy()
    assert not np.isin(cands, pos).any()
    p = O.proposal(host['V'], pos)
    obs = np.bincount(cands, minlength=n_item)
    keep = p > 0
    chi2, pval = scipy.stats.chisquare(obs[keep], p[keep] * cands.size)
    assert pval > 1e-4, (chi2, pval)
    # a visibly different law fails the same test: the uniform law over the non-positives
    uni = keep / keep.sum()
    assert scipy.stats.chisquare(obs[keep], uni[keep] * cands.size)[1] < 1e-12


def test_logq_correction_is_an_unbiased_estimate():
    """sum_{q >= 1} exp(s_q - bias[q-1]) over the candidates of one user: its mean over 64 k pairs is
    sum_{i not in P_u} exp(s_i) within five standard errors; the column-0 negatives are uniform over the non-positives."""
    from sslrec_b200 import engine as E
    n_item = 60
    m, rowptr, cols, pos, host, pop = _one_user(n_item, beta=0.75)
    B, M = 1 << 16, 8
    rs = np.random.RandomState(8)
    free = np.setdiff1d(np.arange(n_item), pos)
    negs = torch.from_numpy(free[rs.randint(0, len(free), B)]).cuda()
    users = torch.zeros(B, dtype=torch.int64, device='cuda')
    cands, bias = E.neg_candidates(users, negs, M, rowptr, cols, n_item, 0xABCDEF, pop=pop, want_bias=True)
    # item scores that grow with popularity, so the uncorrected estimate is visibly biased
    s = torch.from_numpy(0.5 * np.log(host['V'] / host['V'].mean()) + 0.3 * rs.standard_normal(n_item)).cuda()
    est = torch.exp(s[cands] - bias.double()).sum(1)
    want = float(torch.exp(s[torch.from_numpy(free).cuda()]).sum())
    mean, se = float(est.mean()), float(est.std()) / math.sqrt(B)
    assert abs(mean - want) <= 5 * se, (mean, want, se)
    # without the correction the estimate is far off (the draw is not uniform)
    naive = float(torch.exp(s[cands]).sum(1).mean()) * len(free) / M
    assert abs(naive - want) > 20 * se, (naive, want, se)


# ---- the logQ forward --------------------------------------------------------------------------------------------------------

def _case(B, M, d, n_user=300, n_item=400, seed=0):
    g = torch.Generator().manual_seed(seed)
    users, items = torch.randn(n_user, d, generator=g), torch.randn(n_item, d, generator=g)
    ancs, poss = torch.randint(0, n_user, (B,), generator=g), torch.randint(0, n_item, (B,), generator=g)
    cands = torch.randint(0, n_item, (B, M), generator=g)
    ancs[::2] = ancs[::2] % 3
    cands[::3] = cands[::3] % 7
    bias = (torch.randn(B, M, generator=g) * 2 - 1).float()
    return users, items, ancs, poss, cands, bias


def _fwd(fn, users, items, ancs, poss, cands, tau, bias=None):
    from sslrec_b200._lib import lib
    B, M = cands.shape
    d = users.shape[1]
    f = dict(device='cuda', dtype=torch.float32)
    out = torch.empty(B, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 2, **f)
    a = [users.data_ptr(), d, items.data_ptr(), d, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, M, d, tau,
         *[t.data_ptr() for t in out]]
    if bias is not None:
        a.append(bias.data_ptr())
    assert getattr(lib, fn)(*a, torch.cuda.current_stream().cuda_stream) == 0
    return out


def _term64(users, items, ancs, poss, cands, bias, tau):
    s = S.scores64(users, items, ancs, poss, cands, tau)
    sh = torch.cat([s[:, :1], s[:, 1:] - bias.to(s.dtype)], 1)
    return (torch.logsumexp(sh, 1) - s[:, 0]).sum(), sh


@pytest.mark.parametrize('B,M,d,tau', [(1, 1, 4, 0.02), (333, 8, 32, 0.1), (4096, 64, 64, 0.02), (257, 256, 128, 0.2), (129, 31, 12, 0.5)])
def test_logq_forward_against_float32_and_float64(B, M, d, tau):
    from sslrec_b200 import engine as E
    users, items, ancs, poss, cands, bias = _case(B, M, d, seed=B + M)
    leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
    ac, pc, cc, bc = ancs.cuda(), poss.cuda(), cands.cuda(), bias.cuda()
    loss = E.ssm_loss_sum(leaves[0], leaves[1], ac, pc, cc, tau, bias=bc)
    assert torch.equal(loss, E.ssm_loss_sum(leaves[0], leaves[1], ac, pc, cc, tau, bias=bc))
    loss.backward()
    _, s, _, nrm = _fwd('ssl_ssm_fwd_logq', users.cuda(), items.cuda(), ac, pc, cc, tau, bc)
    u = users[ancs].numpy()
    c = items[torch.cat([poss[:, None], cands], 1)].numpy()
    _, w_s, _, w_nrm = O.forward32_logq(u, c, tau, bias.numpy(), expf=np.exp, logf=np.log)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), w_s.view(np.uint32))
    assert np.array_equal(nrm.cpu().numpy().view(np.uint32), w_nrm.view(np.uint32))
    # float64: the bounds of tests/test_gpu_ssm.py, with the softmax weights of s^
    ref_leaves = [t.double().cuda().requires_grad_(True) for t in (users, items)]
    ref, sh = _term64(ref_leaves[0], ref_leaves[1], ac, pc, cc, bc, tau)
    ref.backward()
    tol = 1e-5 * max(1.0, abs(ref.item())) + 4e-7 * B / tau + 2.4e-7 * B * float(bias.abs().max())   # + the rounding of s - bias
    assert abs(loss.item() - ref.item()) <= tol, (loss.item(), ref.item())
    u64, i64 = users.double().cuda(), items.double().cuda()
    ids = torch.cat([pc[:, None], cc], 1)
    ur, cr = u64[ac], i64[ids]
    nu = torch.sqrt(S.EPS + (ur * ur).sum(1))
    nq = torch.sqrt(S.EPS + (cr * cr).sum(2))
    sr = torch.einsum('bd,bqd->bq', ur, cr) / (nu[:, None] * nq * tau)
    wa = torch.softmax(sh.detach(), 1)
    wa[:, 0] += 1
    a = wa / (nu[:, None] * nq * tau)
    e = wa * sr.abs() / (nq * nq)
    gc = (a[..., None] * ur[:, None, :]).abs() + (e[..., None] * cr).abs()
    gu = (a[..., None] * cr).abs().sum(1) + ((wa * sr.abs()).sum(1) / (nu * nu))[:, None] * ur.abs()
    A = (torch.zeros_like(u64).index_add_(0, ac, gu), torch.zeros_like(i64).index_add_(0, ids.reshape(-1), gc.reshape(-1, d)))
    for got, want, amag in zip(leaves, ref_leaves, A):
        H.close(got.grad, want.grad, 2e-4, 2e-4 * amag.cpu().numpy() + 1e-12, 'grad')


def test_zero_bias_is_the_plain_forward():
    users, items, ancs, poss, cands, _ = _case(1000, 33, 64, seed=4)
    args = [t.cuda() for t in (users, items, ancs, poss, cands)]
    zero = torch.zeros(1000, 33, device='cuda')
    a = _fwd('ssl_ssm_fwd_logq', *args, 0.05, zero)
    b = _fwd('ssl_ssm_fwd', *args, 0.05)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_bad_arguments_are_rejected_and_write_nothing():
    from sslrec_b200._lib import lib
    dev = 'cuda'
    users = torch.zeros(4, dtype=torch.int64, device=dev)
    rowptr = torch.zeros(2, dtype=torch.int32, device=dev)
    cols = torch.zeros(1, dtype=torch.int32, device=dev)
    table = torch.zeros(10, 2, dtype=torch.int32, device=dev)
    fl = torch.zeros(10, device=dev)
    cands = torch.full((4, 8), -7, dtype=torch.int64, device=dev)
    bias = torch.full((4, 8), -7.0, device=dev)
    tbl = torch.zeros(10, 32, device=dev)
    outs = [torch.full((4,), -7.0, device=dev), torch.full((4, 9), -7.0, device=dev), torch.full((4, 9), -7.0, device=dev),
            torch.full((4, 10), -7.0, device=dev)]
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()

    def cand(B=4, M=8, n_item=10, nulls=(), table_ptr=None):
        a = [p(users), p(users), B, M, p(rowptr), p(cols), n_item, table_ptr or p(table), p(fl), p(fl), p(fl), 1.0, 1, None, p(cands),
             p(bias), s]
        for i in nulls:
            a[i] = None
        return lib.ssl_neg_candidates_pop(*a)

    def fwd(B=4, M=8, dim=32, st=32, tau=0.1, nulls=(), tbl_ptr=None):
        a = [tbl_ptr or p(tbl), st, p(tbl), st, p(users), p(users), p(cands), B, M, dim, tau] + [p(t) for t in outs] + [p(bias), s]
        for i in nulls:
            a[i] = None
        return lib.ssl_ssm_fwd_logq(*a)

    for rc in (cand(M=1), cand(M=257), cand(B=-1), cand(B=1 << 31), cand(n_item=0), cand(n_item=1 << 31), cand(nulls=(0,)),
               cand(nulls=(1,)), cand(nulls=(4,)), cand(nulls=(5,)), cand(nulls=(7,)), cand(nulls=(8,)), cand(nulls=(9,)),
               cand(nulls=(10,)), cand(nulls=(14,)), cand(table_ptr=p(table) + 4),
               fwd(M=0), fwd(M=257), fwd(dim=0), fwd(dim=30), fwd(dim=132), fwd(st=31), fwd(tau=0.0), fwd(tau=float('nan')), fwd(B=-1),
               fwd(tbl_ptr=p(tbl) + 4), fwd(nulls=(0,)), fwd(nulls=(6,)), fwd(nulls=(11,)), fwd(nulls=(14,)), fwd(nulls=(15,))):
        assert rc == -1
    assert cand(B=0) == 0 and fwd(B=0) == 0
    torch.cuda.synchronize()
    assert (cands == -7).all() and (bias == -7).all() and all((t == -7).all() for t in outs)


# ---- models ------------------------------------------------------------------------------------------------------------------

MODES = {'dns': {}, 'mixgcf': dict(mixgcf=True), 'ssm': dict(ssm_temperature=0.1)}


@pytest.mark.parametrize('key', BPR_MODELS)
def test_key_null_is_the_key_absent_bit_for_bit(key):
    from sslrec_b200.optim import FusedAdam
    runs = []
    for train in (dict(ssm_temperature=0.1), dict(ssm_temperature=0.1, neg_popularity=None), dict(ssm_temperature=0.1, neg_popularity=0.75)):
        m, _, _ = make_run(key, device='cuda', train=dict(deterministic=True, dns_candidates=8, **train))
        opt = FusedAdam(m.parameters(), lr=1e-2)
        runs.append(([_step(m, opt, b) for b in _batches(key, n=2)], m._seeds.count))
    (absent, n_absent), (null, n_null), (pop, n_pop) = runs
    assert n_absent == n_null == n_pop                   # the same seed sequence
    for k, (a, b) in enumerate(zip(absent, null)):
        _assert_equal(a, b, (key, k))
    assert all(torch.isfinite(t).all() for t in pop[0][0].values())
    assert not torch.equal(pop[0][0]['ssm_loss'], absent[0][0]['ssm_loss'])


def _train(key, mode, graphed, n=6):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    m, _, _ = make_run(key, device='cuda', train=dict(deterministic=True, dns_candidates=8, neg_popularity=0.75, **MODES[mode]))
    opt = FusedAdam(m.parameters(), lr=1e-2)
    batches = _batches(key, n=n)
    ncl = key == 'ncl'
    out = []
    if graphed:
        torch.manual_seed(0)
        step = GraphedStep(m, opt, batches[0], warmup=2, recluster=ncl)
        for k, b in enumerate(batches[1:], start=1):
            loss, parts = step(b, recluster=ncl and k == 3)
            out.append(loss.clone())
        step.close()
    else:
        m._graph_mode = key == 'hccf'             # the path GraphedStep takes
        torch.manual_seed(0)
        for k, b in enumerate([batches[0]] * 2 + batches[1:]):
            opt.zero_grad()
            loss, parts = m.cal_loss(b)
            loss.backward()
            opt.step()
            if k >= 2:
                out.append(loss.detach().clone())
        m._graph_mode = False
    torch.cuda.synchronize()
    return out, {n_: p.detach().clone() for n_, p in m.named_parameters()}


@pytest.mark.parametrize('mode', list(MODES))
@pytest.mark.parametrize('key', BPR_MODELS)
def test_two_runs_and_graph_replay_are_bit_identical(key, mode):
    first, second, graphed = _train(key, mode, False), _train(key, mode, False), _train(key, mode, True)
    for other, what in ((second, 'eager run 2'), (graphed, 'graph replay')):
        assert len(other[0]) == len(first[0]) == 5
        for k, (a, b) in enumerate(zip(first[0], other[0])):
            assert torch.equal(a, b), (key, mode, what, k)
        for n_ in first[1]:
            assert torch.equal(first[1][n_], other[1][n_]), (key, mode, what, n_)


@pytest.mark.parametrize('key,views', [('simgcl', (0, 2)), ('sgl', (0,))])
def test_restricted_views_mark_every_candidate(monkeypatch, key, views):
    from sslrec_b200 import engine as E
    m, _, _ = make_run(key, device='cuda', train=dict(ssm_temperature=0.1, dns_candidates=32, neg_popularity=1.0))
    seen = {}
    ssm_loss_sum = E.ssm_loss_sum

    def keep(users, items, ancs, poss, cands, temp, bias=None):
        seen['cands'], seen['bias'] = cands, bias
        return ssm_loss_sum(users, items, ancs, poss, cands, temp, bias=bias)

    monkeypatch.setattr(E, 'ssm_loss_sum', keep)
    loss, _ = m.cal_loss(_batches(key, n=1)[0])
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and seen['cands'].shape[1] == 32 and seen['bias'].shape == seen['cands'].shape
    st = m._state
    rows = (seen['cands'].reshape(-1) + m.user_num).cpu()
    for v in views:
        assert v in st.restricted_views
        bits = st.prop.views[v].row_bits.cpu().to(torch.int64)
        assert (((bits[rows >> 5] >> (rows & 31)) & 1) == 1).all(), v


@pytest.mark.parametrize('key', BPR_MODELS)
def test_beta_zero_bias_is_the_uniform_correction(monkeypatch, key):
    """beta = 0: every bias entry is ln M - ln(n_item - deg_u) within fp32 rounding, and the loss is the uncorrected float64
    term on the same candidates with every negative score shifted by it."""
    from sslrec_b200 import engine as E
    M, tau = 16, 0.1
    m, _, _ = make_run(key, device='cuda', train=dict(ssm_temperature=tau, dns_candidates=M, neg_popularity=0))
    seen = {}
    ssm_loss_sum = E.ssm_loss_sum

    def keep(users, items, ancs, poss, cands, temp, bias=None):
        seen.update(ancs=ancs, poss=poss, cands=cands, bias=bias)
        seen['loss'] = ssm_loss_sum(users, items, ancs, poss, cands, temp, bias=bias)
        return seen['loss']

    monkeypatch.setattr(E, 'ssm_loss_sum', keep)
    m.cal_loss(_batches(key, n=1)[0])
    torch.cuda.synchronize()
    rowptr, _ = m._train_csr(torch.device('cuda'))
    deg = (rowptr[1:] - rowptr[:-1]).double()
    ancs = seen['ancs']
    want = math.log(M) - torch.log(m.item_num - deg[ancs])
    b = seen['bias'].double()
    assert (b - want[:, None]).abs().max().item() <= 2.0 ** -21 * math.log(max(M, m.item_num))
    # the loss on the model's tables: ssl_ssm_fwd_logq against the float64 plain term with shifted negative scores
    users, items = torch.randn(m.user_num, 32, device='cuda'), torch.randn(m.item_num, 32, device='cuda')
    got = E.ssm_loss_sum(users, items, ancs, seen['poss'], seen['cands'], tau, bias=seen['bias'])
    s = S.scores64(users.double(), items.double(), ancs, seen['poss'], seen['cands'], tau)
    sh = torch.cat([s[:, :1], s[:, 1:] - want[:, None]], 1)
    ref = float((torch.logsumexp(sh, 1) - s[:, 0]).sum())
    B = ancs.numel()
    assert abs(got.item() - ref) <= 1e-5 * max(1.0, abs(ref)) + 4e-7 * B / tau + 2e-6 * B, (got.item(), ref)


# ---- whole steps against float64 ---------------------------------------------------------------------------------------------

POP_BETA = 0.75


def _whole_step_rows():
    """Every row of ``test_gpu_mixgcf.whole_step_rows(ssm=True)`` at beta 0.75; LightGCN and HCCF at hyper_num 128 also at beta
    1 and 0, d = 64, on both routes."""
    rows = [pytest.param(*p.values, POP_BETA, id=f'{p.id}-beta{POP_BETA}') for p in whole_step_rows(ssm=True)]
    for m, hp in (('lightgcn', {}), ('hccf', dict(hyper_num=128, keep_rate=0.5))):
        for beta in (1.0, 0.0):
            for det in (False, True):
                rows.append(pytest.param(m, 'paths', hp, 64, 8, H.BPR_TERM_TAU, det, beta, id=H.bpr_term_case_id(
                    (m, hp, 64, 8, H.BPR_TERM_TAU)) + ('-det' if det else '') + f'-beta{beta}'))
    return rows


@pytest.mark.parametrize('model_key,case_name,hp_over,dim,M,tau,deterministic,beta', _whole_step_rows())
def test_whole_step_against_float64(monkeypatch, model_key, case_name, hp_over, dim, M, tau, deterministic, beta):
    """The sampled softmax step with popularity candidates against float64:

    - the candidates and the fp32 bias the term received are tests/pop_oracle's draw and bias for the step's own pairs, last
      seed and training matrix, bit for bit (so the users are the anchors, column 0 the loader's negative, and the bias is this
      step's);
    - that bias is within pop_oracle.bias_tol of bias64, the float64 bias from its definition;
    - loss, every term and every parameter's gradient are within the path_errors bounds of the float64 oracle whose BPR term is
      pop_oracle.term64_logq on those candidates and bias64 (ssl_test_helpers.bpr_term_oracle);
    - the same step is outside those bounds of the uncorrected float64 term, so the correction matters on the row."""
    seen = {}
    got, cands, model, (case, hp, adj, dr, st) = whole_step(monkeypatch, model_key, case_name, hp_over, dim, M, deterministic,
                                                            dict(ssm_temperature=tau, neg_popularity=beta), 'ssm_loss_sum', 4, seen)
    assert model.neg_popularity == beta and 'bpr_loss' not in got['parts'] and seen['bias'] is not None
    want, want_bias = H.pop_draw(case, case['ancs'], case['negs'], M, beta, H.assert_step_seed(model))
    assert np.array_equal(cands.numpy(), want)
    bias = seen['bias'].cpu().numpy()
    assert np.array_equal(bias.view(np.uint32), want_bias.view(np.uint32))
    args = (case['ancs'], want, case['rows'], case['cols'], case['n_user'], case['n_item'], beta, M)
    b64 = O.bias64(*args)
    bias_frac = float((np.abs(bias - b64) / O.bias_tol(*args)).max())
    ancs, poss = torch.from_numpy(case['ancs']), torch.from_numpy(case['poss'])

    def ref(term):
        return H.bpr_term_oracle(model_key, case, hp, adj, dr, st, torch.float64, term, 'ssm_loss')

    errs = H.path_errors(got, ref(lambda u, i, _: O.term64_logq(u, i, ancs, poss, cands, tau, b64)))
    plain = H.path_errors(got, ref(lambda u, i, _: S.term64(u, i, ancs, poss, cands, tau)))
    worst = max(errs, key=errs.get)
    print(f'neg_popularity {model_key}-{case_name}-{hp_over}-d{dim}-M{M}-tau{tau}-beta{beta}{"-det" if deterministic else ""}: '
          f'largest error {errs[worst]:.3f} of its bound ({worst}); bias {bias_frac:.3f} of its bound; uncorrected term '
          f'{max(plain.values()):.3g}x its bound')
    assert bias_frac <= 1.0, bias_frac
    assert errs[worst] <= 1.0, errs
    assert max(plain.values()) > 1.0, ('the uncorrected term passes', plain)


@pytest.mark.parametrize('key', BPR_MODELS)
def test_every_step_applies_its_own_bias(monkeypatch, key):
    """Two cal_loss calls on different batches: each passes the sampled softmax the bias of its own candidates and users, and
    its candidates are the draw of its own seed (a bias kept from an earlier step would match the other batch)."""
    from sslrec_b200 import engine as E
    from oracle import inputs
    m, _, _ = make_run(key, device='cuda', train=dict(deterministic=True, ssm_temperature=0.1, dns_candidates=8,
                                                      neg_popularity=POP_BETA))
    case = inputs.make_case('tiny')
    seen = []
    ssm_loss_sum = E.ssm_loss_sum

    def keep(users, items, ancs, poss, cands, temp, bias=None):
        seen.append((ancs.clone(), cands.clone(), None if bias is None else bias.clone()))
        return ssm_loss_sum(users, items, ancs, poss, cands, temp, bias=bias)

    monkeypatch.setattr(E, 'ssm_loss_sum', keep)
    biases = []
    for k, batch in enumerate(_batches(key, n=2)):
        loss, _ = m.cal_loss(batch)
        loss.backward()
        torch.cuda.synchronize()
        assert len(seen) == k + 1
        ancs, cands, bias = (t.cpu().numpy() for t in seen[k])
        assert np.array_equal(ancs, batch[0].cpu().numpy())
        want, want_bias = H.pop_draw(case, ancs, batch[2].cpu().numpy(), 8, POP_BETA, H.assert_step_seed(m))
        assert np.array_equal(cands, want), k
        assert np.array_equal(bias.view(np.uint32), want_bias.view(np.uint32)), k
        biases.append(bias)
    assert not np.array_equal(*biases)


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('key,hp', [('simgcl', {}), ('ncl', {'epoch_period': 2})])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph):
    import test_gpu_resume as R
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, dns_candidates=8, ssm_temperature=0.1, neg_popularity=0.75)
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
