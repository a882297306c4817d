"""The sampled softmax loss (optional key train.ssm_temperature) on the GPU.

Kernels, through ``engine.ssm_loss_sum`` and the C ABI: the scores and norms equal the float32 restatement of
tests/ssm_oracle.forward32 bit for bit (every FMA emulated exactly; they involve no exp or log); the loss and every gradient row
are within the fp32 bound stated below of the float64 term on duplicate-heavy batches; the train.deterministic route equals its
restatement (the staged per-position contributions added in position order) bit for bit; a relaunch is bit-identical; rejected
arguments write nothing.

Models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL): the key absent is the key null bit for bit, and with M = 1 the step draws
the plain step's seeds; under train.deterministic two runs and a CUDA-graph replay are bit-identical; SimGCL's and SGL's
restricted views mark every candidate.  All six, on both gradient routes: the whole step equals the float64 oracle
(oracle/cf_oracle with the injected masks, noise, k-means state and SVD factors, its BPR term replaced by tests/ssm_oracle.term64
on the step's candidates over the tables of ssl_test_helpers.bpr_tables) within the golden tolerances, for every parameter's
gradient, on the goldens and on the cases of tests/test_gpu_mixgcf.whole_step_rows (also at tau 0.02); tests/test_host_ssm.py
shows on the host that the float32 oracle meets these bounds and one at tau (1 + 1e-3) does not.  SimGCL and NCL resumed from a
mid-run checkpoint end bit-identical to an uninterrupted run."""
import ctypes as C

import numpy as np
import pytest
import torch

import ssl_test_helpers as H
import ssm_oracle as S
from test_gpu_hard_negatives import _assert_equal, _batches, _step
from test_gpu_mixgcf import whole_step, whole_step_rows
from test_host_resume import make_run

pytestmark = pytest.mark.gpu

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def _case(B, M, d, n_user=300, n_item=400, seed=0):
    """Tables and a duplicate-heavy batch: half of the pairs share a few users and positives, a third of the candidate rows a
    few items, and some candidates are the pair's positive."""
    g = torch.Generator().manual_seed(seed)
    users, items = torch.randn(n_user, d, generator=g), torch.randn(n_item, d, generator=g)
    ancs, poss = torch.randint(0, n_user, (B,), generator=g), torch.randint(0, n_item, (B,), generator=g)
    cands = torch.randint(0, n_item, (B, M), generator=g)
    ancs[::2] = ancs[::2] % 3
    poss[::2] = poss[::2] % 5
    cands[::3] = cands[::3] % 7
    cands[::4, -1] = poss[::4]
    return users, items, ancs, poss, cands


def _fwd(users, items, ancs, poss, cands, tau):
    from sslrec_b200._lib import lib
    B, M = cands.shape
    d = users.shape[1]
    f = dict(device='cuda', dtype=torch.float32)
    out = torch.empty(B, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 2, **f)
    assert lib.ssl_ssm_fwd(users.data_ptr(), d, items.data_ptr(), d, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, M, d, tau,
                           *[t.data_ptr() for t in out], torch.cuda.current_stream().cuda_stream) == 0
    return out


@pytest.mark.parametrize('B,M,d,tau', [(1, 1, 4, 0.02), (333, 8, 32, 0.1), (4096, 64, 64, 0.02), (257, 256, 128, 0.2), (70, 33, 48, 1.0),
                                       (129, 31, 12, 0.02)])
def test_scores_relaunch_and_float64_bound(B, M, d, tau):
    from sslrec_b200 import engine as E
    users, items, ancs, poss, cands = _case(B, M, d, seed=B + M)
    leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
    ac, pc, cc = ancs.cuda(), poss.cuda(), cands.cuda()
    loss = E.ssm_loss_sum(leaves[0], leaves[1], ac, pc, cc, tau)
    again = E.ssm_loss_sum(leaves[0], leaves[1], ac, pc, cc, tau)
    assert torch.equal(loss, again)
    loss.backward()
    # scores and norms: the documented fp32 arithmetic, bit for bit
    _, s, _, nrm = _fwd(users.cuda(), items.cuda(), ac, pc, cc, tau)
    u = users[ancs].numpy()
    c = items[torch.cat([poss[:, None], cands], 1)].numpy()
    _, w_s, _, w_nrm = S.forward32(u, c, tau, expf=np.exp, logf=np.log)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), w_s.view(np.uint32))
    assert np.array_equal(nrm.cpu().numpy().view(np.uint32), w_nrm.view(np.uint32))
    # float64 term; fp32 bound: |loss| within 1e-5 max(1, |ref|) + 4e-7 B / tau (each scale-1/tau score carries ~d/2 ulp of a
    # unit cosine); every gradient element within 2e-4 (|ref| + A), A the element's sum of the magnitudes of its per-position
    # terms in float64 (w_0 = p_0 - 1 counted as p_0 + 1, the size of the operands of its subtraction): a term's error is of
    # the order of d u / tau of that magnitude through the scores (u = 2^-24), and the float atomics add up to B (M + 2) terms
    # into one row in any order, so on duplicate-heavy rows and confident pairs the error scales with A, not with the
    # (cancelling) result
    ref_leaves = [t.double().cuda().requires_grad_(True) for t in (users, items)]
    ref = S.term64(ref_leaves[0], ref_leaves[1], ac, pc, cc, tau)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(1.0, abs(ref.item())) + 4e-7 * B / tau, (loss.item(), ref.item())
    for got, want, a in zip(leaves, ref_leaves, _abs_contributions(users, items, ac, pc, cc, tau)):
        H.close(got.grad, want.grad, 2e-4, 2e-4 * a.cpu().numpy() + 1e-12, 'grad')


def _abs_contributions(users, items, ancs, poss, cands, tau):
    """float64 [n_user, d], [n_item, d]: per element the sum of |contribution| over the positions that add into it (the
    backward's terms of include/sslrec_b200.h, a26)."""
    u, it = users.double().cuda(), items.double().cuda()
    ids = torch.cat([poss[:, None], cands], 1)
    ur, cr = u[ancs], it[ids]                                            # [B, d], [B, M+1, d]
    nu = torch.sqrt(S.EPS + (ur * ur).sum(1))
    nq = torch.sqrt(S.EPS + (cr * cr).sum(2))
    s = torch.einsum('bd,bqd->bq', ur, cr) / (nu[:, None] * nq * tau)
    wa = torch.softmax(s, 1)
    wa[:, 0] += 1                    # |w_0| = |p_0 - 1| is formed by a subtraction of operands up to p_0 + 1 in magnitude
    a = wa / (nu[:, None] * nq * tau)
    e = wa * s.abs() / (nq * nq)
    gc = (a[..., None] * ur[:, None, :]).abs() + (e[..., None] * cr).abs()
    gu = (a[..., None] * cr).abs().sum(1) + ((wa * s.abs()).sum(1) / (nu * nu))[:, None] * ur.abs()
    A_u = torch.zeros_like(u).index_add_(0, ancs, gu)
    A_i = torch.zeros_like(it).index_add_(0, ids.reshape(-1), gc.reshape(-1, u.shape[1]))
    return A_u, A_i


def test_nan_score_makes_the_loss_nan():
    from sslrec_b200 import engine as E
    users, items, ancs, poss, cands = (t.cuda() for t in _case(8, 4, 16))
    items[cands[3, 2]] = float('nan')
    lb = _fwd(users, items, ancs, poss, cands, 0.1)[0]
    bad = (cands == cands[3, 2]).any(1) | (poss == cands[3, 2])
    assert torch.isnan(lb[bad]).all() and torch.isfinite(lb[~bad]).all()
    assert torch.isnan(E.ssm_loss_sum(users, items, ancs, poss, cands, 0.1))


def test_deterministic_route_is_its_ordered_restatement(monkeypatch):
    """Under train.deterministic every sink row is sink + (((c_p1 + c_p2) + ...)) over its positions in order, the c_p being
    the kernel's staged contributions (numbering in csrc/ssm.cuh); restated here with one torch add per position."""
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import lib
    monkeypatch.setattr(E, 'DETERMINISTIC', True)
    B, M, d, tau = 300, 8, 32, 0.05
    users, items, ancs, poss, cands = _case(B, M, d, seed=3)
    leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
    ac, pc, cc = ancs.cuda(), poss.cuda(), cands.cuda()
    (E.ssm_loss_sum(leaves[0], leaves[1], ac, pc, cc, tau) * 0.5).backward()
    _, s, w, nrm = _fwd(leaves[0].detach(), leaves[1].detach(), ac, pc, cc, tau)
    ids = torch.cat([pc, cc.view(-1)])
    ug, ig = leaves[0].detach()[ac].contiguous(), leaves[1].detach()[ids].contiguous()
    ar = torch.arange(B, device='cuda')
    ci = torch.arange(B, B * (M + 1), device='cuda')
    f = dict(device='cuda', dtype=torch.float32)
    su, si = torch.full((B, d), -0.0, **f), torch.full((B * (M + 1), d), -0.0, **f)
    half = torch.tensor(0.5, **f)
    assert lib.ssl_ssm_bwd(ug.data_ptr(), d, ig.data_ptr(), d, ar.data_ptr(), ar.data_ptr(), ci.data_ptr(), B, M, d, tau, s.data_ptr(),
                           w.data_ptr(), nrm.data_ptr(), half.data_ptr(), 1.0, su.data_ptr(), d, si.data_ptr(), d,
                           torch.cuda.current_stream().cuda_stream) == 0

    def ordered(n_rows, stage, rows):
        sink = torch.zeros(n_rows, d, **f)
        for p, r in enumerate(rows.tolist()):
            sink[r] = sink[r] + stage[p]
        return sink

    assert torch.equal(leaves[0].grad, ordered(users.shape[0], su, ac))
    assert torch.equal(leaves[1].grad, ordered(items.shape[0], si, ids))


def test_bad_arguments_are_rejected_and_write_nothing():
    from sslrec_b200._lib import lib
    dev = 'cuda'
    ids = torch.zeros(4, dtype=torch.int64, device=dev)
    cands = torch.zeros(4, 8, dtype=torch.int64, device=dev)
    tbl = torch.zeros(10, 32, device=dev)
    outs = [torch.full((4,), -7.0, device=dev), torch.full((4, 9), -7.0, device=dev), torch.full((4, 9), -7.0, device=dev),
            torch.full((4, 10), -7.0, device=dev)]
    sink = torch.full((10, 32), -7.0, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    tp = p(tbl)

    def fwd(B=4, M=8, dim=32, st=32, tau=0.1, nulls=(), tbl_ptr=tp):
        a = [tbl_ptr, st, tp, st, p(ids), p(ids), p(cands), B, M, dim, tau] + [p(t) for t in outs] + [s]
        for i in nulls:
            a[i] = None
        return lib.ssl_ssm_fwd(*a)

    def bwd(B=4, M=8, dim=32, st=32, gst=32, tau=0.1, nulls=(), sink_ptr=None):
        a = [tp, st, tp, st, p(ids), p(ids), p(cands), B, M, dim, tau, p(outs[1]), p(outs[2]), p(outs[3]), None, 1.0, p(sink), gst,
             sink_ptr or p(sink), gst, s]
        for i in nulls:
            a[i] = None
        return lib.ssl_ssm_bwd(*a)

    for rc in (fwd(M=0), fwd(M=257), fwd(dim=0), fwd(dim=30), fwd(dim=132), fwd(st=31), fwd(st=34), fwd(tau=0.0), fwd(tau=-1.0),
               fwd(tau=float('inf')), fwd(tau=float('nan')), fwd(B=-1), fwd(B=1 << 31), fwd(tbl_ptr=tp + 4),
               fwd(nulls=(0,)), fwd(nulls=(2,)), fwd(nulls=(4,)), fwd(nulls=(5,)), fwd(nulls=(6,)), fwd(nulls=(11,)), fwd(nulls=(14,)),
               bwd(M=0), bwd(M=257), bwd(dim=36 + 100), bwd(st=31), bwd(gst=30), bwd(tau=0.0), bwd(B=-2), bwd(sink_ptr=p(sink) + 8),
               bwd(nulls=(0,)), bwd(nulls=(6,)), bwd(nulls=(11,)), bwd(nulls=(13,)), bwd(nulls=(16,)), bwd(nulls=(18,))):
        assert rc == -1
    assert fwd(B=0) == 0 and bwd(B=0) == 0
    torch.cuda.synchronize()
    assert all((t == -7).all() for t in outs) and (sink == -7).all()


# ---- models ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('key', BPR_MODELS)
def test_key_null_is_the_key_absent_bit_for_bit(key):
    from sslrec_b200.optim import FusedAdam
    runs = []
    for train in (dict(deterministic=True), dict(deterministic=True, ssm_temperature=None), dict(deterministic=True, ssm_temperature=0.1)):
        m, _, _ = make_run(key, device='cuda', train=train)
        opt = FusedAdam(m.parameters(), lr=1e-2)
        runs.append(([_step(m, opt, b) for b in _batches(key, n=2)], m._seeds.count))
    (plain, n_plain), (null, n_null), (ssm, n_ssm) = runs
    assert n_plain == n_null == n_ssm               # M = 1: the loader's negatives, no extra seed
    for k, (a, b) in enumerate(zip(plain, null)):
        _assert_equal(a, b, (key, k))
    assert 'ssm_loss' in ssm[0][0] and 'bpr_loss' not in ssm[0][0] and 'bpr_loss' in plain[0][0]
    assert all(torch.isfinite(t).all() for t in ssm[0][0].values())


def _train(key, graphed, n=6):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    m, _, _ = make_run(key, device='cuda', train=dict(deterministic=True, ssm_temperature=0.1, dns_candidates=8))
    opt = FusedAdam(m.parameters(), lr=1e-2)
    batches = _batches(key, n=n)
    ncl = key == 'ncl'
    out = []
    if graphed:
        torch.manual_seed(0)
        step = GraphedStep(m, opt, batches[0], warmup=2, recluster=ncl)
        for k, b in enumerate(batches[1:], start=1):
            loss, parts = step(b, recluster=ncl and k == 3)
            out.append((loss.clone(), parts['ssm_loss'].clone()))
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
                out.append((loss.detach().clone(), parts['ssm_loss'].detach().clone()))
        m._graph_mode = False
    torch.cuda.synchronize()
    assert m.dns_negs is None
    return out, {n_: p.detach().clone() for n_, p in m.named_parameters()}


@pytest.mark.parametrize('key', BPR_MODELS)
def test_two_runs_and_graph_replay_are_bit_identical(key):
    first, second, graphed = _train(key, False), _train(key, False), _train(key, True)
    for other, what in ((second, 'eager run 2'), (graphed, 'graph replay')):
        assert len(other[0]) == len(first[0]) == 5
        for k, (a, b) in enumerate(zip(first[0], other[0])):
            assert all(torch.equal(x, y) for x, y in zip(a, b)), (key, what, k)
        for n_ in first[1]:
            assert torch.equal(first[1][n_], other[1][n_]), (key, what, n_)


@pytest.mark.parametrize('key,views', [('simgcl', (0, 2)), ('sgl', (0,))])
def test_restricted_views_mark_every_candidate(monkeypatch, key, views):
    from sslrec_b200 import engine as E
    m, _, _ = make_run(key, device='cuda', train=dict(ssm_temperature=0.1, dns_candidates=32))
    seen = {}
    ssm_loss_sum = E.ssm_loss_sum

    def keep(users, items, ancs, poss, cands, temp):
        seen['cands'] = cands
        return ssm_loss_sum(users, items, ancs, poss, cands, temp)

    monkeypatch.setattr(E, 'ssm_loss_sum', keep)
    loss, parts = m.cal_loss(_batches(key, n=1)[0])
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and seen['cands'].shape[1] == 32
    st = m._state
    rows = (seen['cands'].reshape(-1) + m.user_num).cpu()
    for v in views:
        assert v in st.restricted_views
        bits = st.prop.views[v].row_bits.cpu().to(torch.int64)
        assert (((bits[rows >> 5] >> (rows & 31)) & 1) == 1).all(), v


@pytest.mark.parametrize('model_key,case_name,hp_over,dim,M,tau,deterministic', whole_step_rows(ssm=True))
def test_whole_step_against_float64(monkeypatch, model_key, case_name, hp_over, dim, M, tau, deterministic):
    """The step equals the float64 oracle with its BPR term replaced by ssm_oracle.term64 on the step's candidates
    (ssl_test_helpers.bpr_term_oracle): loss, every term and every parameter's gradient within the path_errors bounds."""
    got, cands, model, (case, hp, adj, dr, st) = whole_step(monkeypatch, model_key, case_name, hp_over, dim, M, deterministic,
                                                            dict(ssm_temperature=tau), 'ssm_loss_sum', 4)
    assert model.ssm_temperature == tau and 'bpr_loss' not in got['parts']
    ancs, poss = torch.from_numpy(case['ancs']), torch.from_numpy(case['poss'])
    ref = H.bpr_term_oracle(model_key, case, hp, adj, dr, st, torch.float64,
                            lambda u, i, _: S.term64(u, i, ancs, poss, cands, tau), 'ssm_loss')
    errs = H.path_errors(got, ref)
    worst = max(errs, key=errs.get)
    print(f'ssm {model_key}-{case_name}-{hp_over}-d{dim}-M{M}-tau{tau}{"-det" if deterministic else ""}: largest error '
          f'{errs[worst]:.3f} of its bound ({worst})')
    assert errs[worst] <= 1.0, errs


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('key,hp', [('simgcl', {}), ('ncl', {'epoch_period': 2})])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph):
    import test_gpu_resume as R
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, dns_candidates=8, ssm_temperature=0.1)
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
