"""MixGCF negatives (optional key train.mixgcf) on the GPU.

Kernels, through ``engine.mixgcf_bpr_sum`` and the C ABI: the mixing weights equal tests/mixgcf_oracle.alpha bit for bit, also
from the device seed word and in a CUDA-graph replay that reads a new seed; the picks equal a float32 restatement of the
documented arithmetic (every FMA of the chains emulated exactly in float64 and rounded once); the loss and every gradient row
are within the fp32 bound stated below of the float64 term on duplicate-heavy batches; the train.deterministic route equals its
restatement (the staged per-position contributions added in position order) bit for bit; a relaunch is bit-identical; rejected
arguments write nothing.

Models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL): the key false is the key absent bit for bit; under train.deterministic two
runs and a CUDA-graph replay are bit-identical; with injected alpha = 0 and M = 1 the loss and gradients equal the plain step
within fp32 rounding.  All six, on both gradient routes: the whole step equals the float64 oracle (oracle/cf_oracle with the
injected masks, noise, k-means state and SVD factors, its BPR term replaced by the MixGCF term of tests/mixgcf_oracle on the
model's own alpha and picks over the layer tables of ssl_test_helpers.bpr_tables) within the golden tolerances, for every
parameter's gradient, on the goldens and on the split-hub graph of ssl_test_helpers.path_case at d = 20, 64, 128 (NCL's context
layer beyond, inside and at the last mixed layer; HCCF at two hyper widths), and at d = 64 with train.neg_popularity, whose
candidates are tests/pop_oracle's draw for the step's seed bit for bit; its picks are float64's wherever the score gap is
decided.  tests/test_host_mixgcf.py shows on the host that the float32 oracle meets these bounds and slightly wrong MixGCF terms
do not.  SimGCL and NCL resumed from a mid-run checkpoint end bit-identical to an uninterrupted run."""
import numpy as np
import pytest
import torch

import mixgcf_oracle as X
import ssl_test_helpers as H
from oracle import cf_oracle as O
from oracle import inputs, replay
from test_gpu_hard_negatives import _assert_equal, _batches, _step
from test_host_resume import make_run

pytestmark = pytest.mark.gpu

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def _case(B, M, L1, d, n_user=300, n_item=400, seed=0, dup=True):
    """Tables and a batch; ``dup``: half of the pairs share a few users, positives and candidates (duplicate-heavy)."""
    g = torch.Generator().manual_seed(seed)
    users, items = torch.randn(n_user, d, generator=g), torch.randn(n_item, d, generator=g)
    layers = [torch.randn(n_item, d, generator=g) * 0.5 for _ in range(L1)]
    ancs, poss = torch.randint(0, n_user, (B,), generator=g), torch.randint(0, n_item, (B,), generator=g)
    cands = torch.randint(0, n_item, (B, M), generator=g)
    if dup:
        ancs[::2] = ancs[::2] % 3
        poss[::2] = poss[::2] % 5
        cands[::3] = cands[::3] % 7
    return users, items, layers, ancs, poss, cands


def _f32(x):
    return x.float().double()


def _fma(a, b, c):
    """fp32 fmaf on float64 carriers: a * b is exact in float64, the sum is rounded once to float64 and then to float32 (double
    rounding differs from fmaf only when the float64 sum lies exactly halfway between two float32 values, which these random
    inputs do not produce)."""
    return _f32(a * b + c)


def _restated_picks(users, layers, ancs, poss, cands, alpha):
    """[B, L+1] picks of the documented float32 arithmetic: m = fmaf(a, X[p], (1 - a) X[c]), s = sequential FMA chain over k."""
    u = users.double().cuda()[ancs]                                     # [B, d]
    a = alpha.double().cuda()[:, None, :, None]
    a1 = _f32(1 - a)
    xp = torch.stack([x.double().cuda()[poss] for x in layers], 1)[:, None]
    xc = torch.stack([x.double().cuda()[cands] for x in layers], 2)     # [B, M, L+1, d]
    m = _fma(a, xp, _f32(a1 * xc))
    s = torch.zeros(m.shape[:3], dtype=torch.float64, device='cuda')
    for k in range(m.shape[3]):
        s = _fma(u[:, None, None, k], m[..., k], s)
    s = torch.where(torch.isnan(s), torch.full_like(s, -float('inf')), s)
    j = torch.argmax((s == s.max(1, keepdim=True).values).to(torch.int8), dim=1)
    return cands.cuda().gather(1, j)


@pytest.mark.parametrize('B,M,L1,d', [(1, 1, 1, 4), (333, 8, 4, 32), (4096, 64, 4, 64), (257, 256, 8, 128), (70, 33, 3, 60)])
def test_alpha_picks_relaunch_and_float64_bound(B, M, L1, d):
    from sslrec_b200 import engine as E
    users, items, layers, ancs, poss, cands = _case(B, M, L1, d, seed=B + M)
    seed = 0x0123456789ABCDEF ^ B
    leaves = [t.cuda().requires_grad_(True) for t in [users, items] + layers]
    ac, pc, cc = ancs.cuda(), poss.cuda(), cands.cuda()
    loss, picks, alpha = E.mixgcf_bpr_sum(leaves[0], leaves[1], leaves[2:], ac, pc, cc, seed)
    assert np.array_equal(alpha.cpu().numpy(), X.alpha(B, L1, seed))
    assert torch.equal(picks, _restated_picks(users, layers, ancs, poss, cands, alpha.cpu()))
    again = E.mixgcf_bpr_sum(leaves[0], leaves[1], leaves[2:], ac, pc, cc, seed)
    assert all(torch.equal(x, y) for x, y in zip((loss, picks, alpha), again))
    loss.backward()
    # float64 term on the same alpha and picks; fp32 bound (the golden tolerances): |loss| within 1e-5 max(1, |ref|), every
    # gradient element within 2e-4 |ref| + 5e-6 max|ref| (d-term FMA chains, at most 2 B (L + 1) atomic adds per row, u = 2^-24)
    ref_leaves = [t.double().cuda().requires_grad_(True) for t in [users, items] + layers]
    ref = X.term(ref_leaves[0], ref_leaves[1], ref_leaves[2:], ac, pc, picks, alpha)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(1.0, abs(ref.item()))
    for got, want in zip(leaves, ref_leaves):
        H.close(got.grad, want.grad, 2e-4, 5e-6 * want.grad.abs().max().item() + 1e-12, 'grad')
    # the fp32 picks agree with the float64 argmax on almost every pair (they may differ only where the top two nearly tie)
    p64 = X.picks(users, layers, ancs, poss, cands, alpha.cpu())
    assert (p64.cuda() == picks).float().mean() > 0.9


def test_device_seed_and_graph_replay_draw_the_oracle_alpha():
    from sslrec_b200 import engine as E
    B, M, L1, d = 500, 8, 4, 64
    users, items, layers, ancs, poss, cands = (t.cuda() if torch.is_tensor(t) else [x.cuda() for x in t] for t in _case(B, M, L1, d))
    s1, s2 = 0x1111222233334444, 0x7777000011112222
    word = torch.tensor([s1], dtype=torch.int64, device='cuda')
    dseed = E.DevSeed(s1 ^ 0x5555)              # a wrong host value: the device word must win
    dseed.ptr = word.data_ptr()
    with torch.no_grad():
        _, _, alpha = E.mixgcf_bpr_sum(users, items, layers, ancs, poss, cands, dseed)
        assert np.array_equal(alpha.cpu().numpy(), X.alpha(B, L1, s1))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            out = E.mixgcf_bpr_sum(users, items, layers, ancs, poss, cands, dseed)
        torch.cuda.current_stream().wait_stream(s)
        word.fill_(s2)
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out[2].cpu().numpy(), X.alpha(B, L1, s2))
        assert torch.equal(out[1], E.mixgcf_bpr_sum(users, items, layers, ancs, poss, cands, s2)[1])


def test_deterministic_route_is_its_ordered_restatement(monkeypatch):
    """Under train.deterministic every sink row is sink + (((c_p1 + c_p2) + ...)) over its positions in order, the c_p being
    the kernel's staged contributions (numbering in csrc/mixgcf.cuh); restated here with one torch add per position."""
    import ctypes as C
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import lib
    monkeypatch.setattr(E, 'DETERMINISTIC', True)
    B, M, L1, d = 300, 8, 3, 32
    users, items, layers, ancs, poss, cands = _case(B, M, L1, d, seed=3)
    leaves = [t.cuda().requires_grad_(True) for t in [users, items] + layers]
    ac, pc, cc = ancs.cuda(), poss.cuda(), cands.cuda()
    loss, picks, alpha = E.mixgcf_bpr_sum(leaves[0], leaves[1], leaves[2:], ac, pc, cc, 99)
    (loss * 0.5).backward()
    # the restatement: forward through the C ABI for coef and nhat, then the staged backward
    f = dict(device='cuda', dtype=torch.float32)
    lb, coef, nhat = torch.empty(B, **f), torch.empty(B, **f), torch.empty(B, d, **f)
    pk, al = torch.empty(B, L1, dtype=torch.int64, device='cuda'), torch.empty(B, L1, **f)
    lt = [t.detach() for t in leaves[2:]]
    s = torch.cuda.current_stream().cuda_stream
    assert lib.ssl_mixgcf_bpr_fwd(leaves[0].data_ptr(), d, leaves[1].data_ptr(), d, (C.c_void_p * L1)(*[t.data_ptr() for t in lt]),
                                  (C.c_int64 * L1)(*[d] * L1), L1, ac.data_ptr(), pc.data_ptr(), cc.data_ptr(), B, M, d, 99, None, None,
                                  lb.data_ptr(), coef.data_ptr(), pk.data_ptr(), al.data_ptr(), nhat.data_ptr(), s) == 0
    assert torch.equal(pk, picks) and torch.equal(al, alpha)
    ug, pg = leaves[0].detach()[ac].contiguous(), leaves[1].detach()[pc].contiguous()
    ar = torch.arange(B, device='cuda')
    ids = (ar + B)[:, None].expand(B, L1).contiguous()
    su, si = torch.full((B, d), -0.0, **f), torch.full((B, d), -0.0, **f)
    sl = [torch.full((2 * B, d), -0.0, **f) for _ in range(L1)]
    half = torch.tensor(0.5, **f)
    assert lib.ssl_mixgcf_bpr_bwd(ug.data_ptr(), d, pg.data_ptr(), d, ar.data_ptr(), ar.data_ptr(), ids.data_ptr(), B, L1, d,
                                  nhat.data_ptr(), al.data_ptr(), coef.data_ptr(), half.data_ptr(), 1.0, su.data_ptr(), d, si.data_ptr(), d,
                                  (C.c_void_p * L1)(*[t.data_ptr() for t in sl]), (C.c_int64 * L1)(*[d] * L1), s) == 0

    def ordered(n_rows, stage, rows):
        sink = torch.zeros(n_rows, d, **f)
        for p, r in enumerate(rows.tolist()):
            sink[r] = sink[r] + stage[p]
        return sink

    assert torch.equal(leaves[0].grad, ordered(users.shape[0], su, ac))
    assert torch.equal(leaves[1].grad, ordered(items.shape[0], si, pc))
    for l in range(L1):
        assert torch.equal(leaves[2 + l].grad, ordered(items.shape[0], sl[l], torch.cat([pc, picks[:, l]]))), l


def test_bad_arguments_are_rejected_and_write_nothing():
    import ctypes as C
    from sslrec_b200._lib import lib
    dev = 'cuda'
    ids = torch.zeros(4, dtype=torch.int64, device=dev)
    cands = torch.zeros(4, 8, dtype=torch.int64, device=dev)
    tbl = torch.zeros(10, 32, device=dev)
    outs = [torch.full((4,), -7.0, device=dev), torch.full((4,), -7.0, device=dev), torch.full((4, 2), -7, dtype=torch.int64, device=dev),
            torch.full((4, 2), -7.0, device=dev), torch.full((4, 32), -7.0, device=dev)]
    sink = torch.full((10, 32), -7.0, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()

    def fwd(B=4, M=8, L1=2, dim=32, st=32, lst=32, nulls=(), null_layer=False):
        a = [p(tbl), st, p(tbl), st, (C.c_void_p * 2)(p(tbl), None if null_layer else p(tbl)), (C.c_int64 * 2)(lst, 32), L1, p(ids), p(ids),
             p(cands), B, M, dim, 1, None, None] + [p(t) for t in outs] + [s]
        for i in nulls:
            a[i] = None
        return lib.ssl_mixgcf_bpr_fwd(*a)

    def bwd(B=4, L1=2, dim=32, st=32, gst=32, nulls=(), null_layer=False):
        a = [p(tbl), st, p(tbl), st, p(ids), p(ids), p(outs[2]), B, L1, dim, p(outs[4]), p(outs[3]), p(outs[1]), None, 1.0, p(sink), gst,
             p(sink), gst, (C.c_void_p * 2)(p(sink), None if null_layer else p(sink)), (C.c_int64 * 2)(gst, 32), s]
        for i in nulls:
            a[i] = None
        return lib.ssl_mixgcf_bpr_bwd(*a)

    for rc in (fwd(M=0), fwd(M=257), fwd(L1=0), fwd(L1=9), fwd(dim=0), fwd(dim=129), fwd(st=31), fwd(lst=16), fwd(B=-1), fwd(B=1 << 31),
               fwd(nulls=(0,)), fwd(nulls=(2,)), fwd(nulls=(4,)), fwd(nulls=(5,)), fwd(nulls=(7,)), fwd(nulls=(8,)), fwd(nulls=(9,)),
               fwd(nulls=(16,)), fwd(nulls=(20,)), fwd(null_layer=True),
               bwd(L1=0), bwd(L1=9), bwd(dim=129), bwd(st=31), bwd(gst=16), bwd(B=-2), bwd(nulls=(0,)), bwd(nulls=(6,)),
               bwd(nulls=(10,)), bwd(nulls=(15,)), bwd(nulls=(19,)), bwd(nulls=(20,)), bwd(null_layer=True)):
        assert rc == -1
    assert fwd(B=0) == 0 and bwd(B=0) == 0
    torch.cuda.synchronize()
    assert all((t == -7).all() for t in outs) and (sink == -7).all()


# ---- models ------------------------------------------------------------------------------------------------------------------

def _run(key, **train):
    m, tr, dh = make_run(key, device='cuda', train=dict(deterministic=True, **train))
    return m, tr


@pytest.mark.parametrize('key', BPR_MODELS)
def test_key_false_is_the_key_absent_bit_for_bit(key):
    from sslrec_b200.optim import FusedAdam
    runs = []
    for train in (dict(deterministic=True), dict(deterministic=True, mixgcf=False)):
        m, _, _ = make_run(key, device='cuda', train=train)
        opt = FusedAdam(m.parameters(), lr=1e-2)
        runs.append(([_step(m, opt, b) for b in _batches(key, n=2)], m._seeds.count, m.mixgcf_picks))
    (plain, n_plain, _), (off, n_off, picks) = runs
    assert n_plain == n_off and picks is None
    for k, (a, b) in enumerate(zip(plain, off)):
        _assert_equal(a, b, (key, k))


@pytest.mark.parametrize('key', BPR_MODELS)
def test_alpha_zero_and_one_candidate_is_the_plain_step(key):
    """alpha = 0, M = 1: the mixed negative is the loader's negative summed over the layers, so the step is the plain step up
    to the order of the fp32 layer sum and of the gradient adds."""
    from sslrec_b200.optim import FusedAdam
    mix, _ = _run(key, mixgcf=True)
    plain, _ = _run(key)
    plain.load_state_dict(mix.state_dict())
    om, op = FusedAdam(mix.parameters(), lr=1e-2), FusedAdam(plain.parameters(), lr=1e-2)
    L1 = mix.layer_num + 1
    for k, batch in enumerate(_batches(key, n=2)):
        plain._seeds.load_state_dict(mix._seeds.state_dict())
        mix._mix_alpha_in = torch.zeros(batch[0].numel(), L1, device='cuda')
        a = _step(mix, om, batch)
        b = _step(plain, op, batch)
        assert torch.equal(mix.mixgcf_picks, batch[2][:, None].expand(-1, L1)) and (mix.mixgcf_alpha == 0).all()
        assert mix._seeds.count == plain._seeds.count + 1            # the mixing seed, drawn last
        for t in a[0]:
            assert abs(float(a[0][t]) - float(b[0][t])) <= 1e-5 * max(1.0, abs(float(b[0][t]))), (key, k, t)
        for n in b[1]:
            H.close(a[1][n], b[1][n], 1e-3, 1e-5 * b[1][n].abs().max().item() + 1e-12, f'{key} step {k} grad {n}')
        mix.load_state_dict(plain.state_dict())                      # the next step starts from the same parameters again


def _train(key, graphed, n=6):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    m, _ = _run(key, mixgcf=True, dns_candidates=8)
    opt = FusedAdam(m.parameters(), lr=1e-2)
    batches = _batches(key, n=n)
    ncl = key == 'ncl'
    out = []
    if graphed:
        torch.manual_seed(0)
        step = GraphedStep(m, opt, batches[0], warmup=2, recluster=ncl)
        for k, b in enumerate(batches[1:], start=1):
            loss, parts = step(b, recluster=ncl and k == 3)
            out.append((loss.clone(), m.mixgcf_picks.clone(), m.mixgcf_alpha.clone()))
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
                out.append((loss.detach().clone(), m.mixgcf_picks.clone(), m.mixgcf_alpha.clone()))
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


def whole_step_rows(ssm: bool):
    """(model_key, case name, hyper-parameter overrides, dim, M, sampled-softmax tau or None, deterministic) of the whole-step
    tests: the goldens' ``small`` rows, then every case of ``ssl_test_helpers.bpr_term_cases`` on the default route and, at
    d = 64, M = 8 and the default tau, on the train.deterministic route too."""
    tau = H.BPR_TERM_TAU if ssm else None
    rows = [pytest.param(m, 'small', {}, 64, 8, tau, False, id=f'{m}-small') for m in ('lightgcn', 'simgcl', 'sgl')]
    for c in H.bpr_term_cases(ssm):
        m, hp, d, M, t = c
        for det in (False, True) if (d, M, t) == (64, 8, tau) else (False,):
            rows.append(pytest.param(m, 'paths', hp, d, M, t, det, id=H.bpr_term_case_id(c) + ('-det' if det else '')))
    return rows


def whole_step(monkeypatch, model_key, case_name, hp_over, dim, M, deterministic, train, term_fn, cands_at, seen=None):
    """One cal_loss + backward of the model on a golden case or a ``bpr_term_setup`` case, with the draws, NCL's k-means and
    LightGCL's SVD factors injected (tests/test_gpu_model_paths._gpu_model) and the train keys ``train``; the candidates are
    captured from ``engine.<term_fn>`` (argument ``cands_at``).  -> (dict(loss, parts, grads) of float64 numpy, the
    candidates, the model, (case, hp, adj, draws, state)).  ``seen``: a dict that also receives the term's ``bias`` keyword
    (None when it is not passed), as the step passed it."""
    import sslrec_b200.config as cfgmod
    from sslrec_b200 import engine as E
    from test_gpu_model_paths import _batch, _gpu_model
    if case_name == 'paths':
        case, hp, adj, dr, st = H.bpr_term_setup(model_key, hp_over, dim)
    else:
        hp, case = replay.load_golden(model_key, case_name)['hp'], inputs.make_case(case_name)
        adj = O.normalized_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
        dr = replay.draws(model_key, case, hp, adj)
        st = H.path_state(model_key, case, hp, adj, dr)
    margin = H.kink_margin(model_key, case, hp, adj, dr, st)
    assert margin > H.KINK_MARGIN, f'ill-posed case: a kink input within {margin:.2e} of its |term| sum'
    default = cfgmod.default_config

    def with_train(name, **kw):
        cfg = default(name, **kw)
        cfg['train'].update(train, dns_candidates=M, deterministic=deterministic)
        return cfg

    monkeypatch.setattr(cfgmod, 'default_config', with_train)
    model = _gpu_model(model_key, case, hp, adj, dr, st)
    assert E.deterministic() == deterministic and model.dns_candidates == M
    seen = {} if seen is None else seen
    fn = getattr(E, term_fn)

    def keep(*args, **kwargs):
        seen['cands'] = args[cands_at].clone()
        seen['bias'] = None if kwargs.get('bias') is None else kwargs['bias'].clone()
        return fn(*args, **kwargs)

    monkeypatch.setattr(E, term_fn, keep)
    model.zero_grad()
    loss, parts = model.cal_loss(_batch(model_key, case['ancs'], case['poss'], case['negs']))
    loss.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    got = dict(loss=loss.item(), parts={k: float(v) for k, v in parts.items()},
               grads={k: p.grad.double().cpu().numpy() for k, p in model.named_parameters()})
    assert seen['cands'].shape == (len(case['ancs']), M)
    return got, seen['cands'].cpu(), model, (case, hp, adj, dr, st)


POP_BETA = 0.75


def _mixgcf_rows():
    """``whole_step_rows(ssm=False)`` with train.neg_popularity absent, then every BPR model at d = 64, M = 8 on both routes
    with popularity candidates (beta 0.75)."""
    rows = [pytest.param(*p.values, None, id=p.id) for p in whole_step_rows(ssm=False)]
    for m, hp in H.BPR_TERM_MODELS:
        for det in (False, True):
            rows.append(pytest.param(m, 'paths', hp, 64, 8, None, det, POP_BETA,
                                     id=H.bpr_term_case_id((m, hp, 64, 8, None)) + ('-det' if det else '') + f'-pop{POP_BETA}'))
    return rows


@pytest.mark.parametrize('model_key,case_name,hp_over,dim,M,tau,deterministic,beta', _mixgcf_rows())
def test_whole_step_against_float64(monkeypatch, model_key, case_name, hp_over, dim, M, tau, deterministic, beta):
    """The step equals the float64 oracle with its BPR term replaced by mixgcf_oracle.term on the model's own alpha and picks
    (ssl_test_helpers.bpr_term_oracle): loss, every term and every parameter's gradient within the path_errors bounds; the
    picks are float64's wherever the score gap is decided (the layer rows the kernel mixed, independently of the backward).
    With train.neg_popularity (``beta``) the candidates are also the popularity draw of tests/pop_oracle for the step's own
    seed, pairs and training matrix, bit for bit."""
    train = dict(mixgcf=True) if beta is None else dict(mixgcf=True, neg_popularity=beta)
    got, cands, model, (case, hp, adj, dr, st) = whole_step(monkeypatch, model_key, case_name, hp_over, dim, M, deterministic,
                                                            train, 'mixgcf_bpr_sum', 5)
    if beta is not None:
        want, _ = H.pop_draw(case, case['ancs'], case['negs'], M, beta, H.assert_step_seed(model))
        assert np.array_equal(cands.numpy(), want)
    picks, alpha = model.mixgcf_picks.cpu(), model.mixgcf_alpha.cpu()
    ancs, poss = torch.from_numpy(case['ancs']), torch.from_numpy(case['poss'])
    ref = H.bpr_term_oracle(model_key, case, hp, adj, dr, st, torch.float64,
                            lambda u, i, ls: X.term(u, i, ls, ancs, poss, picks, alpha), 'bpr_loss')
    errs = H.path_errors(got, ref)
    worst = max(errs, key=errs.get)
    print(f'mixgcf {model_key}-{case_name}-{hp_over}-d{dim}-M{M}{"-det" if deterministic else ""}'
          f'{"" if beta is None else f"-pop{beta}"}: largest error {errs[worst]:.3f} of '
          f'its bound ({worst})')
    with torch.no_grad():
        ue, _, layers = H.bpr_tables(model_key, case, hp, adj, dr, H.path_params(model_key, case, dr, torch.float64))
    decided = H.mixgcf_pick_check(ue, layers, ancs, poss, cands, alpha, picks)
    print(f'  picks decided {decided:.4f}')
    assert decided > 0.9, decided
    assert errs[worst] <= 1.0, errs


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('key,hp', [('simgcl', {}), ('ncl', {'epoch_period': 2})])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph):
    import test_gpu_resume as R
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, dns_candidates=8, mixgcf=True)
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
