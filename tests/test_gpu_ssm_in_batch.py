"""In-batch negatives for the sampled softmax (optional key train.ssm_in_batch) on the GPU.

The term, through ``engine.ssm_in_batch_sum``: loss and the gradients into the user rows, the positive rows and every one of the
2B columns against the float64 term of tests/inb_oracle.py, on each contraction kernel (FFMA at d = 20, 48 and 128, 3xTF32,
3xFP16), at tau on both sides of 0.0902, B from 1 to 8192 (2B at and past a 64-column tile, B at and past a 128-row tile),
duplicated ids among the columns, every column one item, zero weights, weights spanning four decades or scaled by 2^+-30, and
cosines near -1 as well as near 1; the kernel the forward took is the one ``contraction_kind`` names for the weights' range.  The
FP32-FMA route (USE_TENSOR_CORES False) agrees with the tensor-core one.  Under train.deterministic the gradients are the staged
per-position contributions added in position order, bit for bit, and two runs are bit-identical.  ssl_nce_bwd_cols rejects bad
arguments and writes nothing.  A temperature whose terms would fall below the flush of ex2.approx.ftz is refused; at the
smallest accepted one a batch with every cosine <= -0.8 is within the float64 bounds.

Models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL): the key false is the key absent bit for bit; the step draws exactly the
seeds of the plain step; under train.deterministic two runs and a CUDA-graph replay are bit-identical.  The whole step of every
BPR model equals the float64 oracle with its BPR term replaced by the in-batch term, on both gradient routes and each
contraction kernel (ssl_test_helpers.in_batch_step_cases).  SimGCL and NCL resumed from a mid-run checkpoint end bit-identical
to an uninterrupted run."""
import numpy as np
import pytest
import torch

import inb_oracle as IB
import ssl_test_helpers as H
from test_gpu_hard_negatives import _assert_equal, _batches, _step
from test_host_resume import make_run

pytestmark = pytest.mark.gpu

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def _case(B, d, n_user=300, n_item=500, seed=0, wrange=1e4, anti=False):
    """Tables, a duplicate-heavy batch and weights log-uniform over [1, wrange].  ``anti``: every item row is a user's row
    scaled by -1 or (every third item) +1, plus a little noise, so cosines reach both -1 and 1."""
    g = torch.Generator().manual_seed(seed)
    users = torch.randn(n_user, d, generator=g)
    items = torch.randn(n_item, d, generator=g)
    if anti:
        src = torch.randint(0, n_user, (n_item,), generator=g)
        items = -users[src] * (0.5 + torch.rand(n_item, 1, generator=g)) + 1e-3 * torch.randn(n_item, d, generator=g)
        items[::3] = -items[::3]
    ancs, poss, negs = (torch.randint(0, n, (B,), generator=g) for n in (n_user, n_item, n_item))
    ancs[::2] %= 3
    poss[::2] %= 5
    negs[::3] %= 7
    negs[::4] = poss[::4]                        # a pair's negative equal to its positive
    if anti:                                     # pair 1's positive opposes its user, its negative is aligned with it
        items[poss[1]] = -0.7 * users[ancs[1]]
        items[negs[1]] = 1.3 * users[ancs[1]]
    v = torch.exp(torch.rand(n_item, generator=g, dtype=torch.float64) * np.log(wrange)).numpy()
    return users, items, ancs, poss, negs, v


def _run(monkeypatch, users, items, ancs, poss, negs, v, tau, scale=1.0):
    from sslrec_b200 import engine as E
    kinds = []
    kind = E.contraction_kind

    def spy(*a, **k):
        kinds.append(kind(*a, **k))
        return kinds[-1]

    monkeypatch.setattr(E, 'contraction_kind', spy)
    w = E.InBatchWeights(v, 'cuda')
    leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
    loss = E.ssm_in_batch_sum(leaves[0], leaves[1], ancs.cuda(), poss.cuda(), negs.cuda(), tau, w)
    (loss * scale).backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    return loss.item(), [t.grad for t in leaves], kinds[0], w


KERNEL_CASES = [  # (B, d, tau, weight range, anti-aligned rows, tensor cores, the kernel the forward must take)
    (333, 48, 0.1, 1e4, False, True, 'ffma'),
    (1000, 64, 0.1, 1e4, False, True, 'tf32x3'),          # offset 14.4: past the weighted 3xFP16 bound
    (257, 32, 0.05, 1e4, True, True, 'tf32x3'),           # tau < 0.0902: past the 3xFP16 offset bound
    (4096, 64, 0.09, 1e4, False, True, 'tf32x3'),
    (700, 64, 0.095, 1.0, True, True, 'tf32x3'),           # tau > 0.0902 but the weighted bound: 15.2 + 0.5 > 13.5
    (1000, 64, 0.5, 1e4, True, True, 'f16x3'),            # 2.9 + (1 + 13.3) / 2 = 10.0 <= 13.5
    (129, 32, 0.25, 1e2, False, True, 'f16x3'),
    (4096, 64, 0.2, 10.0, True, True, 'f16x3'),            # 7.2 + 2.2
    (1000, 64, 0.1, 1e4, True, False, 'ffma'),
    (512, 128, 0.1, 1e4, True, True, 'ffma'),             # the lane layouts of ssl_nce_bwd_cols: 4 floats per lane, and
    (300, 20, 0.1, 1e4, False, True, 'ffma'),             # 20 of 32 lanes idle
    (8192, 64, 0.1, 1e4, False, True, 'tf32x3'),          # 16384 columns
    (8192, 64, 0.5, 1e4, True, True, 'f16x3'),
]
# one or two pairs; 2B at and past a 64-column tile (B = 32, 33); B at and past a 128-row tile (128, 129)
KERNEL_CASES += [(B, 64, tau, 1e4, B in (33, 129), True, kind) for B in (1, 2, 32, 33, 128, 129)
                 for tau, kind in ((0.1, 'tf32x3'), (0.5, 'f16x3'))]


def _against_float64(loss, grads, users, items, ancs, poss, negs, tau, v32, v_loss=None):
    """The bounds of ``test_term_against_float64`` against inb_oracle.term64 on the fp32 weights ``v32`` (float64 [n_item]);
    ``v_loss``: another table whose float64 loss the loss must meet instead (the gradients keep the bound of ``v32``)."""
    B = ancs.numel()
    ref_leaves = [t.double().cuda().requires_grad_(True) for t in (users, items)]
    ref = IB.term64(ref_leaves[0], ref_leaves[1], ancs, poss, negs, tau, v32)
    ref.backward()
    if v_loss is not None:
        with torch.no_grad():
            ref = IB.term64(users.double().cuda(), items.double().cuda(), ancs, poss, negs, tau, v_loss)
    assert abs(loss - ref.item()) <= 1e-5 * max(1.0, abs(ref.item())) + 4e-7 * B / tau, (loss, ref.item())
    A = IB.abs_scale(users.cuda(), items.cuda(), ancs, poss, negs, tau, v32)
    for got, want, a, what in zip(grads, ref_leaves, A, ('users', 'items')):
        H.close(got, want.grad, 2e-4, 5e-4 * a.cpu().numpy() + 1e-12, what)


@pytest.mark.parametrize('B,d,tau,wrange,anti,tc,kind', KERNEL_CASES)
def test_term_against_float64(monkeypatch, B, d, tau, wrange, anti, tc, kind):
    """Loss within 1e-5 max(1, |ref|) + 4e-7 B / tau (a scale-1/tau score carries ~d/2 ulp of a unit cosine); every gradient
    element within 5e-4 A + 2e-4 |ref|, A the float64 sum of the magnitudes of the terms that add into it (inb_oracle.abs_scale:
    float atomics add up to 2B + 2 terms per row in any order, and each term carries the error of its score)."""
    from sslrec_b200 import engine as E
    monkeypatch.setattr(E, 'USE_TENSOR_CORES', tc)
    users, items, ancs, poss, negs, v = _case(B, d, seed=B + d, wrange=wrange, anti=anti)
    loss, grads, took, w = _run(monkeypatch, users, items, ancs, poss, negs, v, tau)
    assert took == kind, (took, kind, w.range)
    assert w.range == pytest.approx(float(v.max() / v.min()), rel=1e-6)
    _against_float64(loss, grads, users, items, ancs, poss, negs, tau, w.v.double().cpu().numpy())
    if anti:                                      # the rows do reach both ends of the cosine range
        u = torch.nn.functional.normalize(users[ancs].double(), dim=1)
        c = torch.nn.functional.normalize(items[torch.cat([poss, negs])].double(), dim=1)
        cos = u @ c.T
        assert cos.min() < -0.99 and cos.max() > 0.99


def test_fp32_fma_route_agrees_with_the_tensor_cores(monkeypatch):
    from sslrec_b200 import engine as E
    users, items, ancs, poss, negs, v = _case(1500, 64, seed=9, anti=True)
    out = {}
    for tc in (True, False):
        monkeypatch.setattr(E, 'USE_TENSOR_CORES', tc)
        out[tc] = _run(monkeypatch, users, items, ancs, poss, negs, v, 0.1)
    (l1, g1, k1, _), (l0, g0, k0, _) = out[True], out[False]
    assert (k1, k0) == ('tf32x3', 'ffma')
    assert abs(l1 - l0) <= 1e-5 * abs(l0) + 4e-7 * 1500 / 0.1
    A = IB.abs_scale(users.cuda(), items.cuda(), ancs, poss, negs, 0.1, out[True][3].v.double().cpu().numpy())
    for a, b, s in zip(g1, g0, A):
        H.close(a, b, 2e-4, 1e-3 * s.cpu().numpy() + 1e-12, 'tc vs ffma')


def test_deterministic_route_is_its_ordered_restatement(monkeypatch):
    """Under train.deterministic the sinks receive the staged per-position contributions (users: ancs; items: the positives' row
    term at poss, then the 2B columns) added in position order: restated here with one torch add per position from the stages
    the route scattered.  A second run is bit-identical, and both are within the float64 bound."""
    _ordered_restatement(monkeypatch, 300, 64)


@pytest.mark.parametrize('B,d', [(1, 64), (200, 128)])
def test_deterministic_route_is_its_ordered_restatement_at_one_pair_and_d128(monkeypatch, B, d):
    """``test_deterministic_route_is_its_ordered_restatement`` at one pair (two columns) and at the widest row (FFMA)."""
    _ordered_restatement(monkeypatch, B, d)


def _ordered_restatement(monkeypatch, B, d):
    from sslrec_b200 import engine as E
    monkeypatch.setattr(E, 'DETERMINISTIC', True)
    users, items, ancs, poss, negs, v = _case(B, d, seed=3)
    seen = []
    grouped = E._scatter_grouped

    def keep(parts):
        seen.append([(st.clone(), ids.clone()) for st, ids, _, _ in parts])
        return grouped(parts)

    monkeypatch.setattr(E, '_scatter_grouped', keep)
    w = E.InBatchWeights(v, 'cuda')
    runs = []
    for _ in range(2):
        leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
        (E.ssm_in_batch_sum(leaves[0], leaves[1], ancs.cuda(), poss.cuda(), negs.cuda(), 0.1, w) * 0.5).backward()
        runs.append([t.grad.clone() for t in leaves])
    monkeypatch.undo()
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    (su, iu), (si, ii) = seen[0]
    assert torch.equal(iu.cpu(), ancs) and torch.equal(ii.cpu(), torch.cat([poss, poss, negs]))

    def ordered(n_rows, stage, rows):
        sink = torch.zeros(n_rows, stage.shape[1], device='cuda')
        for p, r in enumerate(rows.tolist()):
            sink[r] = sink[r] + stage[p]
        return sink

    assert torch.equal(runs[0][0], ordered(users.shape[0], su, iu))
    assert torch.equal(runs[0][1], ordered(items.shape[0], si, ii))
    loss, grads, _, _ = _run(monkeypatch, users, items, ancs, poss, negs, v, 0.1, scale=0.5)
    A = IB.abs_scale(users.cuda(), items.cuda(), ancs, poss, negs, 0.1, w.v.double().cpu().numpy())
    for a, b, s in zip(runs[0], grads, A):
        H.close(a, b, 2e-4, 1e-3 * s.cpu().numpy() + 1e-12, 'ordered vs atomic')


def test_bad_arguments_are_rejected_and_write_nothing():
    from sslrec_b200._lib import lib
    f = dict(device='cuda', dtype=torch.float32)
    n, d = 8, 32
    part, t, r, w = torch.ones(2, n, d, **f), torch.ones(n, d, **f), torch.ones(n, **f), torch.ones(n, **f)
    ids = torch.zeros(n, dtype=torch.int64, device='cuda')
    sink = torch.full((n, d), -7.0, **f)
    s = torch.cuda.current_stream().cuda_stream
    p = lambda x: x.data_ptr()

    def call(n_split=2, nn=n, dim=d, stride=d, nulls=()):
        a = [p(part), n_split, p(t), p(r), p(w), p(ids), nn, dim, p(sink), stride, s]
        for i in nulls:
            a[i] = None
        return lib.ssl_nce_bwd_cols(*a)

    for rc in (call(n_split=0), call(nn=-1), call(dim=0), call(dim=129), call(stride=31), call(nulls=(0,)), call(nulls=(2,)),
               call(nulls=(3,)), call(nulls=(4,)), call(nulls=(8,))):
        assert rc == -1
    assert call(nn=0) == 0
    torch.cuda.synchronize()
    assert (sink == -7).all()


@pytest.mark.parametrize('B,d,deterministic,kind', [(1000, 64, False, 'tf32x3'), (1000, 64, True, 'tf32x3'),
                                                    (513, 128, False, 'ffma'), (513, 128, True, 'ffma')])
def test_one_item_batch(monkeypatch, B, d, deterministic, kind):
    """Every pair has the same anchor, positive and negative: all 2B columns are one item, so every column's gradient adds
    into one row (the most contended atomic target), the 2B + B row terms into it under the ordered route."""
    from sslrec_b200 import engine as E
    monkeypatch.setattr(E, 'DETERMINISTIC', deterministic)
    users, items, _, _, _, v = _case(B, d, seed=11)
    ancs, poss, negs = torch.full((B,), 2), torch.full((B,), 7), torch.full((B,), 7)
    loss, grads, took, w = _run(monkeypatch, users, items, ancs, poss, negs, v, 0.1)
    assert took == kind
    _against_float64(loss, grads, users, items, ancs, poss, negs, 0.1, w.v.double().cpu().numpy())
    assert grads[1].abs().sum(1).nonzero().flatten().tolist() == [7] and grads[0].abs().sum(1).nonzero().flatten().tolist() == [2]


@pytest.mark.parametrize('tau,kind', [(0.1, 'tf32x3'), (0.5, 'f16x3')])
def test_zero_weights(monkeypatch, tau, kind):
    """Weights of 0 at some of the batch's ids, pair 0's own positive among them: those columns add nothing to any row sum and
    take no column gradient, while the pair's diagonal score still counts."""
    from sslrec_b200 import engine as E
    users, items, ancs, poss, negs, v = _case(400, 64, seed=12)
    zero = [int(poss[0]), int(poss[3]), int(negs[1]), int(negs[10])]
    v[zero] = 0.0
    loss, grads, took, w = _run(monkeypatch, users, items, ancs, poss, negs, v, tau)
    assert took == kind and w.vmin == float(np.float32(v[v > 0].min()))
    _against_float64(loss, grads, users, items, ancs, poss, negs, tau, w.v.double().cpu().numpy())


@pytest.mark.parametrize('tau,kind', [(0.1, 'tf32x3'), (0.5, 'f16x3')])
@pytest.mark.parametrize('exponent', [30, -30])
def test_absolute_weight_scale(monkeypatch, exponent, tau, kind):
    """v times 2^30 or 2^-30 (exact in fp32): each loss_b moves by ln of the scale, the gradients do not.  The loss meets the
    float64 loss of the scaled table, the gradients the bound of the unscaled one; the kernel is the unscaled table's."""
    users, items, ancs, poss, negs, v = _case(600, 64, seed=13)
    v32 = v.astype(np.float32).astype(np.float64)
    scaled = v32 * 2.0 ** exponent
    loss, grads, took, w = _run(monkeypatch, users, items, ancs, poss, negs, scaled, tau)
    assert took == kind and np.array_equal(w.v.double().cpu().numpy(), scaled)
    _against_float64(loss, grads, users, items, ancs, poss, negs, tau, v32, v_loss=scaled)


@pytest.mark.parametrize('which', ['anti', 'partial'])
def test_underflowing_temperature_is_refused(which):
    """At tau = 0.02 the batches of inb_oracle.underflow_batch lose every term of a row ('anti': loss -inf) or a share of each
    row sum far past fp32 grade ('partial') to the flush-to-zero ex2 (tests/test_host_ssm_in_batch.py restates it): the term
    refuses the temperature, naming the bound, and so does the float just below the smallest accepted one."""
    from sslrec_b200 import engine as E
    users, items, ancs, poss, negs, v = IB.underflow_batch(which)
    w = E.InBatchWeights(v, 'cuda')
    tau = IB.smallest_tau(ancs.numel(), w.vmin)
    for bad in (0.02, float(np.nextafter(tau, 0.0))):
        leaves = [t.cuda().requires_grad_(True) for t in (users, items)]
        with pytest.raises(ValueError, match=r'needs 2 log2\(e\) / tau \+ max\(0, log2\(B / min v\)\) <= 125'):
            E.ssm_in_batch_sum(leaves[0], leaves[1], ancs.cuda(), poss.cuda(), negs.cuda(), bad, w)


@pytest.mark.parametrize('tc,kind', [(False, 'ffma'), (True, 'tf32x3')])
@pytest.mark.parametrize('which', ['anti', 'partial'])
def test_smallest_accepted_temperature_is_within_float64(monkeypatch, which, tc, kind):
    """The same batches at the smallest tau the bound accepts (~0.0247 for B = 300, min v ~ 1): every term is a normal fp32
    number, and the loss and gradients meet the float64 bounds of ``test_term_against_float64``."""
    from sslrec_b200 import engine as E
    monkeypatch.setattr(E, 'USE_TENSOR_CORES', tc)
    users, items, ancs, poss, negs, v = IB.underflow_batch(which)
    tau = IB.smallest_tau(ancs.numel(), float(np.float32(v).min()))
    loss, grads, took, w = _run(monkeypatch, users, items, ancs, poss, negs, v, tau)
    assert took == kind and np.isfinite(loss)
    _against_float64(loss, grads, users, items, ancs, poss, negs, tau, w.v.double().cpu().numpy())


# ---- models ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('key', BPR_MODELS)
def test_key_false_is_the_key_absent_and_draws_the_plain_seeds(key):
    from sslrec_b200.optim import FusedAdam
    runs = []
    for train in (dict(deterministic=True, ssm_temperature=0.1), dict(deterministic=True, ssm_temperature=0.1, ssm_in_batch=False),
                  dict(deterministic=True, ssm_temperature=0.1, ssm_in_batch=True), dict(deterministic=True)):
        m, _, _ = make_run(key, device='cuda', train=train)
        opt = FusedAdam(m.parameters(), lr=1e-2)
        runs.append(([_step(m, opt, b) for b in _batches(key, n=2)], m._seeds.count, m))
    (ssm, n_ssm, _), (off, n_off, _), (inb, n_inb, m_inb), (_, n_plain, _) = runs
    for k, (a, b) in enumerate(zip(ssm, off)):
        _assert_equal(a, b, (key, k))
    assert n_ssm == n_off == n_inb == n_plain                 # no candidate draw, no seed
    assert m_inb.dns_negs is None and m_inb._in_batch is not None
    assert 'ssm_loss' in inb[0][0] and all(torch.isfinite(t).all() for t in inb[0][0].values())
    assert not torch.equal(inb[0][0]['ssm_loss'], ssm[0][0]['ssm_loss'])


def _train(key, graphed, n=6):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    m, _, _ = make_run(key, device='cuda', train=dict(deterministic=True, ssm_temperature=0.1, ssm_in_batch=True))
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
        m._graph_mode = key == 'hccf'
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


def _whole_step(monkeypatch, model_key, case_name, hp_over, dim, deterministic, tau, tc=True):
    """One cal_loss + backward with the draws, k-means state and SVD factors injected (test_gpu_model_paths._gpu_model) and
    train.ssm_in_batch; ``tau`` H.IN_BATCH_SMALLEST_TAU: the smallest the term accepts for the case's B and weights.  -> (dict(loss,
    parts, grads) of float64 numpy, the model, (case, hp, adj, draws, state), tau, the kernels the contraction took)."""
    import sslrec_b200.config as cfgmod
    from oracle import cf_oracle as O
    from oracle import inputs, replay
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
    if tau == H.IN_BATCH_SMALLEST_TAU:
        rowptr, cols = H.train_csr(case)
        tau = IB.smallest_tau(len(case['ancs']), E.InBatchWeights.of_matrix(rowptr, cols, case['n_item'], 'cpu').vmin)
    default = cfgmod.default_config

    def with_train(name, **kw):
        cfg = default(name, **kw)
        cfg['train'].update(ssm_temperature=tau, ssm_in_batch=True, deterministic=deterministic)
        return cfg

    kinds = []
    kind = E.contraction_kind

    def spy(*a, **k):                   # the weighted forward is the one caller that passes colscale_range
        out = kind(*a, **k)
        if k.get('colscale_range') is not None:
            kinds.append(out)
        return out

    monkeypatch.setattr(cfgmod, 'default_config', with_train)
    monkeypatch.setattr(E, 'USE_TENSOR_CORES', tc)
    monkeypatch.setattr(E, 'contraction_kind', spy)
    model = _gpu_model(model_key, case, hp, adj, dr, st)
    assert E.deterministic() == deterministic and model.ssm_in_batch
    model.zero_grad()
    loss, parts = model.cal_loss(_batch(model_key, case['ancs'], case['poss'], case['negs']))
    loss.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    got = dict(loss=loss.item(), parts={k: float(v) for k, v in parts.items()},
               grads={k: p.grad.double().cpu().numpy() for k, p in model.named_parameters()})
    return got, model, (case, hp, adj, dr, st), tau, kinds


WHOLE_STEP = [pytest.param(*c[1:], id=c[0]) for c in H.in_batch_step_cases()]
WORST = {}                              # (model, kernel) -> the largest error fraction of the whole-step rows run so far


@pytest.mark.parametrize('model_key,case_name,hp_over,dim,tau,deterministic,tc,kind', WHOLE_STEP)
def test_whole_step_against_float64(monkeypatch, model_key, case_name, hp_over, dim, tau, deterministic, tc, kind):
    """The step equals the float64 oracle with its BPR term replaced by inb_oracle.term64 on the loader's batch, with weights
    from the case's training matrix (ssl_test_helpers.bpr_term_oracle): loss, every term and every parameter's gradient
    (HCCF's hyper weights and LightGCL's Ws among them) within the path_errors bounds.  The weighted forward took ``kind``;
    the weight table is in_batch_weights of the case's training CSR, bit for bit."""
    from sslrec_b200 import engine as E
    got, model, (case, hp, adj, dr, st), tau, kinds = _whole_step(monkeypatch, model_key, case_name, hp_over, dim, deterministic,
                                                                  tau, tc)
    assert kinds == [kind], (kinds, kind)
    assert 'bpr_loss' not in got['parts'] and model.dns_negs is None
    rowptr, cols = H.train_csr(case)
    v = E.in_batch_weights(rowptr, cols, case['n_item']).astype(np.float32)
    assert np.array_equal(model._in_batch.v.cpu().numpy(), v)
    ancs, poss, negs = (torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs'))
    ref = H.bpr_term_oracle(model_key, case, hp, adj, dr, st, torch.float64,
                            lambda u, i, _: IB.term64(u, i, ancs, poss, negs, tau, v.astype(np.float64)), 'ssm_loss')
    errs = H.path_errors(got, ref)
    worst = max(errs, key=errs.get)
    WORST[model_key, kind] = max(WORST.get((model_key, kind), 0.0), errs[worst])
    print(f'in-batch {model_key}{hp_over}-{case_name}-d{dim}-tau{tau:.6g}{"-det" if deterministic else ""}-{kind}: largest '
          f'error {errs[worst]:.3f} of its bound ({worst}); worst so far per (model, kernel): '
          + ', '.join(f'{m}/{k} {e:.3f}' for (m, k), e in sorted(WORST.items())))
    assert errs[worst] <= 1.0, errs


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('key,hp', [('simgcl', {}), ('ncl', {'epoch_period': 2})])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph):
    import test_gpu_resume as R
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, ssm_temperature=0.1, ssm_in_batch=True)
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
