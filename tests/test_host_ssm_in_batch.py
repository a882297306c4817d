"""In-batch negatives for the sampled softmax (train.ssm_in_batch) without a GPU: the key's bad values, acceptance on the six BPR
models and every refusal (no temperature, drawn candidates, popularity draws, DirectAU, a row-sharded model, data-parallel
gradient sync), the checkpoint record; ``engine.in_batch_weights`` against a brute-force float64 restatement of p_i and r_i;
the loaders' sampling law itself (HostBatchLoader with ``sample_negs`` over many epochs: the column counts by a chi-square test,
the weighted column sum as an unbiased estimate of the catalogue sum within a CLT bound); and the column-backward kernel
(csrc/ssm_in_batch.cuh) under AddressSanitizer through tests/emu, bit for bit against its sequential float32 restatement.
The forward's flush-to-zero terms restated in numpy (tests/inb_oracle.py): at tau = 0.02 they lose whole rows or fp32 grade,
and ``engine.ssm_in_batch_sum`` refuses such a temperature.  On every whole-step case of tests/test_gpu_ssm_in_batch.py: the
float32 oracle meets the GPU test's bounds against float64, and six wrong terms do not."""
import os
import shutil
import subprocess
import types
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from scipy import stats

import inb_oracle as IB
import ssl_test_helpers as H
from sslrec_b200 import engine as E
from test_host_resume import make_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']
ON = dict(ssm_temperature=0.1, ssm_in_batch=True)


# ---- the key -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('value', [1, 0, 'true', None, 2.5, [True]])
def test_bad_values_are_refused_at_construction(value):
    with pytest.raises(ValueError, match='train.ssm_in_batch must be true or false'):
        make_run('lightgcn', train=dict(ssm_temperature=0.1, ssm_in_batch=value))


@pytest.mark.parametrize('model_key', BPR_MODELS)
def test_every_bpr_model_accepts_the_key_and_draws_nothing(model_key):
    m = make_run(model_key, train=ON)[0]
    assert m.neg.in_batch is True and m.ssm_in_batch is True and m.ssm_temperature == 0.1 and m.bpr_loss_name == 'ssm_loss'
    assert m._in_batch is None and m.dns_negs is None
    ancs, negs = torch.arange(6), torch.arange(6) % 3
    before = m._seeds.state_dict()
    assert m._dns_candidates(ancs, negs) is None                 # no candidates, no seed consumed
    assert m._seeds.state_dict() == before and m._mix_seed is None
    for train in ({}, dict(ssm_in_batch=False), dict(ssm_temperature=0.1, ssm_in_batch=False)):
        m = make_run(model_key, train=train)[0]
        assert m.neg.in_batch is False and m.ssm_in_batch is False, train


REFUSED = [  # (train section, message)
    (dict(ssm_in_batch=True), 'train.ssm_in_batch is a form of the sampled softmax: it needs train.ssm_temperature'),
    (dict(ssm_in_batch=True, ssm_temperature=None), 'it needs train.ssm_temperature'),
    (dict(ON, dns_candidates=2), 'train.dns_candidates would be drawn and never read: it must be 1, got 2'),
    (dict(ON, dns_candidates=256), 'must be 1, got 256'),
    (dict(ON, dns_candidates=8, neg_popularity=0.5), 'must be 1, got 8'),
    (dict(ON, neg_popularity=0.5), 'train.neg_popularity draws the candidates of train.dns_candidates'),
    (dict(ON, mixgcf=True), 'train.ssm_temperature and train.mixgcf both replace the BPR term'),
]


@pytest.mark.parametrize('train,match', REFUSED)
def test_combinations_are_refused(train, match):
    with pytest.raises(ValueError, match=match):
        make_run('simgcl', train=train)


def test_directau_is_refused():
    for train in (dict(ssm_in_batch=True), ON):
        key = 'ssm_temperature' if 'ssm_temperature' in train else 'ssm_in_batch'      # the first key the config sets
        with pytest.raises(ValueError, match=f'train.{key}: DirectAU trains without negatives'):
            make_run('directau', train=train)


def test_multi_gpu_is_refused():
    from sslrec_b200.trainer import Trainer
    m, _, dh = make_run('simgcl', train=ON)
    with pytest.raises(ValueError, match="train.ssm_in_batch is single-GPU: a row-sharded model does not contract the batch's items"):
        m.shard_to(types.SimpleNamespace(shard_propagation=False))
    assert m.comm is None
    with pytest.raises(ValueError, match='train.ssm_in_batch is single-GPU: each rank would contract only its share of the batch'):
        Trainer(dh, grad_sync=object())
    _, _, dh = make_run('simgcl', train=dict(ssm_temperature=0.1, ssm_in_batch=False))
    with pytest.raises(ValueError, match='train.ssm_temperature is single-GPU'):        # the key off: the message of today
        Trainer(dh, grad_sync=object())


def test_checkpoints_record_the_key_only_when_it_is_set(tmp_path):
    saved, plain = str(tmp_path / 'inb.pth'), str(tmp_path / 'plain.pth')
    m, tr, _ = make_run('ncl', train=ON)
    rec = tr._resume_record(m, 'host')
    assert rec['ssm_in_batch'] is True and rec['ssm_temperature'] == 0.1
    tr.save_checkpoint(m, saved)
    m, tr, _ = make_run('ncl', train=dict(ssm_temperature=0.1, ssm_in_batch=False))
    rec = tr._resume_record(m, 'host')
    assert 'ssm_in_batch' not in rec and rec == make_run('ncl', train=dict(ssm_temperature=0.1))[1]._resume_record(m, 'host')
    tr.save_checkpoint(m, plain)
    with pytest.raises(ValueError, match='ssm_in_batch: saved True, now None'):
        tr.load_checkpoint(m, saved)
    m, tr, _ = make_run('ncl', train=ON)
    with pytest.raises(ValueError, match='ssm_in_batch: saved None, now True'):
        tr.load_checkpoint(m, plain)
    assert tr.load_checkpoint(m, saved) == 0
    assert m._in_batch is None                    # the weights are not part of a checkpoint


# ---- the weights -------------------------------------------------------------------------------------------------------------

def _csr(n_user, n_item, pairs):
    m = sp.csr_matrix((np.ones(len(pairs)), ([u for u, _ in pairs], [i for _, i in pairs])), shape=(n_user, n_item))
    m.sum_duplicates()
    m.sort_indices()
    return m


def _weights_exact(m):
    """v_i from the definition, in exact rationals: p_i + r_i summed user by user over the items."""
    n_user, n_item = m.shape
    E_ = m.nnz
    q = [Fraction(0)] * n_item
    for u in range(n_user):
        row = set(m.indices[m.indptr[u]:m.indptr[u + 1]].tolist())
        for i in row:
            q[i] += Fraction(1, E_)
        if row and len(row) < n_item:
            for i in range(n_item):
                if i not in row:
                    q[i] += Fraction(len(row), E_) / (n_item - len(row))
    return np.array([0.0 if x == 0 else float(1 / x) for x in q]), q


def _graphs():
    rng = np.random.default_rng(5)
    out = []
    for n_user, n_item, n_edge in ((7, 9, 20), (12, 30, 80), (40, 25, 300)):
        out.append(('random-%d' % n_item, _csr(n_user, n_item, list(zip(rng.integers(0, n_user, n_edge), rng.integers(0, n_item, n_edge))))))
    # items 0 .. 3 of degree 0, user 0 holding n_item - 1 items, user 1 holding none
    n_item = 12
    pairs = [(0, i) for i in range(1, n_item)] + [(u, int(i)) for u in range(2, 9) for i in rng.integers(4, n_item, 3)]
    out.append(('cold-items-full-user', _csr(9, n_item, pairs)))
    out.append(('one-item', _csr(5, 1, [(0, 0), (2, 0), (4, 0)])))            # every user with an edge holds every item: r = 0
    out.append(('one-user-all', _csr(3, 4, [(0, i) for i in range(4)] + [(1, 2)])))
    # Zipf-skewed popularity: the weights span several orders of magnitude
    n_item = 300
    z = 1.0 / np.arange(1, n_item + 1) ** 1.2
    items = rng.choice(n_item, 3000, p=z / z.sum())
    out.append(('zipf', _csr(200, n_item, list(zip(rng.integers(0, 200, 3000), items)))))
    return out


@pytest.mark.parametrize('name,m', _graphs(), ids=[g[0] for g in _graphs()])
def test_weights_match_their_definition(name, m):
    want, q = _weights_exact(m)
    got = E.in_batch_weights(m.indptr, m.indices, m.shape[1])
    assert got.dtype == np.float64 and got.shape == (m.shape[1],)
    assert np.array_equal(got == 0, want == 0), name                 # exactly the items no column can hold
    live = want > 0
    assert np.allclose(got[live], want[live], rtol=1e-13, atol=0), (name, np.max(np.abs(got[live] / want[live] - 1)))
    # sum_i (p_i + r_i): 1 for the positive slot plus the share of the edges whose user has a non-positive (a user who holds
    # every item cannot be served a negative; the weights give it none)
    n_item = m.shape[1]
    deg = np.diff(m.indptr)
    assert sum(q) == 1 + Fraction(int(deg[deg < n_item].sum()), m.nnz), name
    w = E.InBatchWeights(got, 'cpu')
    assert w.v.dtype == torch.float32 and np.array_equal(w.v.numpy(), got.astype(np.float32))
    assert w.range == pytest.approx(float(got[live].max() / got[live].min()) if live.any() else 1.0, rel=1e-6)
    if name == 'zipf':
        assert w.range > 10.0


def test_weights_refuse_bad_tables():
    for bad in (np.zeros(4), np.array([1.0, -1.0]), np.array([1.0, np.inf]), np.ones((2, 2))):
        with pytest.raises(ValueError):
            E.InBatchWeights(bad, 'cpu')


# ---- the sampling law of the loaders -----------------------------------------------------------------------------------------

def test_the_loaders_columns_follow_the_law_the_weights_assume():
    """HostBatchLoader over PairwiseTrnData with ``sample_negs`` re-drawn every epoch, on a 6 x 8 graph with 19 edges in batches of
    5 (a last batch of 4): per item, the column count over all batches against sum_k B_k (p_i + r_i) by a chi-square test, and the
    per-batch Hansen-Hurwitz estimate sum_c v[id_c] / B f(id_c) whose mean must reach sum_i f(i) within 5 standard errors."""
    from sslrec_b200.data_handler import HostBatchLoader, PairwiseTrnData
    rng = np.random.default_rng(3)
    n_user, n_item = 6, 8
    pairs = [(0, 0), (0, 1), (0, 2), (0, 3), (0, 4), (0, 5), (0, 6), (1, 0), (1, 1), (2, 0), (2, 2), (2, 5), (3, 1),
             (4, 0), (4, 3), (4, 6), (5, 0), (5, 4), (5, 2)]          # 19 edges; item 7 is cold, user 0 has one non-positive
    m = _csr(n_user, n_item, pairs)
    ds = PairwiseTrnData(m.tocoo())
    loader = HostBatchLoader(ds, 5)
    v = E.in_batch_weights(m.indptr, m.indices, n_item)
    q = np.array([float(x) for x in _weights_exact(m)[1]])
    f = rng.standard_normal(n_item) + 2.0
    target = f.sum()
    np.random.seed(11)
    torch.manual_seed(11)
    counts, expect, alt, est = np.zeros(n_item), np.zeros(n_item), np.zeros(n_item), []
    p_pos = np.bincount(m.indices, minlength=n_item) / m.nnz
    for _ in range(3000):
        ds.sample_negs()
        for ancs, poss, negs in loader:
            ids = np.concatenate([poss.numpy(), negs.numpy()]).astype(np.int64)
            B = len(poss)
            counts += np.bincount(ids, minlength=n_item)
            expect += B * q
            alt += B * (p_pos + 1.0 / n_item)     # a wrong law: negatives uniform over every item
            est.append(float(np.sum(v[ids] / B * f[ids])))
    assert np.all(q > 0) and counts.sum() == pytest.approx(expect.sum(), rel=1e-12)
    chi2 = float(np.sum((counts - expect) ** 2 / expect))
    assert stats.chi2.sf(chi2, n_item - 1) > 1e-3, chi2
    chi2_alt = float(np.sum((counts - alt) ** 2 / alt))          # the test has the power to tell the two apart
    assert stats.chi2.sf(chi2_alt, n_item - 1) < 1e-12, chi2_alt
    n_batches = len(est)
    est = np.array(est)
    se = est.std(ddof=1) / np.sqrt(n_batches)
    assert abs(est.mean() - target) <= 5 * se, (est.mean(), target, se)
    assert se < 0.01 * abs(target)                # and the bound is tight enough to mean something


# ---- the column-backward kernel on the host ----------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'ssm_in_batch_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'ssm_in_batch_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


# (n columns, n_split, dim, stride extra, mode: 0 stage / 1 permuted ids onto a prior sink / 2 repeated ids)
EMU_CASES = [(1, 1, 4, 0, 0), (7, 3, 12, 4, 0), (9, 1, 32, 0, 1), (33, 4, 64, 0, 0), (70, 5, 128, 8, 1), (130, 64, 48, 4, 0),
             (257, 2, 64, 0, 1), (40, 3, 36, 0, 2), (300, 7, 64, 0, 2), (16, 9, 128, 0, 2)]


@pytest.mark.parametrize('case', EMU_CASES, ids=lambda c: 'n%d-split%d-d%d-x%d-mode%d' % c)
def test_column_backward_matches_its_sequential_restatement_on_the_host(emulator, case):
    r = subprocess.run([emulator] + [str(v) for v in case] + [str(sum(case) + 1)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert 'bad=0' in r.stdout


# ---- the forward's flush-to-zero terms and the temperature bound -------------------------------------------------------------

@pytest.mark.parametrize('which', ['anti', 'partial'])
def test_flushed_terms_underflow_at_small_tau_and_the_bound_refuses_it(which):
    """At tau = 0.02 the kernels' terms fp32(ex2.approx.ftz(S - offset)) w_c (inb_oracle.rowsum32) lose the batches of
    inb_oracle.underflow_batch: every row sum of 'anti' is 0 (loss -inf), and each row sum of 'partial' misses far more than
    fp32 grade.  ``engine.ssm_in_batch_sum`` refuses both before touching a device, with a message naming the bound, and so
    does the next float below the smallest accepted tau; at that tau the same restatement is fp32 grade."""
    users, items, ancs, poss, negs, v = IB.underflow_batch(which)
    B = len(ancs)
    cos = IB.cosines(users, items, ancs, poss, negs)
    w = v.astype(np.float32)[np.concatenate([poss, negs])] / np.float32(B)
    weights = E.InBatchWeights(v, 'cpu')
    r32, r64 = IB.rowsum32(cos, w, 0.02), IB.rowsum64(cos, w, 0.02)
    rel = np.abs(r32 / r64 - 1)
    s_bb = cos[np.arange(B), np.arange(B)] / 0.02
    with np.errstate(divide='ignore'):
        loss = float(np.sum(np.log(r32) + 1 / 0.02 - s_bb))
    print(f'{which} at tau 0.02: loss {loss}, row sums flushed to 0: {int((r32 == 0).sum())} of {B}, '
          f'largest relative row-sum error {rel.max():.3g}')
    if which == 'anti':
        assert cos.max() <= -0.8 and (r32 == 0).all() and loss == -np.inf
    else:
        assert (r32 > 0).all() and rel.min() >= 1e-4
    bound = r'needs 2 log2\(e\) / tau \+ max\(0, log2\(B / min v\)\) <= 125'
    tau = IB.smallest_tau(B, weights.vmin)
    for bad in (0.02, float(np.nextafter(tau, 0.0))):
        with pytest.raises(ValueError, match=bound):
            E.ssm_in_batch_sum(users, items, ancs, poss, negs, bad, weights)
    assert 0.024 < tau < 0.025 and E.in_batch_binades(B, tau, weights.vmin) <= E.IN_BATCH_MAX_BINADES
    rel = np.abs(IB.rowsum32(cos, w, tau) / IB.rowsum64(cos, w, tau) - 1)
    assert rel.max() <= 1e-5, rel.max()


def test_temperature_bound():
    """in_batch_binades: 2 log2(e) / tau, plus log2(B / vmin) only when the smallest weight vmin / B is below 1 (a larger
    weight cannot pull ex2's own result above the flush); ``vmin`` is the smallest positive weight after fp32 rounding."""
    assert E.in_batch_binades(4096, 0.1, 1.0) == pytest.approx(2 * E.LOG2E / 0.1 + 12, rel=1e-15)
    assert E.in_batch_binades(1, 0.1, 2.0 ** 30) == pytest.approx(2 * E.LOG2E / 0.1, rel=1e-15)
    assert IB.smallest_tau(1, 2.0 ** 30) == IB.smallest_tau(1, 1.0)
    assert 0.0255 < IB.smallest_tau(4096, 1.0) < 0.0256
    w = E.InBatchWeights(np.array([0.0, 3.0, 1e-3 + 1e-12, 7.0]), 'cpu')
    assert w.vmin == float(np.float32(1e-3 + 1e-12))
    # every temperature of the existing in-batch cases is far inside the bound (B <= 8192, weights >= 2^-30)
    assert E.in_batch_binades(8192, 0.05, 2.0 ** -30) < E.IN_BATCH_MAX_BINADES


# ---- whole steps on host draws: the float32 oracle meets the bounds of tests/test_gpu_ssm_in_batch.py, wrong terms miss ----------

def _step_cases():
    seen, out = set(), []
    for rid, m, name, hp, d, tau, _, _, _ in H.in_batch_step_cases():
        if name == 'paths' and (m, repr(hp), d, tau) not in seen:
            seen.add((m, repr(hp), d, tau))
            out.append(pytest.param(m, hp, d, tau, id=rid))
    return out


def _popularity_only(case):
    """The popularity-only law v = 1 / p_i (the negative slot's r_i dropped; a cold item clamped to p_i = 1 / |E|)."""
    p = np.bincount(case['cols'], minlength=case['n_item']) / len(case['cols'])
    return 1.0 / np.maximum(p, 1.0 / len(case['cols']))


@pytest.mark.parametrize('model_key,hp_over,dim,tau', _step_cases())
def test_whole_step_float32_meets_the_bounds_and_wrong_terms_do_not(model_key, hp_over, dim, tau):
    """The float32 oracle is within path_errors of float64 on every whole-step case of the GPU test; each wrong term misses
    them, by the reported factor: tau (1 + 1e-3), uniform weights, the popularity-only law, de-duplicated columns, the
    columns ordered [negs; poss] (the diagonal read from the negatives).  w_c not divided by B shifts every loss_b by ln B
    and leaves the gradients alone: its loss misses and its gradients pass."""
    case, hp, adj, dr, st = H.bpr_term_setup(model_key, hp_over, dim)
    assert H.kink_margin(model_key, case, hp, adj, dr, st) > H.KINK_MARGIN
    ancs, poss, negs = (torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs'))
    rowptr, cols = H.train_csr(case)
    v = E.in_batch_weights(rowptr, cols, case['n_item']).astype(np.float32).astype(np.float64)
    if tau == H.IN_BATCH_SMALLEST_TAU:
        tau = IB.smallest_tau(len(ancs), E.InBatchWeights(v, 'cpu').vmin)
        assert 0.023 < tau < 0.025, tau

    def run(dtype, t=tau, w=v, **kw):
        return H.bpr_term_oracle(model_key, case, hp, adj, dr, st, dtype,
                                 lambda u, i, _: IB.term64(u, i, ancs, poss, negs, t, w, **kw), 'ssm_loss')

    ref = run(torch.float64)
    ok = H.path_errors(run(torch.float32), ref)
    assert max(ok.values()) <= 1.0, ok
    wrong = {'tau (1 + 1e-3)': dict(t=tau * (1 + 1e-3)), 'uniform weights': dict(w=np.ones_like(v)),
             'popularity-only weights': dict(w=_popularity_only(case)), 'de-duplicated columns': dict(dedup=True),
             'columns [negs; poss]': dict(swap=True)}
    report = [f'float32 {max(ok.values()):.3f}']
    for what, kw in wrong.items():
        bad = H.path_errors(run(torch.float32, **kw), ref)
        assert max(bad.values()) > 1.0, (what, 'passes', bad)
        report.append(f'{what} {max(bad.values()):.3g}')
    bad = H.path_errors(run(torch.float32, per_b=False), ref)
    grads = {k: e for k, e in bad.items() if k.startswith('grad_')}
    assert bad['loss'] > 1.0 and bad['part_ssm_loss'] > 1.0 and max(grads.values()) <= 1.0, bad
    report.append(f'w_c undivided: loss {bad["loss"]:.3g}, gradients {max(grads.values()):.3f}')
    print('largest error as a fraction of its bound: ' + ', '.join(report))
