"""In-batch negatives for the sampled softmax (train.ssm_in_batch) without a GPU: the key's bad values, acceptance on the six BPR
models and every refusal (no temperature, drawn candidates, popularity draws, DirectAU, a row-sharded model, data-parallel
gradient sync), the checkpoint record; ``engine.in_batch_weights`` against a brute-force float64 restatement of p_i and r_i;
the loaders' sampling law itself (HostBatchLoader with ``sample_negs`` over many epochs: the column counts by a chi-square test,
the weighted column sum as an unbiased estimate of the catalogue sum within a CLT bound); and the column-backward kernel
(csrc/ssm_in_batch.cuh) under AddressSanitizer through tests/emu, bit for bit against its sequential float32 restatement."""
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
