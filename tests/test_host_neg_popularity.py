"""Popularity-proportional candidates (train.neg_popularity) without a GPU.

The key's validation and refusals (a value that is not a number in [0, 1], train.dns_candidates below 2, DirectAU, a row-sharded
model, data-parallel gradient sync) and the training checkpoint's record of the key.  The host tables of engine.pop_tables: the
integer weights sum to n_item 2^32 exactly and the shares the alias table realises, recomputed from {thr, alias} in integers,
equal them exactly; beta = 0 is uniform with every column self-aliased; Zipf-skewed degrees, items of degree 0, n_item = 1; the
same table on every call; the per-user tables, a user who has every item included.  The numpy draw oracle (tests/pop_oracle)
against a scalar restatement of the documented rule and its cap.  The draw kernel and the logQ forward of csrc/ssm.cuh run on the
host under AddressSanitizer (tests/emu/pop_negs_emu.cpp) and equal the oracle and the float32 restatement bit for bit; with
bias = 0 the logQ forward equals ssm_fwd_kernel bit for bit.  On every whole-step case of tests/test_gpu_neg_popularity.py, on
host draws: the fp32 bias is within pop_oracle.bias_tol of bias64 (beta 0, 0.75 and 1); the float32 oracle with it meets the GPU
test's bounds against the float64 oracle with bias64, and five wrong corrections (none, column 0 corrected as a popularity
draw, lz_pop = 0, the bias of permuted anchors, tables of beta 0.7) do not."""
import math
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
import scipy.sparse as sp

import torch

import pop_oracle as O
import ssl_test_helpers as H
import ssm_oracle as S
from oracle import philox as P
from sslrec_b200 import engine as E
from test_host_resume import make_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']
K = 1 << 32


# ---- the key ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('value', [True, False, -0.1, 1.5, 2, -1, float('inf'), float('nan'), '0.5', [0.5]])
def test_bad_values_are_refused_at_construction(value):
    with pytest.raises(ValueError, match=r'train.neg_popularity must be a number in \[0, 1\] or null'):
        make_run('lightgcn', train=dict(neg_popularity=value, dns_candidates=8))


@pytest.mark.parametrize('key', BPR_MODELS)
def test_every_bpr_model_accepts_the_key(key):
    for beta in (0, 1, 0.75):
        m = make_run(key, train=dict(neg_popularity=beta, dns_candidates=8))[0]
        assert m.neg_popularity == float(beta) and m._pop is None
    for train in ({}, dict(neg_popularity=None), dict(neg_popularity=None, dns_candidates=8)):
        assert make_run(key, train=train)[0].neg_popularity is None


def test_one_candidate_and_directau_are_refused():
    with pytest.raises(ValueError, match='which must then be >= 2, got 1'):
        make_run('lightgcn', train=dict(neg_popularity=0.5))
    with pytest.raises(ValueError, match='which must then be >= 2, got 1'):
        make_run('lightgcn', train=dict(neg_popularity=0.5, ssm_temperature=0.1))
    assert make_run('directau', train=dict(neg_popularity=None))[0].neg_popularity is None
    with pytest.raises(ValueError, match='train.neg_popularity: DirectAU trains without negatives'):
        make_run('directau', train=dict(neg_popularity=0.5))


def test_multi_gpu_is_refused():
    from sslrec_b200.trainer import Trainer
    m, _, dh = make_run('simgcl', train=dict(neg_popularity=0.5, dns_candidates=8))
    m.dns_candidates = 1                       # the draw key alone must refuse the row-sharded model
    with pytest.raises(ValueError, match='train.neg_popularity is single-GPU'):
        m.shard_to(types.SimpleNamespace(shard_propagation=False))
    assert m.comm is None
    with pytest.raises(ValueError, match='single-GPU'):
        Trainer(dh, grad_sync=object())
    _, _, dh = make_run('simgcl', train=dict(neg_popularity=None, dns_candidates=1))
    Trainer(dh, grad_sync=object())             # without the key nothing changes


def test_grad_sync_names_the_key():
    from sslrec_b200 import config
    from sslrec_b200.trainer import Trainer
    _, _, dh = make_run('simgcl', train=dict(neg_popularity=0.5, dns_candidates=8))
    config.configs['train']['dns_candidates'] = 1          # the earlier refusal would name train.dns_candidates
    with pytest.raises(ValueError, match='train.neg_popularity is single-GPU'):
        Trainer(dh, grad_sync=object())


def test_checkpoints_record_the_key_only_when_it_is_set(tmp_path):
    a, plain = str(tmp_path / 'a.pth'), str(tmp_path / 'plain.pth')
    m, tr, _ = make_run('ncl', train=dict(neg_popularity=0.5, dns_candidates=8))
    assert tr._resume_record(m, 'host')['neg_popularity'] == 0.5
    tr.save_checkpoint(m, a)
    m, tr, _ = make_run('ncl', train=dict(dns_candidates=8))
    assert 'neg_popularity' not in tr._resume_record(m, 'host')
    tr.save_checkpoint(m, plain)
    with pytest.raises(ValueError, match='neg_popularity: saved 0.5, now None'):
        tr.load_checkpoint(m, a)
    m, tr, _ = make_run('ncl', train=dict(neg_popularity=0.75, dns_candidates=8))
    with pytest.raises(ValueError, match='neg_popularity: saved 0.5, now 0.75'):
        tr.load_checkpoint(m, a)
    with pytest.raises(ValueError, match='neg_popularity: saved None, now 0.75'):
        tr.load_checkpoint(m, plain)
    m, tr, _ = make_run('ncl', train=dict(neg_popularity=0.5, dns_candidates=8))
    assert tr.load_checkpoint(m, a) == 0
    assert m._pop is None                       # the tables are not part of a checkpoint


# ---- the host tables ---------------------------------------------------------------------------------------------------------

def _csr(rows, cols, n_user, n_item):
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    m.sum_duplicates()
    m.sort_indices()
    return m.indptr.astype(np.int64), m.indices.astype(np.int64)


def _zipf_graph(n_user, n_item, n_edge, seed, a=1.2):
    """Zipf-skewed item degrees; the items above n_item * 0.8 never occur (degree 0)."""
    rs = np.random.RandomState(seed)
    hot = max(1, int(n_item * 0.8))
    cols = (rs.zipf(a, n_edge) - 1) % hot
    rows = rs.randint(0, n_user, n_edge)
    return _csr(rows, cols, n_user, n_item)


def _check_table(t, indptr, indices, n_item, beta):
    V, table = t['V'], t['table']
    assert V.dtype == np.int64 and int(V.sum()) == n_item * K and int(V.min()) >= 1
    assert table.shape == (n_item, 2) and table.dtype == np.uint32
    assert np.array_equal(O.column_shares(table), V)
    # each V_i is within one unit of its real-valued target n_item 2^32 w_i / sum w
    w = (np.bincount(indices, minlength=n_item) + 1.0) ** beta
    x = w * float(n_item * K) / math.fsum(w.tolist())
    assert np.abs(V - x).max() <= 1.0 + 8 * 2.0 ** -52 * x.max()


@pytest.mark.parametrize('beta', [0.0, 0.25, 0.75, 1.0])
def test_alias_table_realises_the_weights_exactly(beta):
    indptr, indices = _zipf_graph(300, 1009, 20000, 1)
    t = E.pop_tables(indptr, indices, 1009, beta)
    _check_table(t, indptr, indices, 1009, beta)
    deg = np.bincount(indices, minlength=1009)
    assert (deg[int(1009 * 0.8):] == 0).all()
    t2 = E.pop_tables(indptr, indices, 1009, beta)
    for k in t:
        assert np.array_equal(t[k], t2[k]), k                      # the same table on every call
    if beta > 0:
        assert (t['table'][:, 1] != np.arange(1009)).any()
        assert t['V'][np.argmax(deg)] > t['V'][int(1009 * 0.9)]   # the hottest item outweighs a degree-0 one


def test_beta_zero_is_uniform_with_every_column_self_aliased():
    indptr, indices = _zipf_graph(50, 333, 3000, 2)
    t = E.pop_tables(indptr, indices, 333, 0)
    assert (t['V'] == K).all()
    assert np.array_equal(t['table'][:, 1], np.arange(333, dtype=np.uint32))
    assert np.array_equal(t['lp'], np.full(333, np.float32(-math.log(333))))
    # the uniform draw: item = column
    rs = np.random.RandomState(0)
    x, y = rs.randint(0, 2 ** 32, 1000, dtype=np.uint64).astype(np.uint32), rs.randint(0, 2 ** 32, 1000, dtype=np.uint64).astype(np.uint32)
    assert np.array_equal(O.alias_item(t['table'], 333, x, y), (x.astype(np.uint64) * 333 >> np.uint64(32)).astype(np.int64))


def test_one_item_and_a_single_hot_item():
    t = E.pop_tables(np.array([0, 1, 1]), np.array([0]), 1, 0.75)
    assert t['V'].tolist() == [K] and t['table'].tolist() == [[0, 0]] and t['lp'].tolist() == [0.0]
    assert t['lz_pop'].tolist() == [0.0, 0.0] and t['lz_uni'].tolist() == [0.0, 0.0]     # user 0 has every item; user 1 none
    # one item holding almost every interaction
    rows = np.arange(5000) % 400
    cols = np.where(np.arange(5000) < 4990, 3, np.arange(5000) % 17)
    indptr, indices = _csr(rows, cols, 400, 17)
    for beta in (0.5, 1.0):
        t = E.pop_tables(indptr, indices, 17, beta)
        _check_table(t, indptr, indices, 17, beta)


def test_per_user_tables():
    n_item = 23
    rows = np.array([0] * n_item + [1] * (n_item - 1) + [2, 2, 2])
    cols = np.array(list(range(n_item)) + [i for i in range(n_item) if i != 7] + [1, 5, 9])
    rows = np.concatenate([rows, np.arange(3, 40)])
    cols = np.concatenate([cols, np.arange(3, 40) % 4])
    indptr, indices = _csr(rows, cols, 41, n_item)
    t = E.pop_tables(indptr, indices, n_item, 0.75)
    V, T = t['V'], n_item * K
    for u in range(41):
        row = indices[indptr[u]:indptr[u + 1]]
        left = T - int(V[row].sum())
        assert t['lz_pop'][u] == (np.float32(math.log(left / T)) if left else 0.0), u
        assert t['lz_uni'][u] == (np.float32(math.log(n_item - len(row))) if len(row) < n_item else 0.0), u
    assert t['lz_pop'][0] == 0.0 and t['lz_uni'][0] == 0.0                # every item: 0 in both
    assert t['lz_pop'][1] == np.float32(math.log(int(V[7]) / T))            # every item but 7: log q(7)
    assert t['lz_uni'][1] == 0.0 and t['lz_uni'][40] == np.float32(math.log(n_item))
    assert np.array_equal(t['lp'], np.log(V / float(T)).astype(np.float32))


def test_one_million_items_round_exactly():
    rs = np.random.RandomState(4)
    n_item = 1 << 20
    cols = np.unique((rs.zipf(1.1, 400000) - 1) % n_item)
    indptr = np.array([0, len(cols)])
    t = E.pop_tables(indptr, cols, n_item, 0.75)
    assert int(t['V'].sum()) == n_item * K and int(t['V'].min()) >= 1
    assert np.array_equal(O.column_shares(t['table']), t['V'])


# ---- the draw oracle ---------------------------------------------------------------------------------------------------------

def _scalar_candidate(u, b, j, indptr, indices, n_item, table, seed):
    pos = set(indices[indptr[u]:indptr[u + 1]].tolist())
    for t in range(128):
        r = P.philox4x32_10(b, j, t // 2, O.TAG_DNSP, seed)
        x, y = int(r[2 * (t % 2)]), int(r[2 * (t % 2) + 1])
        c = (x * n_item) >> 32
        thr, alias = int(table[c, 0]), int(table[c, 1])
        item = c if alias == c or y < thr else alias
        if item not in pos:
            return item
    return item


def test_draw_oracle_matches_a_scalar_restatement_and_the_cap():
    n_item = 37
    indptr, indices = _zipf_graph(40, n_item, 600, 3)
    # user 0 every item (the capped draw), user 1 every item but 11
    rows = np.concatenate([np.zeros(n_item, np.int64), np.ones(n_item - 1, np.int64)])
    cols = np.concatenate([np.arange(n_item), np.delete(np.arange(n_item), 11)])
    m = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(40, n_item)).tolil()
    m[0, :] = 0
    m[1, :] = 0
    m = (m.tocsr() + sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(40, n_item))).tocsr()
    m.data[:] = 1
    m.sort_indices()
    indptr, indices = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    t = E.pop_tables(indptr, indices, n_item, 0.75)
    rs = np.random.RandomState(1)
    users = rs.randint(0, 40, 29)
    users[:3] = [0, 1, 0]
    negs = rs.randint(0, n_item, 29)
    seed = 0xDEADBEEF12345678
    got = O.neg_candidates(users, negs, 9, indptr, indices, n_item, t['table'], seed)
    assert np.array_equal(got[:, 0], negs)
    for b in range(29):
        for j in range(1, 9):
            assert got[b, j] == _scalar_candidate(users[b], b, j, indptr, indices, n_item, t['table'], seed), (b, j)
    assert (got[1, 1:] == 11).all()
    r = P.philox4x32_10(0, 1, 63, O.TAG_DNSP, seed)
    assert got[0, 1] == O.alias_item(t['table'], n_item, r[2:3], r[3:4])[0]      # 128 rejected: the last draw
    assert not np.array_equal(got, O.neg_candidates(users, negs, 9, indptr, indices, n_item, t['table'], seed + 1))


# ---- the kernels on the host -------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def emulator(tmp_path_factory):
    if shutil.which('g++') is None:
        pytest.skip('needs g++')
    exe = str(tmp_path_factory.mktemp('emu') / 'pop_negs_emu')
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-fsanitize=address', '-fno-omit-frame-pointer', '-pthread', '-Wno-unknown-pragmas',
           '-I', os.path.join(ROOT, 'sslrec_b200', 'csrc'), '-I', os.path.join(ROOT, 'tests', 'emu'),
           os.path.join(ROOT, 'tests', 'emu', 'pop_negs_emu.cpp'), '-o', exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _run(emulator, tmp_path, mode, parts):
    fin, fout = str(tmp_path / 'in.bin'), str(tmp_path / 'out.bin')
    with open(fin, 'wb') as f:
        for a in parts:
            a.tofile(f)
    r = subprocess.run([emulator, mode, fin, fout], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return fout


@pytest.mark.parametrize('B,M,n_item,beta', [(1, 2, 1, 0.5), (37, 8, 97, 0.75), (300, 3, 1000, 1.0), (9, 256, 61, 0.0),
                                             (257, 33, 250, 0.5)])
def test_draw_kernel_is_the_oracle_on_the_host(emulator, tmp_path, B, M, n_item, beta):
    n_user = 40
    indptr, indices = _zipf_graph(n_user, n_item, 15 * n_user, B + M)
    # user 0 has every item (lz 0, capped draw)
    rows = np.concatenate([np.repeat(np.arange(n_user), np.diff(indptr)), np.zeros(n_item, np.int64)])
    cols = np.concatenate([indices, np.arange(n_item)])
    indptr, indices = _csr(rows, cols, n_user, n_item)
    t = E.pop_tables(indptr, indices, n_item, beta)
    rs = np.random.RandomState(B)
    users = rs.randint(0, n_user, B)
    users[0] = 0
    negs = rs.randint(0, n_item, B)
    seed = 0x0123456789ABCDEF ^ M
    ln_m = np.float32(math.log(M))
    fout = _run(emulator, tmp_path, 'draw', [
        np.array([B, M, n_item, n_user, len(indices)], np.int64), np.array([seed], np.uint64), np.array([ln_m], np.float32),
        indptr.astype(np.int32), indices.astype(np.int32), np.ascontiguousarray(t['table']), t['lp'], t['lz_pop'], t['lz_uni'],
        users.astype(np.int64), negs.astype(np.int64)])
    with open(fout, 'rb') as f:
        cands = np.fromfile(f, np.int64, B * M).reshape(B, M)
        bias = np.fromfile(f, np.float32, B * M).reshape(B, M)
        cands2 = np.fromfile(f, np.int64, B * M).reshape(B, M)
    want = O.neg_candidates(users, negs, M, indptr, indices, n_item, t['table'], seed)
    assert np.array_equal(cands, want) and np.array_equal(cands2, want)
    assert np.array_equal(bias.view(np.uint32), O.bias(users, want, t['lp'], t['lz_pop'], t['lz_uni']).view(np.uint32))
    assert (bias[users == 0] == np.where(np.arange(M) == 0, ln_m, (ln_m + t['lp'][cands[users == 0]]).astype(np.float32))).all()


@pytest.mark.parametrize('B,M,d,tau', [(1, 1, 4, 0.02), (37, 8, 32, 0.1), (70, 33, 48, 0.02), (9, 256, 64, 0.5), (130, 3, 128, 0.07)])
def test_logq_forward_is_its_restatement_on_the_host(emulator, tmp_path, B, M, d, tau):
    rs = np.random.default_rng(B + M + d)
    nu, ni = 31, 47 + M
    ut = rs.standard_normal((nu, d)).astype(np.float32)
    it = rs.standard_normal((ni, d)).astype(np.float32)
    ancs, poss, cands = rs.integers(0, nu, B), rs.integers(0, ni, B), rs.integers(0, ni, (B, M))
    cands[::3, -1] = poss[::3]
    u, c = ut[ancs], it[np.concatenate([poss[:, None], cands], 1)]
    out = {}
    for name, bias in (('bias', (rs.standard_normal((B, M)) * 3 - 2).astype(np.float32)), ('zero', np.zeros((B, M), np.float32))):
        fout = _run(emulator, tmp_path, 'ssm', [np.array([B, M, d, nu, ni], np.int64), np.array([tau], np.float32), ut, it,
                                                ancs.astype(np.int64), poss.astype(np.int64), cands.astype(np.int64), bias])
        Q = M + 1
        got = np.split(np.fromfile(fout, np.float32), np.cumsum([B, B * Q, B * Q, B * (Q + 1)] * 2)[:-1])
        logq, plain = got[:4], got[4:]
        want = O.forward32_logq(u, c, tau, bias)
        for k, (g, w) in enumerate(zip(logq, want)):
            assert np.array_equal(g.view(np.uint32), w.ravel().view(np.uint32)), (name, k)
        out[name] = (logq, plain)
    # bias = 0: the logq forward is the plain forward bit for bit (and s is raw either way)
    for g, w in zip(*out['zero']):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
    plain = S.forward32(u, c, tau)
    assert np.array_equal(out['bias'][0][1].view(np.uint32), plain[1].ravel().view(np.uint32))


# ---- whole-step cases of tests/test_gpu_neg_popularity.py::test_whole_step_against_float64, on host draws ------------------------

CASES = H.bpr_term_cases(ssm=True)
BETA, SEED = 0.75, 0x5EED0123456789AB


def _host_draw(case, M, beta):
    """The popularity candidates of the case's batch on host tables -> (rowptr, cols, tables, candidates)."""
    rowptr, cols = H.train_csr(case)
    t = E.pop_tables(rowptr, cols, case['n_item'], beta)
    return rowptr, cols, t, O.neg_candidates(case['ancs'], case['negs'], M, rowptr, cols, case['n_item'], t['table'], SEED)


@pytest.mark.parametrize('beta', [0.0, BETA, 1.0])
@pytest.mark.parametrize('model_key,hp_over,dim,M,tau', CASES, ids=[H.bpr_term_case_id(c) for c in CASES])
def test_fp32_bias_is_within_its_bound_of_bias64(model_key, hp_over, dim, M, tau, beta):
    case = H.path_case(dim, seed=H.BPR_TERM_SEEDS.get((model_key, dim, hp_over.get('hyper_num')), 41))
    _, _, t, cands = _host_draw(case, M, beta)
    b32 = O.bias(case['ancs'], cands, t['lp'], t['lz_pop'], t['lz_uni'])
    args = (case['ancs'], cands, case['rows'], case['cols'], case['n_user'], case['n_item'], beta, M)
    frac = np.abs(b32 - O.bias64(*args)) / O.bias_tol(*args)
    print(f'{H.bpr_term_case_id((model_key, hp_over, dim, M, tau))} beta {beta}: fp32 bias {frac.max():.3f} of its bound')
    assert frac.max() <= 1.0, frac.max()


def _mutations(case, M, t, cands):
    """Slightly wrong fp32 biases of the same candidates: name -> [B, M] float32, or None for no correction."""
    ancs = case['ancs']
    f = np.float32
    col0_pop = O.bias(ancs, cands, t['lp'], t['lz_pop'], t['lz_uni'])
    col0_pop[:, 0] = (f(math.log(M)) + t['lp'][case['negs']]).astype(f) - t['lz_pop'][ancs]
    rowptr, cols = H.train_csr(case)
    t07 = E.pop_tables(rowptr, cols, case['n_item'], 0.7)
    return {
        'no correction': None,
        'column 0 as a popularity draw': col0_pop,
        'lz_pop = 0': O.bias(ancs, cands, t['lp'], np.zeros_like(t['lz_pop']), t['lz_uni']),
        'anchors permuted': O.bias(ancs[np.random.RandomState(7).permutation(len(ancs))], cands, t['lp'], t['lz_pop'], t['lz_uni']),
        'tables of beta 0.7': O.bias(ancs, cands, t07['lp'], t07['lz_pop'], t07['lz_uni']),
    }


@pytest.mark.parametrize('model_key,hp_over,dim,M,tau', CASES, ids=[H.bpr_term_case_id(c) for c in CASES])
def test_whole_step_float32_meets_the_bounds_and_wrong_corrections_do_not(model_key, hp_over, dim, M, tau):
    """The float32 oracle with the fp32 bias of pop_oracle.bias is within the GPU test's bounds of the float64 oracle with
    bias64 (both on the same host-drawn popularity candidates, beta 0.75); with a wrong bias (none, column 0 corrected as a
    popularity draw, lz_pop = 0, the bias of permuted anchors, tables of beta 0.7) it is outside them."""
    case, hp, adj, dr, st = H.bpr_term_setup(model_key, hp_over, dim)
    assert H.kink_margin(model_key, case, hp, adj, dr, st) > H.KINK_MARGIN
    ancs, poss = torch.from_numpy(case['ancs']), torch.from_numpy(case['poss'])
    _, _, t, cands = _host_draw(case, M, BETA)
    b64 = O.bias64(case['ancs'], cands, case['rows'], case['cols'], case['n_user'], case['n_item'], BETA, M)
    c = torch.from_numpy(cands)

    def run(dtype, bias):
        term = ((lambda u, i, _: S.term64(u, i, ancs, poss, c, tau)) if bias is None else
                (lambda u, i, _: O.term64_logq(u, i, ancs, poss, c, tau, bias)))
        return H.bpr_term_oracle(model_key, case, hp, adj, dr, st, dtype, term, 'ssm_loss')

    ref = run(torch.float64, b64)
    ok = max(H.path_errors(run(torch.float32, O.bias(case['ancs'], cands, t['lp'], t['lz_pop'], t['lz_uni'])), ref).values())
    bad = {name: max(H.path_errors(run(torch.float32, b), ref).values()) for name, b in _mutations(case, M, t, cands).items()}
    print(f'{H.bpr_term_case_id((model_key, hp_over, dim, M, tau))}: float32 oracle {ok:.3f} of the bound; wrong biases ' +
          ', '.join(f'{k} {v:.3g}x' for k, v in bad.items()))
    assert ok <= 1.0, ok
    assert min(bad.values()) > 1.0, ('a wrong bias passes', bad)
