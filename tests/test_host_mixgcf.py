"""MixGCF negatives (train.mixgcf) without a GPU: the numpy restatement of ssl_mixgcf_bpr_fwd's mixing weights
(tests/mixgcf_oracle.alpha) against a scalar restatement of the documented draw, the float64 picks and term of the oracle on
a hand-made case, the key's validation and refusals (a value that is not a bool, DirectAU, more than 8 layers, a row-sharded
model, data-parallel gradient sync) and the training checkpoint's record of the key."""
import types

import numpy as np
import pytest
import torch

import mixgcf_oracle as X
from oracle import philox as P
from test_host_resume import make_run

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


def test_alpha_oracle_matches_a_scalar_restatement():
    seed = 0xC0FFEE0123456789
    got = X.alpha(37, 5, seed)
    assert got.dtype == np.float32 and got.shape == (37, 5)
    for b in range(37):
        for l in range(5):
            w = int(P.philox4x32_10(b, l, 0, X.TAG_MIXA, seed)[0])
            assert got[b, l] == np.float32((w >> 8) / 16777216.0), (b, l)
    assert ((got >= 0) & (got < 1)).all()
    assert not np.array_equal(got, X.alpha(37, 5, seed + 1))
    assert np.array_equal(X.alpha(37, 5, seed)[:, :3], X.alpha(37, 3, seed))     # a pair's weights do not depend on L


def test_oracle_picks_and_term_on_a_hand_made_case():
    users = torch.tensor([[1.0, 0.0]])
    items = torch.tensor([[0.0, 0.0], [0.5, 0.0], [2.0, 1.0], [2.0, -1.0], [float('nan'), 0.0]])
    layers = [items, items * torch.tensor([-1.0, 1.0])]          # layer 1 reverses the order of the first coordinate
    ancs, poss = torch.tensor([0, 0]), torch.tensor([1, 1])
    cands = torch.tensor([[1, 2, 3], [4, 0, 4]])
    a = torch.tensor([[0.5, 0.0], [0.25, 0.0]])
    got = X.picks(users, layers, ancs, poss, cands, a)
    # pair 0: layer 0 ties between 2 and 3 (lowest j wins), layer 1 prefers item 1; pair 1: NaN never wins
    assert got.tolist() == [[2, 1], [0, 0]]
    a = a.double()
    want = 0.0
    for b in range(2):
        nhat = sum(a[b, l] * x[1].double() + (1 - a[b, l]) * x[got[b, l]].double() for l, x in enumerate(layers))
        want += float(torch.nn.functional.softplus(users[0].double() @ nhat - users[0].double() @ items[1].double()))
    assert abs(float(X.term(users.double(), items.double(), [x.double() for x in layers], ancs, poss, got, a)) - want) < 1e-12


@pytest.mark.parametrize('value', [1, 0, 'true', None, 2.5])
def test_bad_values_are_refused_at_construction(value):
    with pytest.raises(ValueError, match='train.mixgcf must be true or false'):
        make_run('lightgcn', train=dict(mixgcf=value))


@pytest.mark.parametrize('key', BPR_MODELS)
def test_every_bpr_model_accepts_the_key(key):
    m, _, _ = make_run(key, train=dict(mixgcf=True, dns_candidates=8))
    assert m.mixgcf and m.mixgcf_picks is None and m.mixgcf_alpha is None and m.dns_negs is None
    assert not make_run(key)[0].mixgcf
    assert not make_run(key, train=dict(mixgcf=False))[0].mixgcf


def test_directau_is_refused():
    assert not make_run('directau', train=dict(mixgcf=False))[0].mixgcf
    with pytest.raises(ValueError, match='train.mixgcf: DirectAU trains without negatives'):
        make_run('directau', train=dict(mixgcf=True))


def test_more_than_eight_layers_are_refused():
    assert make_run('lightgcn', train=dict(mixgcf=True), model=dict(layer_num=7))[0].mixgcf
    with pytest.raises(ValueError, match='at most 8 layers'):
        make_run('lightgcn', train=dict(mixgcf=True), model=dict(layer_num=8))
    assert not make_run('lightgcn', model=dict(layer_num=8))[0].mixgcf     # without the key nothing changes


def test_multi_gpu_is_refused():
    from sslrec_b200.trainer import Trainer
    m, _, dh = make_run('simgcl', train=dict(mixgcf=True))
    with pytest.raises(ValueError, match='train.mixgcf is single-GPU'):
        m.shard_to(types.SimpleNamespace(shard_propagation=False))
    assert m.comm is None
    with pytest.raises(ValueError, match='train.mixgcf is single-GPU'):
        Trainer(dh, grad_sync=object())
    m, _, dh = make_run('simgcl', train=dict(mixgcf=False))
    Trainer(dh, grad_sync=object())             # without the key nothing changes


def test_checkpoints_record_the_key_only_when_it_is_set(tmp_path):
    plain, mixed = str(tmp_path / 'plain.pth'), str(tmp_path / 'mixed.pth')
    m, tr, _ = make_run('ncl', train=dict(mixgcf=True, dns_candidates=8))
    rec = tr._resume_record(m, 'host')
    assert rec['mixgcf'] is True and rec['dns_candidates'] == 8
    tr.save_checkpoint(m, mixed)
    m, tr, _ = make_run('ncl', train=dict(mixgcf=False, dns_candidates=8))
    assert 'mixgcf' not in tr._resume_record(m, 'host')
    tr.save_checkpoint(m, plain)
    with pytest.raises(ValueError, match='mixgcf: saved True, now None'):
        tr.load_checkpoint(m, mixed)
    m, tr, _ = make_run('ncl', train=dict(mixgcf=True, dns_candidates=8))
    with pytest.raises(ValueError, match='mixgcf: saved None, now True'):
        tr.load_checkpoint(m, plain)
    assert tr.load_checkpoint(m, mixed) == 0
    # a record of a run without either key is what it was before the key existed
    m, tr, _ = make_run('ncl')
    assert not {'mixgcf', 'dns_candidates'} & set(tr._resume_record(m, 'host'))
