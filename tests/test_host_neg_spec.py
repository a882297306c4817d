"""The negative-sampling keys of the BPR models (engine.NegSpec) without a GPU, one table per check over the four keys
train.dns_candidates, train.mixgcf, train.ssm_temperature and train.neg_popularity: each key's bad values and their message,
its acceptance on every BPR model, the refusal of DirectAU, of a row-sharded model and of data-parallel gradient sync, and the
training checkpoint's record of the key."""
import dataclasses
import types

import pytest

from sslrec_b200 import engine as E
from test_host_resume import make_run

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']
INF, NAN = float('inf'), float('nan')

# key: (bad values, the message they raise, the other train keys of the run)
BAD = {
    'dns_candidates': ([0, 257, -3, 2.5, True, '8', None], 'dns_candidates', {}),
    'mixgcf': ([1, 0, 'true', None, 2.5], 'train.mixgcf must be true or false', {}),
    'ssm_temperature': ([True, False, 0, 0.0, -0.5, -2, INF, NAN, '0.1', [0.1], 1e-50, 1e39],
                        'train.ssm_temperature must be a finite number > 0 or null', {}),
    'neg_popularity': ([True, False, -0.1, 1.5, 2, -1, INF, NAN, '0.5', [0.5]],
                       r'train.neg_popularity must be a number in \[0, 1\] or null', dict(dns_candidates=8)),
}

# key: (its NegSpec field, (train section, the field's value) pairs that set it, train sections that leave it off)
ACCEPT = {
    'dns_candidates': ('candidates', [(dict(dns_candidates=256), 256)], [{}]),
    'mixgcf': ('mixgcf', [(dict(mixgcf=True, dns_candidates=8), True)], [{}, dict(mixgcf=False)]),
    'ssm_temperature': ('ssm_temperature', [(dict(ssm_temperature=0.1, dns_candidates=8), 0.1), (dict(ssm_temperature=2), 2.0)],
                        [{}, dict(ssm_temperature=None)]),
    'neg_popularity': ('popularity', [(dict(neg_popularity=b, dns_candidates=8), float(b)) for b in (0, 1, 0.75)],
                       [{}, dict(neg_popularity=None), dict(neg_popularity=None, dns_candidates=8)]),
}

# key: (a train section that sets it, one that leaves it off)
SET_OFF = {
    'dns_candidates': (dict(dns_candidates=2), dict(dns_candidates=1)),
    'mixgcf': (dict(mixgcf=True), dict(mixgcf=False)),
    'ssm_temperature': (dict(ssm_temperature=0.1), dict(ssm_temperature=None)),
    'neg_popularity': (dict(neg_popularity=0.5), dict(neg_popularity=None)),
}

# key: (the train section of a multi-GPU run that is refused, of one that is not)
MULTI_GPU = {
    'dns_candidates': (dict(dns_candidates=8), {}),
    'mixgcf': (dict(mixgcf=True), dict(mixgcf=False)),
    'ssm_temperature': (dict(ssm_temperature=0.1), dict(ssm_temperature=None)),
    'neg_popularity': (dict(neg_popularity=0.5, dns_candidates=8), dict(neg_popularity=None, dns_candidates=1)),
}

# key: (the other train keys, the value saved, another value (None: the key has one), the value that leaves the key off)
RECORD = {
    'dns_candidates': ({}, 8, 4, 1),
    'mixgcf': (dict(dns_candidates=8), True, None, False),
    'ssm_temperature': (dict(dns_candidates=8), 0.1, 0.2, None),
    'neg_popularity': (dict(dns_candidates=8), 0.5, 0.75, None),
}


@pytest.mark.parametrize('key,value', [(k, v) for k, (values, _, _) in BAD.items() for v in values])
def test_bad_values_are_refused_at_construction(key, value):
    _, match, other = BAD[key]
    with pytest.raises(ValueError, match=match):
        make_run('lightgcn', train={**other, key: value})


@pytest.mark.parametrize('model_key', BPR_MODELS)
@pytest.mark.parametrize('key', list(ACCEPT))
def test_every_bpr_model_accepts_the_key(key, model_key):
    field, on, off = ACCEPT[key]
    for train, value in on:
        m = make_run(model_key, train=train)[0]
        got = getattr(m.neg, field)
        assert got == value and type(got) is type(value), train
        assert m.dns_negs is None and m.mixgcf_picks is None and m.mixgcf_alpha is None and m._pop is None
        assert m.bpr_loss_name == ('bpr_loss' if m.neg.ssm_temperature is None else 'ssm_loss')
    for train in off:
        m = make_run(model_key, train=train)[0]
        assert getattr(m.neg, field) == getattr(E.NegSpec(), field) and m.bpr_loss_name == 'bpr_loss', train


def test_directau_is_refused():
    for key, (on, off) in SET_OFF.items():
        assert make_run('directau', train=off)[0].neg == E.NegSpec(), key
        with pytest.raises(ValueError, match=f'train.{key}: DirectAU trains without negatives'):
            make_run('directau', train=on)


def test_multi_gpu_is_refused():
    from sslrec_b200.trainer import Trainer
    for key, (on, off) in MULTI_GPU.items():
        m, _, dh = make_run('simgcl', train=on)
        if key == 'neg_popularity':
            m.neg = dataclasses.replace(m.neg, candidates=1)         # the draw key alone must refuse the row-sharded model
        with pytest.raises(ValueError, match=f'train.{key} is single-GPU'):
            m.shard_to(types.SimpleNamespace(shard_propagation=False))
        assert m.comm is None, key
        named = 'dns_candidates' if on.get('dns_candidates', 1) > 1 else key          # the first key the config sets
        with pytest.raises(ValueError, match=f'train.{named} is single-GPU'):
            Trainer(dh, grad_sync=object())
        _, _, dh = make_run('simgcl', train=off)
        Trainer(dh, grad_sync=object())             # without the key nothing changes


def test_checkpoints_record_the_key_only_when_it_is_set(tmp_path):
    for key, (other, a, b, off) in RECORD.items():
        saved, plain = str(tmp_path / f'{key}.pth'), str(tmp_path / f'{key}-plain.pth')

        def run(value):
            return make_run('ncl', train={**other, key: value})

        m, tr, _ = run(a)
        rec = tr._resume_record(m, 'host')
        assert rec[key] == a and type(rec[key]) is type(a) and rec['dns_candidates'] == 8, key
        tr.save_checkpoint(m, saved)
        m, tr, _ = run(off)
        assert key not in tr._resume_record(m, 'host')
        tr.save_checkpoint(m, plain)
        with pytest.raises(ValueError, match=f'{key}: saved {a!r}, now None'):
            tr.load_checkpoint(m, saved)
        if b is not None:
            m, tr, _ = run(b)
            with pytest.raises(ValueError, match=f'{key}: saved {a!r}, now {b!r}'):
                tr.load_checkpoint(m, saved)
            with pytest.raises(ValueError, match=f'{key}: saved None, now {b!r}'):
                tr.load_checkpoint(m, plain)
        m, tr, _ = run(a)
        with pytest.raises(ValueError, match=f'{key}: saved None, now {a!r}'):
            tr.load_checkpoint(m, plain)
        assert tr.load_checkpoint(m, saved) == 0, key
        assert m._pop is None                       # the popularity tables are not part of a checkpoint
    # a record of a run without any of the keys is what it was before they existed
    m, tr, _ = make_run('ncl')
    assert not set(RECORD) & set(tr._resume_record(m, 'host'))
