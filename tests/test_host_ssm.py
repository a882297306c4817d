"""The sampled softmax loss (train.ssm_temperature) without a GPU: the key's validation and refusals (a value that is not a
finite number > 0, the key together with train.mixgcf, DirectAU, a row-sharded model, data-parallel gradient sync), the
training checkpoint's record of the key, and the oracle's identities (M = 1 is softplus(s_0' - s_+); the fp32 restatement
against float64)."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ssm_oracle as S
from test_host_resume import make_run

BPR_MODELS = ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf', 'lightgcl']


@pytest.mark.parametrize('value', [True, False, 0, 0.0, -0.5, -2, float('inf'), float('nan'), '0.1', [0.1], 1e-50, 1e39])
def test_bad_values_are_refused_at_construction(value):
    with pytest.raises(ValueError, match='train.ssm_temperature must be a finite number > 0 or null'):
        make_run('lightgcn', train=dict(ssm_temperature=value))


@pytest.mark.parametrize('key', BPR_MODELS)
def test_every_bpr_model_accepts_the_key(key):
    m, _, _ = make_run(key, train=dict(ssm_temperature=0.1, dns_candidates=8))
    assert m.ssm_temperature == 0.1 and m.bpr_loss_name == 'ssm_loss' and m.dns_negs is None
    assert make_run(key, train=dict(ssm_temperature=2))[0].ssm_temperature == 2.0          # an int is a number
    for train in ({}, dict(ssm_temperature=None)):
        m = make_run(key, train=train)[0]
        assert m.ssm_temperature is None and m.bpr_loss_name == 'bpr_loss'


def test_mixgcf_is_refused():
    with pytest.raises(ValueError, match='train.ssm_temperature and train.mixgcf both replace the BPR term'):
        make_run('lightgcn', train=dict(ssm_temperature=0.1, mixgcf=True))
    assert make_run('lightgcn', train=dict(ssm_temperature=0.1, mixgcf=False))[0].ssm_temperature == 0.1


def test_directau_is_refused():
    assert make_run('directau', train=dict(ssm_temperature=None))[0].ssm_temperature is None
    with pytest.raises(ValueError, match='train.ssm_temperature: DirectAU trains without negatives'):
        make_run('directau', train=dict(ssm_temperature=0.1))


def test_multi_gpu_is_refused():
    from sslrec_b200.trainer import Trainer
    m, _, dh = make_run('simgcl', train=dict(ssm_temperature=0.1))
    with pytest.raises(ValueError, match='train.ssm_temperature is single-GPU'):
        m.shard_to(types.SimpleNamespace(shard_propagation=False))
    assert m.comm is None
    with pytest.raises(ValueError, match='train.ssm_temperature is single-GPU'):
        Trainer(dh, grad_sync=object())
    m, _, dh = make_run('simgcl', train=dict(ssm_temperature=None))
    Trainer(dh, grad_sync=object())             # without the key nothing changes


def test_checkpoints_record_the_key_only_when_it_is_set(tmp_path):
    a, b, plain = str(tmp_path / 'a.pth'), str(tmp_path / 'b.pth'), str(tmp_path / 'plain.pth')
    m, tr, _ = make_run('ncl', train=dict(ssm_temperature=0.1, dns_candidates=8))
    rec = tr._resume_record(m, 'host')
    assert rec['ssm_temperature'] == 0.1 and rec['dns_candidates'] == 8
    tr.save_checkpoint(m, a)
    m, tr, _ = make_run('ncl', train=dict(ssm_temperature=0.2, dns_candidates=8))
    tr.save_checkpoint(m, b)
    with pytest.raises(ValueError, match='ssm_temperature: saved 0.1, now 0.2'):
        tr.load_checkpoint(m, a)
    m, tr, _ = make_run('ncl', train=dict(dns_candidates=8))
    assert 'ssm_temperature' not in tr._resume_record(m, 'host')
    tr.save_checkpoint(m, plain)
    with pytest.raises(ValueError, match='ssm_temperature: saved 0.1, now None'):
        tr.load_checkpoint(m, a)
    m, tr, _ = make_run('ncl', train=dict(ssm_temperature=0.1, dns_candidates=8))
    with pytest.raises(ValueError, match='ssm_temperature: saved None, now 0.1'):
        tr.load_checkpoint(m, plain)
    assert tr.load_checkpoint(m, a) == 0


def _case(B, M, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    users, items = torch.randn(30, d, generator=g, dtype=torch.float64), torch.randn(50, d, generator=g, dtype=torch.float64)
    return users, items, torch.randint(0, 30, (B,), generator=g), torch.randint(0, 50, (B,), generator=g), torch.randint(0, 50, (B, M), generator=g)


def test_oracle_with_one_candidate_is_softplus_of_the_score_gap():
    users, items, ancs, poss, cands = _case(40, 1, 16)
    tau = 0.07
    s = S.scores64(users, items, ancs, poss, cands, tau)
    want = F.softplus(s[:, 1] - s[:, 0]).sum()
    assert abs(float(S.term64(users, items, ancs, poss, cands, tau)) - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
    # cosine scores: scaling a row changes them only through the 1e-8 of the norm
    assert torch.allclose(S.scores64(users * 3, items * 0.5, ancs, poss, cands, tau), s, rtol=1e-7, atol=0)


def test_fp32_restatement_is_close_to_float64():
    users, items, ancs, poss, cands = _case(64, 33, 48, seed=1)
    u = users[ancs].float().numpy()
    c = items[torch.cat([poss[:, None], cands], 1)].float().numpy()
    tau = 0.2
    loss, s, w, nrm = S.forward32(u, c, tau, expf=np.exp, logf=np.log)
    ids = torch.arange(64)
    cid = torch.arange(64, 64 + 64 * 34).view(64, 34)
    ut, ct = torch.from_numpy(u).double().requires_grad_(True), torch.from_numpy(c.reshape(-1, 48)).double().requires_grad_(True)
    s64 = S.scores64(ut, ct, ids, cid[:, 0] - 64, cid[:, 1:] - 64, tau)
    assert np.abs(s - s64.detach().numpy()).max() <= 1e-5 / tau
    ref = torch.logsumexp(s64, 1) - s64[:, 0]
    assert np.abs(loss - ref.detach().numpy()).max() <= 1e-5 * max(1.0, float(ref.abs().max()))
    ref.sum().backward()
    g_u, g_c = S.backward32(u, c, tau, s, w, nrm, 1.0)
    assert np.abs(g_u - ut.grad.numpy()).max() <= 1e-5 * float(ut.grad.abs().max())
    assert np.abs(g_c.reshape(-1, 48) - ct.grad.numpy()).max() <= 1e-5 * float(ct.grad.abs().max())


def test_fma32_is_exact():
    rng = np.random.default_rng(3)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) for _ in range(3))
    from fractions import Fraction
    got = S.fma32(a, b, c)
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = np.float32(float(exact))       # float(Fraction) is correctly rounded; one more rounding can only tie at a midpoint
        lo, hi = np.nextafter(r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))
        best = min((abs(Fraction(float(v)) - exact), v) for v in (lo, r, hi))[1]
        assert got[i] == best, i
    # exact halfway cases in float32 that float64 rounding alone would break
    x = np.float32(1 + 2 ** -23)
    assert S.fma32(x, x, np.float32(-1)) == np.float32(2 ** -22 + 2 ** -46)
