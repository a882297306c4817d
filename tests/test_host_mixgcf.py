"""MixGCF negatives (train.mixgcf) without a GPU: the numpy restatement of ssl_mixgcf_bpr_fwd's mixing weights
(tests/mixgcf_oracle.alpha) against a scalar restatement of the documented draw, the float64 picks and term of the oracle on
a hand-made case, and the refusal of more than 8 layers (the key itself: tests/test_host_neg_spec.py).  On every whole-step
case of tests/test_gpu_mixgcf.py, on host draws: the float32 oracle meets the GPU test's bounds against float64, and three slightly
wrong MixGCF terms (layers 1 .. L reversed, each layer's gradient routed one layer deeper, the positive's share detached) do not."""
import numpy as np
import pytest
import torch

import dns_oracle as D
import mixgcf_oracle as X
import ssl_test_helpers as H
from oracle import philox as P
from test_host_resume import make_run


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


def test_more_than_eight_layers_are_refused():
    assert make_run('lightgcn', train=dict(mixgcf=True), model=dict(layer_num=7))[0].mixgcf
    with pytest.raises(ValueError, match='at most 8 layers'):
        make_run('lightgcn', train=dict(mixgcf=True), model=dict(layer_num=8))
    assert not make_run('lightgcn', model=dict(layer_num=8))[0].mixgcf     # without the key nothing changes


# ---- whole-step cases of tests/test_gpu_mixgcf.py::test_whole_step_against_float64, on host draws ------------------------------

SEED = 0x5EED0123456789AB
CASES = H.bpr_term_cases(ssm=False)


def _host_draws(case, M, L1):
    """Candidates (tests/dns_oracle on the training CSR) and mixing weights (mixgcf_oracle.alpha) of a case, drawn on the host."""
    rowptr, cols = H.train_csr(case)
    cands = D.neg_candidates(case['ancs'], case['negs'], M, rowptr, cols, case['n_item'], SEED)
    return torch.from_numpy(cands), torch.from_numpy(X.alpha(len(case['ancs']), L1, SEED))


def _positive_detached_term(users, items, layers, ancs, poss, pick_ids, alpha_t):
    """mixgcf_oracle.term with no gradient through the positive's share alpha_l X_l[p] of the mixed negative."""
    a = alpha_t.to(users.dtype)
    nhat = sum(a[:, l, None] * x.detach()[poss] + (1 - a[:, l, None]) * x[pick_ids[:, l]] for l, x in enumerate(layers))
    u = users[ancs]
    return torch.nn.functional.softplus((u * nhat).sum(1) - (u * items[poss]).sum(1)).sum()


def _reversed(layers):
    """Layers 1 .. L in reverse order."""
    return layers[:1] + layers[:0:-1]


def _one_layer_deeper(layers):
    """The values of every layer, the gradient of layer l < L routed into layer l + 1."""
    return [x.detach() + (y - y.detach()) for x, y in zip(layers, layers[1:])] + layers[-1:]


@pytest.mark.parametrize('model_key,hp_over,dim,M,tau', CASES, ids=[H.bpr_term_case_id(c) for c in CASES])
def test_whole_step_float32_meets_the_bounds_and_wrong_oracles_do_not(model_key, hp_over, dim, M, tau):
    """The float32 oracle is within the GPU test's bounds of float64 on the same picks and alphas, and its picks agree with
    float64's wherever the gap is decided; each slightly wrong MixGCF term is outside the bounds."""
    case, hp, adj, dr, st = H.bpr_term_setup(model_key, hp_over, dim)
    assert H.kink_margin(model_key, case, hp, adj, dr, st) > H.KINK_MARGIN
    ancs, poss = torch.from_numpy(case['ancs']), torch.from_numpy(case['poss'])
    cands, alpha = _host_draws(case, M, hp['layer_num'] + 1)
    tables = {}
    for dt in (torch.float64, torch.float32):
        with torch.no_grad():
            ue, _, layers = H.bpr_tables(model_key, case, hp, adj, dr, H.path_params(model_key, case, dr, dt))
        tables[dt] = ue.double(), [x.double() for x in layers]
    (u64, l64), (u32, l32) = tables[torch.float64], tables[torch.float32]
    picks = X.picks(u64, l64, ancs, poss, cands, alpha)
    decided = H.mixgcf_pick_check(u64, l64, ancs, poss, cands, alpha, X.picks(u32, l32, ancs, poss, cands, alpha))
    assert decided > 0.9, decided

    def run(dtype, term=X.term, layers_of=lambda ls: ls):
        return H.bpr_term_oracle(model_key, case, hp, adj, dr, st, dtype,
                                 lambda u, i, ls: term(u, i, layers_of(ls), ancs, poss, picks, alpha), 'bpr_loss')

    ref = run(torch.float64)
    ok = H.path_errors(run(torch.float32), ref)
    assert max(ok.values()) <= 1.0, ok
    for what, kw in (('layers 1 .. L reversed', dict(layers_of=_reversed)), ('gradients one layer deeper', dict(layers_of=_one_layer_deeper)),
                     ('positive share detached', dict(term=_positive_detached_term))):
        bad = H.path_errors(run(torch.float32, **kw), ref)
        assert max(bad.values()) > 1.0, (what, bad)
