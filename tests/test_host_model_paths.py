"""The model-level path cases of tests/test_gpu_model_paths.py, checked on the host: the cases are what they claim to be
(split hub rows on both sides, isolated rows, a repeated and ragged batch), every kink is well posed, the float32 oracle
meets the GPU test's bounds against float64 (so they are achievable), and two slightly wrong float32 oracles do not (so
they are tight enough to catch a wrong operand): one with an entry of the item hub's row dropped, one with the
temperature scaled by 1 + 1e-3."""
import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
import ssl_test_helpers as H


def _drop_hub_entry(adj):
    """The adjacency with the first entry of the item hub's row set to 0 (positions, and so the injected masks, unchanged)."""
    row = adj.n_user + H.HUB_ITEM
    k = int(np.flatnonzero(adj.rows == row)[0])
    vals = adj.vals.copy()
    vals[k] = 0.0
    return O.Adj(adj.rows, adj.cols, vals, adj.n_user, adj.n_item)


@pytest.mark.parametrize('batch', [300, 100])
def test_path_case_shape(batch):
    case = H.path_case(48, batch)
    U, I = case['n_user'], case['n_item']
    assert len(set(zip(case['rows'].tolist(), case['cols'].tolist()))) == len(case['rows'])       # no duplicate edges
    du, di = np.bincount(case['rows'], minlength=U), np.bincount(case['cols'], minlength=I)
    assert 128 < du[H.HUB_USER] <= 200 and di[H.HUB_ITEM] >= 300          # split rows (> 128 entries) on both sides
    assert (du == 0).sum() >= 3 and (di == 0).sum() >= 3
    ancs, poss, negs = case['ancs'], case['poss'], case['negs']
    assert len(ancs) == batch and batch % 64 != 0
    assert len(np.unique(ancs)) < batch and (ancs == H.HUB_USER).sum() >= 3
    assert H.HUB_ITEM in poss and H.HUB_ITEM in negs and (di[negs] == 0).any()
    edges = set(zip(case['rows'].tolist(), case['cols'].tolist()))
    assert all((a, p) in edges for a, p in zip(ancs.tolist(), poss.tolist()))


@pytest.mark.parametrize('model_key,dim,tau,batch,hyper_num', H.PATH_CASES, ids=[H.path_case_id(c) for c in H.PATH_CASES])
def test_float32_oracle_meets_the_bounds_and_wrong_oracles_do_not(model_key, dim, tau, batch, hyper_num, monkeypatch):
    case, hp, adj, dr, st = H.path_setup(model_key, dim, tau, batch, hyper_num)
    margin = H.kink_margin(model_key, case, hp, adj, dr, st)
    assert margin > H.KINK_MARGIN, margin
    ref = H.path_oracle(model_key, case, hp, adj, dr, st, torch.float64)
    ok = H.path_errors(H.path_oracle(model_key, case, hp, adj, dr, st, torch.float32), ref)
    assert max(ok.values()) <= 1.0, ok

    wrong_adj = _drop_hub_entry(adj)
    if model_key == 'lightgcl':          # LightGCL builds its own adjacency inside the oracle
        lightgcl_adjacency = O.lightgcl_adjacency
        monkeypatch.setattr(O, 'lightgcl_adjacency', lambda *a: _drop_hub_entry(lightgcl_adjacency(*a)))
        wrong_adj = adj
    bad = H.path_errors(H.path_oracle(model_key, case, hp, wrong_adj, dr, st, torch.float32), ref)
    monkeypatch.undo()
    assert max(bad.values()) > 1.0, ('a dropped hub entry passes', bad)

    if tau is not None:
        key = 'temp' if model_key == 'lightgcl' else 'temperature'
        hp_bad = dict(hp, **{key: hp[key] * (1 + 1e-3)})
        bad = H.path_errors(H.path_oracle(model_key, case, hp_bad, adj, dr, st, torch.float32), ref)
        assert max(bad.values()) > 1.0, ('tau * (1 + 1e-3) passes', bad)
