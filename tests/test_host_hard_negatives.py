"""Dynamic negative sampling (train.dns_candidates) without a GPU: the numpy restatement of ssl_neg_candidates's draws
(tests/dns_oracle.neg_candidates) against a scalar restatement of the documented rule, its 64-block cap and the float64
selection of the oracle (the key itself: tests/test_host_neg_spec.py)."""
import numpy as np
import scipy.sparse as sp
import torch

import dns_oracle as D
from oracle import inputs
from oracle import philox as P


def _csr(rows, cols, n_user, n_item):
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    m.sum_duplicates()
    m.sort_indices()
    return m.indptr, m.indices


def _scalar_candidate(u, b, j, rowptr, cols, n_item, seed):
    """Candidate j >= 1 of pair b, one draw at a time: word t % 4 of block t // 4 keyed (b, j, block, TAG_DNSC), multiply-shift,
    rejected while a training positive of u; after 64 blocks the last draw is kept."""
    pos = set(cols[rowptr[u]:rowptr[u + 1]].tolist())
    for t in range(256):
        w = int(P.philox4x32_10(b, j, t // 4, D.TAG_DNSC, seed)[t % 4])
        c = (w * n_item) >> 32
        if c not in pos:
            return c
    return c


def test_candidate_oracle_matches_a_scalar_restatement():
    rows, cols = inputs.bipartite_edges(40, 30, 500, 3)
    rowptr, cidx = _csr(rows, cols, 40, 30)
    rs = np.random.RandomState(1)
    users, negs = rs.randint(0, 40, size=23), rs.randint(0, 30, size=23)
    seed = 0xDEADBEEF12345678
    got = D.neg_candidates(users, negs, 7, rowptr, cidx, 30, seed)
    assert got.shape == (23, 7) and np.array_equal(got[:, 0], negs)
    for b in range(23):
        for j in range(1, 7):
            assert got[b, j] == _scalar_candidate(users[b], b, j, rowptr, cidx, 30, seed), (b, j)
    assert not np.array_equal(got, D.neg_candidates(users, negs, 7, rowptr, cidx, 30, seed + 1))


def test_candidate_cap_and_a_user_with_one_free_item():
    n_item = 6
    # user 0 has every item (the draw is capped: the last of 256 draws), user 1 every item but 4
    rows = np.array([0] * n_item + [1] * (n_item - 1))
    cols = np.array(list(range(n_item)) + [0, 1, 2, 3, 5])
    rowptr, cidx = _csr(rows, cols, 2, n_item)
    got = D.neg_candidates([0, 1, 0, 1], [5, 4, 2, 4], 9, rowptr, cidx, n_item, 99)
    for b in (0, 2):
        for j in range(1, 9):
            last = int(P.philox4x32_10(b, j, 63, D.TAG_DNSC, 99)[3])
            assert got[b, j] == (last * n_item) >> 32
    assert (got[[1, 3], 1:] == 4).all()


def test_oracle_selection_ties_and_nan():
    u = torch.tensor([[1.0, 0.0]])
    items = torch.tensor([[0.5, 0.0], [2.0, 1.0], [2.0, -1.0], [float('nan'), 0.0], [-1.0, 0.0]])
    ancs = torch.tensor([0, 0, 0])
    cands = torch.tensor([[0, 1, 2], [3, 2, 1], [3, 3, 3]])
    assert D.hard_negatives(u, items, ancs, cands).tolist() == [1, 2, 3]       # tie to the lowest j; NaN skipped; all NaN -> j = 0
