"""TEST INFRASTRUCTURE -- restatements of the popularity-proportional candidates (optional key train.neg_popularity), which have
no counterpart in the reference: the alias-table draw of ssl_neg_candidates_pop in numpy on the Philox blocks of oracle/philox.py,
its fp32 logQ bias, the logQ-corrected sampled softmax forward (ssl_ssm_fwd_logq) as a sequential float32 restatement on top of
tests/ssm_oracle, and the distribution an alias table realises, in integers.  In float64 from the definition alone (no integer
weights, no alias table): the logQ bias (bias64) with its fp32 error bound, and the logQ-corrected term (term64_logq)."""
from __future__ import annotations

import math

import numpy as np
import torch

import ssm_oracle as S
from oracle.philox import philox4x32_10

TAG_DNSP = 0x444E5350          # "DNSP", the fourth counter word of every popularity candidate block (csrc/pop_negs.cuh)
K = 1 << 32


def column_shares(table: np.ndarray) -> np.ndarray:
    """int64 [n]: the 2^32-units share of every item over all columns of an alias table [n, 2] {thr, alias}: column c gives c its
    thr and alias[c] the rest, or c all 2^32 when alias[c] == c."""
    thr, alias = table[:, 0].astype(np.int64), table[:, 1].astype(np.int64)
    c = np.arange(len(table))
    own = np.where(alias == c, K, thr)
    out = np.zeros(len(table), np.int64)
    np.add.at(out, c, own)
    np.add.at(out, alias, np.where(alias == c, 0, K - thr))
    return out


def alias_item(table: np.ndarray, n_item: int, x, y) -> np.ndarray:
    """The item of draws (x, y) (uint32 arrays): column c = (x n_item) >> 32, c if alias[c] == c or y < thr[c], else alias[c]."""
    c = ((np.asarray(x, np.uint64) * np.uint64(n_item)) >> np.uint64(32)).astype(np.int64)
    thr, alias = table[c, 0].astype(np.uint32), table[c, 1].astype(np.int64)
    return np.where((alias == c) | (np.asarray(y, np.uint32) < thr), c, alias)


def neg_candidates(users, negs, m: int, rowptr, cols, n_item: int, table: np.ndarray, seed: int) -> np.ndarray:
    """[B, m] candidates on the draws of ssl_neg_candidates_pop: column 0 is ``negs``; candidate j >= 1 of pair b takes the
    draws (r.x, r.y), (r.z, r.w) of the blocks keyed (b, j, blk, TAG_DNSP), blk < 64, rejected while a training positive of
    users[b]; after 128 draws the last is kept."""
    users = np.asarray(users, dtype=np.int64)
    rowptr = np.asarray(rowptr, dtype=np.int64)
    B = len(users)
    out = np.zeros((B, m), dtype=np.int64)
    out[:, 0] = np.asarray(negs, dtype=np.int64)
    pos = {(int(u), int(c)) for u in np.unique(users) for c in cols[rowptr[u]:rowptr[u + 1]]}
    bb, jj = (a.ravel() for a in np.meshgrid(np.arange(B), np.arange(1, m), indexing='ij'))
    todo = np.arange(bb.size)
    for blk in range(64):
        if not todo.size:
            break
        r = philox4x32_10(bb[todo], jj[todo], blk, TAG_DNSP, seed)
        live = np.ones(todo.size, dtype=bool)
        for x, y in ((r[0], r[1]), (r[2], r[3])):
            sel = np.flatnonzero(live)
            cand = alias_item(table, n_item, x[sel], y[sel])
            out[bb[todo[sel]], jj[todo[sel]]] = cand
            hit = np.fromiter(((int(u), int(c)) in pos for u, c in zip(users[bb[todo[sel]]], cand)), dtype=bool, count=sel.size)
            live[sel[~hit]] = False
        todo = todo[live]
    return out


def bias(users, cands: np.ndarray, lp, lz_pop, lz_uni) -> np.ndarray:
    """[B, M] fp32: column 0 ln_m - lz_uni[u], column j (ln_m + lp[c_j]) - lz_pop[u], ln_m = fp32(log M), in that order."""
    f = np.float32
    users = np.asarray(users, np.int64)
    ln_m = f(math.log(cands.shape[1]))
    out = np.empty(cands.shape, f)
    out[:, 0] = ln_m - lz_uni[users]
    out[:, 1:] = (ln_m + lp[cands[:, 1:]]).astype(f) - lz_pop[users][:, None]
    return out


def _logq64(users, cands, rows, cols, n_user: int, n_item: int, beta: float, m: int):
    """float64 [B, m] ln q_j(c_j) of the draw's definition and the magnitude of the terms the fp32 bias is formed from."""
    users, cands = np.asarray(users, np.int64), np.asarray(cands, np.int64)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    assert cands.shape == (len(users), m), (cands.shape, len(users), m)
    assert len(np.unique(rows * n_item + cols)) == len(rows), 'the training pairs must be distinct'
    w = (np.bincount(cols, minlength=n_item).astype(np.float64) + 1.0) ** float(beta)          # w_i = (deg_i + 1)^beta
    W = math.fsum(w.tolist())
    left = np.full(n_user, W)                                                                   # W - sum_{i in P_u} w_i
    np.subtract.at(left, rows, w[cols])
    free = n_item - np.bincount(rows, minlength=n_user)                                         # n_item - deg_u
    assert (free[users] > 0).all(), 'a user with every item has no negative to draw'
    lq = np.empty(cands.shape, np.float64)
    mag = np.empty(cands.shape, np.float64)
    lq[:, 0] = -np.log(free[users])                                                             # column 0: the loader's uniform draw
    mag[:, 0] = np.log(free[users])
    lw, lz = np.log(w / W), np.log(left / W)
    lq[:, 1:] = lw[cands[:, 1:]] - lz[users][:, None]                                           # columns j >= 1: w_c / (W - sum_P w)
    mag[:, 1:] = np.abs(lw[cands[:, 1:]]) + np.abs(lz[users])[:, None]
    return lq, mag + math.log(m)


def bias64(users, cands, rows, cols, n_user: int, n_item: int, beta: float, m: int) -> np.ndarray:
    """float64 [B, m] logQ bias ln(M q_j(c_j)) straight from its definition, on the training pairs (rows, cols) (distinct):
    w_i = (deg_i + 1)^beta; column 0, the loader's uniform negative, q = 1 / (n_item - deg_u); column j >= 1, the popularity
    draw restricted to the non-positives of u, q = w_c / (W - sum_{i in P_u} w_i), W = sum_i w_i.  Shares nothing with
    engine.pop_tables (no integer weights, no alias table)."""
    lq, _ = _logq64(users, cands, rows, cols, n_user, n_item, beta, m)
    return math.log(m) + lq


def bias_tol(users, cands, rows, cols, n_user: int, n_item: int, beta: float, m: int) -> np.ndarray:
    """float64 [B, m]: the bound on |fp32 bias - bias64|, 2^-21 (ln M + |ln q_pop(c)| + |ln Z_u|) (column 0: ln M + ln(n_item -
    deg_u)).  The fp32 bias rounds ln M, lp, lz and two sums, each within 2^-24 of a value no larger than that sum; the table's
    integer weights V_i differ from n_item 2^32 w_i / W by less than one unit, a relative 2^-28 or less on the path graphs."""
    _, mag = _logq64(users, cands, rows, cols, n_user, n_item, beta, m)
    return 2.0 ** -21 * mag


def term64_logq(users, items, ancs, poss, cands, tau, bias_) -> torch.Tensor:
    """ssm_oracle.term64 with the candidate scores shifted by the logQ bias: sum_b lse(s_0, s_q - bias[q-1]) - s_0, in the
    dtype of the tables (``bias_`` [B, M] is cast to it)."""
    s = S.scores64(users, items, ancs, poss, cands, tau)
    sh = torch.cat([s[:, :1], s[:, 1:] - torch.as_tensor(bias_).to(s)], 1)
    return (torch.logsumexp(sh, 1) - s[:, 0]).sum()


def forward32_logq(u: np.ndarray, c: np.ndarray, tau: float, bias_: np.ndarray, expf=S.libm_expf, logf=S.libm_logf):
    """The logQ forward of csrc/ssm.cuh on gathered rows: u [B, d], c [B, M+1, d] (column 0 the positive), bias [B, M] float32 ->
    (loss_b [B], s [B, M+1] raw, w [B, M+1], nrm [B, M+2]): ssm_oracle.forward32 with the softmax on s^_q = s_q - bias[q-1]."""
    f = np.float32
    tau = f(tau)
    B, Q, d = c.shape
    G = S.group_lanes(d)
    nu = np.sqrt(f(S.EPS) + S._dot(u, u))
    nq = np.sqrt(f(S.EPS) + S._dot(c, c))
    dt = S._dot(u[:, None, :], c)
    s = (dt / ((nu[:, None] * nq) * tau)).astype(f)
    sh = s.copy()
    sh[:, 1:] = (s[:, 1:] - bias_).astype(f)
    m = np.fmax.reduce(sh, axis=1, initial=-np.inf).astype(f)
    ex = expf(sh - m[:, None])
    part = np.zeros((B, G), f)
    for q in range(Q):
        part[:, q % G] = part[:, q % G] + ex[:, q]
    Ssum = S._tree(part)
    loss = ((m + logf(Ssum)) - sh[:, 0]).astype(f)
    w = (ex / Ssum[:, None]).astype(f)
    w[:, 0] = w[:, 0] - f(1)
    return loss, s, w, np.concatenate([nu[:, None], nq], 1).astype(f)


def proposal(V: np.ndarray, positives) -> np.ndarray:
    """float64 [n]: the table's distribution V / sum V restricted to the items not in ``positives`` and renormalised."""
    p = V.astype(np.float64)
    p[np.asarray(list(positives), np.int64)] = 0.0
    return p / p.sum()
