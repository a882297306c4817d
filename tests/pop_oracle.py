"""TEST INFRASTRUCTURE -- restatements of the popularity-proportional candidates (optional key train.neg_popularity), which have
no counterpart in the reference: the alias-table draw of ssl_neg_candidates_pop in numpy on the Philox blocks of oracle/philox.py,
its fp32 logQ bias, the logQ-corrected sampled softmax forward (ssl_ssm_fwd_logq) as a sequential float32 restatement on top of
tests/ssm_oracle, and the distribution an alias table realises, in integers."""
from __future__ import annotations

import math

import numpy as np

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
