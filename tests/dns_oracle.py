"""TEST INFRASTRUCTURE -- restatements of dynamic negative sampling (optional key train.dns_candidates), which has no
counterpart in the reference: the candidate draw of ssl_neg_candidates in numpy on the Philox blocks of oracle/philox.py,
and the score-argmax selection of ssl_neg_select in float64."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.philox import philox4x32_10

TAG_DNSC = 0x444E5343          # "DNSC", the fourth counter word of every candidate block (csrc/hard_negs.cu)


def neg_candidates(users, negs, m: int, trn_rowptr, trn_cols, n_item: int, seed: int) -> np.ndarray:
    """[B, m] candidates on the draws of ssl_neg_candidates: column 0 is ``negs``; candidate j >= 1 of pair b is
    ``oracle.philox.sample_negs``'s rejection sampling (same multiply-shift, same 64-block cap keeping the last draw) on the
    blocks keyed (b, j, block, TAG_DNSC)."""
    users = np.asarray(users, dtype=np.int64)
    rowptr = np.asarray(trn_rowptr, dtype=np.int64)
    B = len(users)
    out = np.zeros((B, m), dtype=np.int64)
    out[:, 0] = np.asarray(negs, dtype=np.int64)
    pos = {(int(u), int(c)) for u in np.unique(users) for c in trn_cols[rowptr[u]:rowptr[u + 1]]}
    bb, jj = (a.ravel() for a in np.meshgrid(np.arange(B), np.arange(1, m), indexing='ij'))
    todo = np.arange(bb.size)                                  # candidates whose draws were all rejected so far
    for blk in range(64):
        if not todo.size:
            break
        words = philox4x32_10(bb[todo], jj[todo], blk, TAG_DNSC, seed)
        live = np.ones(todo.size, dtype=bool)
        for t in range(4):
            sel = np.flatnonzero(live)
            cand = ((words[t][sel].astype(np.uint64) * np.uint64(n_item)) >> np.uint64(32)).astype(np.int64)
            out[bb[todo[sel]], jj[todo[sel]]] = cand
            hit = np.fromiter(((int(u), int(c)) in pos for u, c in zip(users[bb[todo[sel]]], cand)), dtype=bool, count=sel.size)
            live[sel[~hit]] = False
        todo = todo[live]
    return out


def scores(user_e: torch.Tensor, item_e: torch.Tensor, ancs: torch.Tensor, cands: torch.Tensor) -> torch.Tensor:
    """The [B, M] float64 scores <E_u[ancs[b]], E_i[cands[b, j]]>."""
    return torch.einsum('bd,bmd->bm', user_e.double()[ancs], item_e.double()[cands])


def hard_negatives(user_e: torch.Tensor, item_e: torch.Tensor, ancs: torch.Tensor, cands: torch.Tensor) -> torch.Tensor:
    """The selected negatives in float64: per pair the candidate with the largest score, ties to the lowest j, NaN scores never
    chosen, candidate 0 when every score is NaN (for scores that are finite or NaN)."""
    s = scores(user_e, item_e, ancs, cands)
    s = torch.where(torch.isnan(s), torch.full_like(s, -math.inf), s)
    j = torch.argmax((s == s.max(1, keepdim=True).values).to(torch.int8), dim=1)      # the first j at the maximum
    return cands.gather(1, j[:, None]).squeeze(1)
