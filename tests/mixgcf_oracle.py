"""TEST INFRASTRUCTURE -- restatements of MixGCF's BPR term (optional key train.mixgcf), which has no counterpart in the
reference: the mixing weights of ssl_mixgcf_bpr_fwd in numpy on the Philox blocks of oracle/philox.py, the per-layer picks in
float64, and the term with its gradients in float64 torch autograd."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.philox import philox4x32_10, u01

TAG_MIXA = 0x4D495841          # "MIXA", the fourth counter word of every alpha block (csrc/mixgcf.cuh)


def alpha(B: int, n_layers: int, seed: int) -> np.ndarray:
    """[B, n_layers] float32: alpha[b, l] = u01(word 0 of the Philox block keyed (b, l, 0, TAG_MIXA))."""
    bb, ll = (a.ravel() for a in np.meshgrid(np.arange(B), np.arange(n_layers), indexing='ij'))
    return u01(philox4x32_10(bb, ll, 0, TAG_MIXA, seed)[0]).reshape(B, n_layers)


def _mixed(layers, poss, cands, alpha_t):
    """[B, M, L+1, d] float64 mixes m_jl = alpha_l X_l[p] + (1 - alpha_l) X_l[c_j]."""
    a = alpha_t.double()[:, None, :, None]
    xp = torch.stack([x.double()[poss] for x in layers], 1)[:, None]                 # [B, 1, L+1, d]
    xc = torch.stack([x.double()[cands] for x in layers], 2)                         # [B, M, L+1, d]
    return a * xp + (1 - a) * xc


def picks(users, layers, ancs, poss, cands, alpha_t) -> torch.Tensor:
    """[B, L+1] picked items in float64: per layer the candidate whose mix scores highest against the user, ties to the lowest
    j, NaN scores never chosen, candidate 0 when every score is NaN."""
    s = torch.einsum('bd,bmld->bml', users.double()[ancs], _mixed(layers, poss, cands, alpha_t))
    s = torch.where(torch.isnan(s), torch.full_like(s, -math.inf), s)
    j = torch.argmax((s == s.max(1, keepdim=True).values).to(torch.int8), dim=1)     # [B, L+1], the first j at the maximum
    return cands.gather(1, j)


def term(users, items, layers, ancs, poss, pick_ids, alpha_t) -> torch.Tensor:
    """sum_b softplus(u . nhat - u . pbar), nhat = sum_l alpha_l X_l[p] + (1 - alpha_l) X_l[pick_l], on the given picks (no
    gradient through the choice).  Differentiable in users, items and every layer; computed in their dtype."""
    a = alpha_t.to(users.dtype)
    nhat = sum(a[:, l, None] * x[poss] + (1 - a[:, l, None]) * x[pick_ids[:, l]] for l, x in enumerate(layers))
    u = users[ancs]
    return F.softplus((u * nhat).sum(1) - (u * items[poss]).sum(1)).sum()
