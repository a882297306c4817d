"""float64 oracle of the in-batch sampled softmax (train.ssm_in_batch; include/sslrec_b200.h, a28), written from its definition
with torch autograd: every pair against the 2B columns [poss; negs] with weights w_c = v[id_c] / B.  Also the smallest
temperature the engine accepts, and a float32 restatement of the kernels' flush-to-zero exponent terms."""
import math

import numpy as np
import torch

EPS = 1e-8
LOG2E = 1.4426950408889634


def _unit(x):
    return x / torch.sqrt(EPS + (x * x).sum(-1, keepdim=True))


def term64(users, items, ancs, poss, negs, tau, v, per_b=True, dedup=False, swap=False):
    """sum_b ln(sum_c w_c exp(s_bc)) - s_bb on the tables' dtype (autograd flows into ``users`` / ``items``); ``v`` [n_item]
    the weights, read at the columns and divided by B.  The keywords state wrong terms, for tests that must tell them apart:
    ``per_b`` False leaves w_c = v[id_c] undivided; ``dedup`` scores each distinct column once; ``swap`` orders the columns
    [negs; poss] and so reads the diagonal from the negatives."""
    ancs, poss, negs = (t.to(users.device).long() for t in (ancs, poss, negs))
    cols = torch.cat([negs, poss] if swap else [poss, negs])
    if dedup:
        cols = torch.unique(cols)
    B = ancs.numel()
    u, c = _unit(users[ancs]), _unit(items[cols])
    s = u @ c.T / tau                                                         # [B, n columns]
    w = torch.as_tensor(v, dtype=users.dtype, device=users.device)[cols] / (B if per_b else 1)
    lse = torch.logsumexp(s + torch.log(w)[None, :], 1)
    diag = (u * _unit(items[poss])).sum(1) / tau if dedup else s.diagonal()
    return (lse - diag).sum()


def abs_scale(users, items, ancs, poss, negs, tau, v):
    """float64 [n_user, d], [n_item, d]: per element the sum over the terms that add into it of |contribution| (the softmax
    weights P_bc over the columns, the diagonal's -u^/tau counted apart): the size the fp32 error of the gradient scales with."""
    with torch.no_grad():
        u64, i64 = users.double(), items.double()
        ancs, poss, negs = (t.to(users.device).long() for t in (ancs, poss, negs))
        cols = torch.cat([poss, negs])
        B = ancs.numel()
        ur, cr = u64[ancs], i64[cols]
        nu = torch.sqrt(EPS + (ur * ur).sum(1))
        nc = torch.sqrt(EPS + (cr * cr).sum(1))
        uh, ch = ur / nu[:, None], cr / nc[:, None]
        s = uh @ ch.T / tau
        w = torch.as_tensor(v, dtype=torch.float64, device=users.device)[cols] / B
        P = torch.softmax(s + torch.log(w)[None, :], 1)                       # [B, 2B]
        Pd = P.clone()
        Pd[torch.arange(B), torch.arange(B)] += 1
        gu = (Pd @ ch.abs() + (Pd * s.abs()).sum(1, keepdim=True) * uh.abs()) / (tau * nu[:, None])
        gc = (Pd.T @ uh.abs() + (Pd * s.abs()).sum(0)[:, None] * ch.abs()) / (tau * nc[:, None])
        A_u = torch.zeros_like(u64).index_add_(0, ancs, gu)
        A_i = torch.zeros_like(i64).index_add_(0, cols, gc)
    return A_u, A_i


def smallest_tau(B, vmin):
    """The smallest float tau that engine.ssm_in_batch_sum accepts for B pairs and smallest live weight ``vmin``: its next
    representable smaller neighbour is refused."""
    from sslrec_b200 import engine as E

    def ok(t):
        return E.in_batch_binades(B, t, vmin) <= E.IN_BATCH_MAX_BINADES

    t = 2.0 * LOG2E / (E.IN_BATCH_MAX_BINADES - max(0.0, math.log2(B / vmin)))
    while not ok(t):
        t = float(np.nextafter(t, np.inf))
    while ok(float(np.nextafter(t, 0.0))):
        t = float(np.nextafter(t, 0.0))
    return t


def ftz_ex2(x):
    """ex2.approx.ftz.f32 up to its approximation: 2^x in float32, 0 where that is below the smallest normal 2^-126."""
    y = np.exp2(np.asarray(x, dtype=np.float64)).astype(np.float32)
    return np.where(y < np.float32(2.0 ** -126), np.float32(0), y)


def rowsum32(cos, w, tau):
    """The forward's row sums as the kernels form them, from float64 cosines [B, n] and weights w [n]: the log2-scaled score
    S = fp32(log2(e) cos / tau) less the offset fp32(log2(e) / tau), one flush-to-zero ex2, then the weight:
    sum_c fp32(ftz_ex2(S - offset)) * w_c (summed in float64, so only the flush and the terms' own rounding remain)."""
    off = np.float32(LOG2E / tau)
    S = (LOG2E * np.asarray(cos, dtype=np.float64) / tau).astype(np.float32)
    E = ftz_ex2((S - off).astype(np.float32)) * np.asarray(w, dtype=np.float32)[None, :]
    return E.astype(np.float64).sum(1)


def underflow_batch(which, B=300, d=64, seed=0):
    """float32 tables, a batch and weights v log-uniform over [1, 4] whose forward underflows at tau = 0.02 (offset 72.1: an
    exponent term with cosine below -0.747 is under 2^-126).  'anti': B users near a direction e and 2B items near -e, every
    cosine <= -0.8, so every term of every row flushes.  'partial': every pair has user 0 (= e); the positive of pair 0 sits at
    cosine -0.5 and the other 2B - 1 columns at cosines in [-0.77, -0.755], so each row keeps one term of 2^-108 and loses
    2B - 1 terms of ~2^-127.  -> users [n_user, d], items [2B, d], ancs, poss, negs (int64 [B]), v float64 [2B]."""
    g = torch.Generator().manual_seed(seed)
    e = torch.nn.functional.normalize(torch.randn(d, generator=g, dtype=torch.float64), dim=0)
    if which == 'anti':
        users = e + 0.3 * torch.randn(B, d, generator=g, dtype=torch.float64) / math.sqrt(d)
        items = -e + 0.3 * torch.randn(2 * B, d, generator=g, dtype=torch.float64) / math.sqrt(d)
        ancs = torch.arange(B)
    else:
        q = torch.randn(2 * B, d, generator=g, dtype=torch.float64)
        q = torch.nn.functional.normalize(q - (q @ e)[:, None] * e[None, :], dim=1)          # unit rows orthogonal to e
        cos = -0.755 - 0.015 * torch.rand(2 * B, generator=g, dtype=torch.float64)
        cos[0] = -0.5
        items = cos[:, None] * e[None, :] + torch.sqrt(1 - cos * cos)[:, None] * q
        users, ancs = e[None, :].clone(), torch.zeros(B, dtype=torch.int64)
    poss, negs = torch.arange(B), torch.arange(B, 2 * B)
    v = torch.exp(torch.rand(2 * B, generator=g, dtype=torch.float64) * math.log(4.0)).numpy()
    return users.float(), items.float(), ancs, poss, negs, v


def cosines(users, items, ancs, poss, negs):
    """float64 [B, 2B] cosines of the batch's users against its columns [poss; negs]."""
    u = _unit(users[ancs].double())
    return (u @ _unit(items[torch.cat([poss, negs])].double()).T).numpy()


def rowsum64(cos, w, tau):
    """The same row sums in float64: sum_c w_c exp(s_bc - 1/tau)."""
    return (np.exp((np.asarray(cos, dtype=np.float64) - 1.0) / tau) * np.asarray(w, dtype=np.float64)[None, :]).sum(1)
