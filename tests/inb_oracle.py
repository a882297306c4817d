"""float64 oracle of the in-batch sampled softmax (train.ssm_in_batch; include/sslrec_b200.h, a28), written from its definition
with torch autograd: every pair against the 2B columns [poss; negs] with weights w_c = v[id_c] / B."""
import torch

EPS = 1e-8


def _unit(x):
    return x / torch.sqrt(EPS + (x * x).sum(-1, keepdim=True))


def term64(users, items, ancs, poss, negs, tau, v):
    """sum_b ln(sum_c w_c exp(s_bc)) - s_bb on float64 tables (autograd flows into ``users`` / ``items``); ``v`` [n_item] the
    weights, read at the columns and divided by B."""
    ancs, poss, negs = (t.to(users.device).long() for t in (ancs, poss, negs))
    cols = torch.cat([poss, negs])
    B = ancs.numel()
    u, c = _unit(users[ancs]), _unit(items[cols])
    s = u @ c.T / tau                                                         # [B, 2B]
    w = torch.as_tensor(v, dtype=torch.float64, device=users.device)[cols] / B
    lse = torch.logsumexp(s + torch.log(w)[None, :], 1)
    return (lse - s.diagonal()).sum()


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
