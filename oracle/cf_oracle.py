"""CPU oracle for the general_cf training hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product package
(``sslrec_b200``) never does: it fails loudly when the CUDA library is absent.

This is a functional restatement (torch CPU tensors, dtype-generic so the same code
runs in float32 -- the reference's arithmetic -- and in float64 for tolerance
budgeting) of the algorithm that HKUDS/SSLRec implements for its ``general_cf``
models.  Every function cites the reference file:line it follows (paths relative to
the reference checkout).  All stochastic inputs (edge masks, node masks, perturbation
noise, dropout masks, k-means seeds) are explicit arguments so that the oracle, the
reference and the CUDA path can be driven by the same bits.

Parity pinning: the reference ships no tests or golden vectors for this path
(SURVEY.md section 4), so the oracle is pinned against the reference itself:
``oracle/gen_golden.py`` imports the unmodified reference from ``$SSLREC_REFERENCE``,
runs it on injected inputs and writes ``tests/golden/*.npz``; ``tests/test_oracle_golden.py``
checks this module against those files.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# a1  adjacency  (data_utils/data_handler_general_cf.py:37-73)
# --------------------------------------------------------------------------------------

@dataclass
class Adj:
    """Normalised bipartite adjacency as COO triplets (no duplicates).

    ``rows``/``cols`` are int64 numpy arrays over the N=U+I node ids, ``vals`` float32.
    Entry order is row-major sorted (row, then col); the reference's own order is a
    scipy artefact (column-sorted) and does not change ``torch.spmm`` results on CPU
    (SURVEY.md section 4), ``coo_order_like_reference`` reproduces it when needed.
    """
    rows: np.ndarray
    cols: np.ndarray
    vals: np.ndarray
    n_user: int
    n_item: int

    @property
    def n(self) -> int:
        return self.n_user + self.n_item

    @property
    def nnz(self) -> int:
        return int(self.rows.shape[0])

    reference_layout: bool = False   # emit COO entries in the reference's (column-sorted) order
    csr_layout: bool = False         # "tuned CPU" variant of SURVEY.md 8(d): the one-line change adj.to_sparse_csr()

    def torch_coo(self, dtype=torch.float32, vals: Optional[torch.Tensor] = None,
                  keep: Optional[np.ndarray] = None) -> torch.Tensor:
        r, c = self.rows, self.cols
        v = torch.from_numpy(self.vals).to(dtype) if vals is None else vals
        if keep is not None:
            k = torch.from_numpy(np.asarray(keep, dtype=bool))
            r, c, v = r[keep], c[keep], v[k]
        if self.reference_layout:
            o = np.lexsort((r, c))
            r, c, v = r[o], c[o], v[torch.from_numpy(o)]
        idx = torch.from_numpy(np.vstack([r, c]).astype(np.int64))
        a = torch.sparse_coo_tensor(idx, v, (self.n, self.n), check_invariants=False)
        return a.coalesce().to_sparse_csr() if self.csr_layout else a

    def torch_csr(self, dtype=torch.float32) -> torch.Tensor:
        return self.torch_coo(dtype).coalesce().to_sparse_csr()


def normalized_adjacency(trn_rows: np.ndarray, trn_cols: np.ndarray, n_user: int, n_item: int) -> Adj:
    """A_hat = D^-1/2 [[0,R],[R^T,0]] D^-1/2 with deg = rowsum + 1e-10 in float64,
    values cast to float32 last.  data_handler_general_cf.py:37-51 (normalisation),
    :53-73 (bipartite stacking, ``!= 0`` binarisation, float32 cast at :71)."""
    trn_rows = np.asarray(trn_rows, dtype=np.int64)
    trn_cols = np.asarray(trn_cols, dtype=np.int64)
    pair = np.unique(trn_rows * n_item + trn_cols)          # binarise: duplicates collapse (:66)
    ur, ic = pair // n_item, pair % n_item
    n = n_user + n_item
    rows = np.concatenate([ur, ic + n_user])
    cols = np.concatenate([ic + n_user, ur])
    deg = np.bincount(rows, minlength=n).astype(np.float64) + 1e-10   # :47
    dinv = np.power(deg, -0.5)                                        # :48
    dinv[np.isinf(dinv)] = 0.0                                        # :49
    vals64 = dinv[cols] * dinv[rows]                                  # :51 (mat.D).T.D
    order = np.lexsort((cols, rows))
    return Adj(rows[order], cols[order], vals64[order].astype(np.float32), n_user, n_item)


def coo_order_like_reference(adj: Adj) -> np.ndarray:
    """Permutation p such that adj.rows[p], adj.cols[p] is the entry order the reference's
    ``_make_torch_adj`` produces (scipy ``(csc.T . D).tocoo()`` -> sorted by col, then row;
    data_handler_general_cf.py:51,69-72).  EdgeDrop masks index entries in that order
    (aug_utils.py:25-30)."""
    return np.lexsort((adj.rows, adj.cols))


# --------------------------------------------------------------------------------------
# a2  propagation,  a8-a10  augmentations
# --------------------------------------------------------------------------------------

def propagate(adj_t: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """Y = A_hat X.  models/general_cf/lightgcn.py:28-29 (``t.spmm``), hccf.py:35-36."""
    return torch.spmm(adj_t, x)


def edge_dropped(adj: Adj, keep_mask: Optional[np.ndarray], keep_rate: float, resize_val: bool,
                 dtype=torch.float32) -> torch.Tensor:
    """EdgeDrop (models/aug_utils.py:18-31): keep entries where mask is true; values divided
    by keep_rate only when ``resize_val`` (:29).  ``keep_mask`` is indexed in *this* Adj's
    entry order; None or keep_rate == 1.0 is the identity (:24)."""
    if keep_mask is None or keep_rate == 1.0:
        return adj.torch_coo(dtype)
    v = torch.from_numpy(adj.vals).to(dtype)
    if resize_val:
        v = v / keep_rate
    return adj.torch_coo(dtype, vals=v, keep=np.asarray(keep_mask, dtype=bool))


def keep_mask_from_uniform(u: torch.Tensor, keep_rate: float) -> torch.Tensor:
    """mask = floor(U[0,1) + keep_rate) as bool.  aug_utils.py:28 (edges), :49 (nodes)."""
    return (u + keep_rate).floor().to(torch.bool)


def node_dropped(embeds: torch.Tensor, node_keep: Optional[torch.Tensor]) -> torch.Tensor:
    """NodeDrop (models/aug_utils.py:40-50): zero whole rows of E0 (mask [N] of 0/1)."""
    if node_keep is None:
        return embeds
    return embeds * node_keep.to(embeds.dtype).view(-1, 1)


def perturbed(embeds: torch.Tensor, uniform: torch.Tensor, eps: float) -> torch.Tensor:
    """EmbedPerturb (models/aug_utils.py:125-132): X + eps * sign(X) * normalize(U, dim=1)."""
    noise = F.normalize(uniform.to(embeds.dtype), p=2, dim=1) * torch.sign(embeds) * eps
    return embeds + noise


# --------------------------------------------------------------------------------------
# a3-a7  per-model forward passes (embeddings)
# --------------------------------------------------------------------------------------

def lightgcn_embeds(adj_t: torch.Tensor, e0: torch.Tensor, layer_num: int) -> torch.Tensor:
    """E = sum_{k=0..L} A^k E0 (sum, not mean).  models/general_cf/lightgcn.py:31-43.
    ``adj_t`` is already edge-dropped by the caller (:36-37)."""
    xs = [e0]
    for _ in range(layer_num):
        xs.append(propagate(adj_t, xs[-1]))
    return sum(xs)


def simgcl_embeds(adj_t: torch.Tensor, e0: torch.Tensor, layer_num: int, eps: float,
                  uniforms: Optional[Sequence[torch.Tensor]]) -> torch.Tensor:
    """SimGCL.forward (models/general_cf/simgcl.py:20-30).  ``uniforms`` = one U[0,1)^{N x d}
    tensor per layer for the perturbed views; None -> clean LightGCN pass (:21-22)."""
    if uniforms is None:
        return lightgcn_embeds(adj_t, e0, layer_num)
    xs = [e0]
    for k in range(layer_num):
        xs.append(perturbed(propagate(adj_t, xs[-1]), uniforms[k], eps))   # :26-27
    return sum(xs)


def sgl_embeds(adj: Adj, e0: torch.Tensor, layer_num: int, augmentation: str, keep_rate: float,
               edge_keep: Optional[np.ndarray] = None, node_keep: Optional[torch.Tensor] = None) -> torch.Tensor:
    """SGL.forward (models/general_cf/sgl.py:20-36): node_drop zeroes rows of E0 (:24-25),
    edge_drop draws one mask per call (:27-28); the random_walk branch of the reference is
    unreachable code (NameError at :31) and is not restated."""
    x0 = e0
    adj_t = adj.torch_coo(e0.dtype)
    if augmentation == 'node_drop' and keep_rate != 1.0:
        x0 = node_dropped(e0, node_keep)
    if augmentation == 'edge_drop' and keep_rate != 1.0:
        adj_t = edge_dropped(adj, edge_keep, keep_rate, False, e0.dtype)
    return lightgcn_embeds(adj_t, x0, layer_num)


def ncl_embeds_list(adj_t: torch.Tensor, e0: torch.Tensor, layer_num: int, high_order: int):
    """NCL.forward (models/general_cf/ncl.py:30-42): max(L, 2*high_order) layers; returns the sum
    of the first L+1 layer outputs and the full list."""
    xs = [e0]
    for _ in range(max(layer_num, 2 * high_order)):
        xs.append(propagate(adj_t, xs[-1]))
    return sum(xs[:layer_num + 1]), xs


def leaky(x: torch.Tensor, slope: float) -> torch.Tensor:
    return F.leaky_relu(x, negative_slope=slope)


def hccf_embeds(adj: Adj, user_e: torch.Tensor, item_e: torch.Tensor, user_w: torch.Tensor, item_w: torch.Tensor,
                layer_num: int, keep_rate: float, mult: float, slope: float,
                edge_keeps: Optional[Sequence[np.ndarray]] = None,
                hyper_keeps: Optional[Sequence[Tuple[torch.Tensor, torch.Tensor]]] = None):
    """HCCF.forward + HGNNLayer (models/general_cf/hccf.py:38-54, :100-108).  Per layer: a fresh
    rescaled EdgeDrop (:33,47) and a fresh dropout (p = 1-keep, inverted scaling) of the hyper
    adjacency H = E_side W mult (:43-44, :48-49).  ``edge_keeps[k]`` / ``hyper_keeps[k]`` inject the
    Bernoulli draws (None -> no drop)."""
    n_user = user_e.shape[0]
    xs = [torch.cat([user_e, item_e], 0)]
    gcn_list, hyper_list = [], []
    uu = user_e @ user_w * mult
    ii = item_e @ item_w * mult
    for k in range(layer_num):
        ek = None if edge_keeps is None else edge_keeps[k]
        a_t = edge_dropped(adj, ek, keep_rate, True, user_e.dtype)
        gcn = propagate(a_t, xs[-1])
        if hyper_keeps is None or keep_rate == 1.0:
            hu, hi = uu, ii
        else:
            ku, ki = hyper_keeps[k]
            hu = uu * ku.to(uu.dtype) / keep_rate          # F.dropout(p=1-keep): kept / (1-p)
            hi = ii * ki.to(ii.dtype) / keep_rate
        xu, xi = xs[-1][:n_user], xs[-1][n_user:]
        hyp_u = leaky(hu @ leaky(hu.T @ xu, slope), slope)  # :105-107
        hyp_i = leaky(hi @ leaky(hi.T @ xi, slope), slope)
        hyp = torch.cat([hyp_u, hyp_i], 0)
        gcn_list.append(gcn)
        hyper_list.append(hyp)
        xs.append(gcn + hyp)
    return sum(xs), gcn_list, hyper_list


# --------------------------------------------------------------------------------------
# a12-a15  losses  (models/loss_utils.py)
# --------------------------------------------------------------------------------------

def bpr_loss_sum(anc: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor) -> torch.Tensor:
    """sum_b softplus(a.n - a.p).  loss_utils.py:7-10 (callers divide by B)."""
    return F.softplus((anc * neg).sum(-1) - (anc * pos).sum(-1)).sum()


def _unit(x: torch.Tensor) -> torch.Tensor:
    return x / torch.sqrt(1e-8 + x.square().sum(-1, keepdim=True))       # loss_utils.py:33-35


def infonce_loss_sum(e1: torch.Tensor, e2: torch.Tensor, all2: torch.Tensor, temp: float) -> torch.Tensor:
    """sum_b [ -(e1^.e2^)/temp + log sum_j exp(e1^.all^_j/temp) ], x^ = x / sqrt(1e-8 + |x|^2);
    no max-subtraction.  loss_utils.py:30-39."""
    n1, n2, na = _unit(e1), _unit(e2), _unit(all2)
    nume = -(n1 * n2 / temp).sum(-1)
    deno = torch.log(torch.exp(n1 @ na.T / temp).sum(-1))
    return (nume + deno).sum()


def infonce_spec_nodes_mean(e1: torch.Tensor, e2: torch.Tensor, nodes: torch.Tensor, temp: float) -> torch.Tensor:
    """-mean_n log( exp(x1_n.x2_n/temp) / (sum_j exp(x1_n.x2_j/temp) + 1e-8) ) with
    x = F.normalize(e + 1e-8).  loss_utils.py:42-51."""
    x1 = F.normalize(e1 + 1e-8, p=2)
    x2 = F.normalize(e2 + 1e-8, p=2)
    p1, p2 = x1[nodes], x2[nodes]
    nume = torch.exp((p1 * p2).sum(-1) / temp)
    deno = torch.exp(p1 @ x2.T / temp).sum(-1) + 1e-8
    return -torch.log(nume / deno).mean()


def reg_sumsq(params: Sequence[torch.Tensor]) -> torch.Tensor:
    """sum_W ||W||_2^2 over all parameters.  loss_utils.py:20-24."""
    tot = 0
    for w in params:
        tot = tot + w.norm(2).square()
    return tot


# --------------------------------------------------------------------------------------
# a16  cal_loss per model
# --------------------------------------------------------------------------------------

def _split(e: torch.Tensor, n_user: int):
    return e[:n_user], e[n_user:]


def lightgcn_loss(adj: Adj, user_e, item_e, batch, layer_num: int, reg_weight: float, keep_rate: float = 1.0,
                  edge_keep: Optional[np.ndarray] = None):
    """LightGCN.cal_loss (models/general_cf/lightgcn.py:45-56)."""
    ancs, poss, negs = batch
    a_t = edge_dropped(adj, edge_keep, keep_rate, False, user_e.dtype)
    e = lightgcn_embeds(a_t, torch.cat([user_e, item_e], 0), layer_num)
    ue, ie = _split(e, adj.n_user)
    bpr = bpr_loss_sum(ue[ancs], ie[poss], ie[negs]) / ancs.shape[0]
    reg = reg_weight * reg_sumsq([user_e, item_e])
    return bpr + reg, {'bpr_loss': bpr, 'reg_loss': reg}


def alignment(x: torch.Tensor, y: torch.Tensor, alpha: int = 2) -> torch.Tensor:
    """loss_utils.py:75-79."""
    x, y = F.normalize(x, dim=-1), F.normalize(y, dim=-1)
    return (x - y).norm(p=2, dim=1).pow(alpha).mean()


def uniformity(x: torch.Tensor) -> torch.Tensor:
    """loss_utils.py:82-86: log of the mean over the B(B-1)/2 row pairs of exp(-2 ||x^_i - x^_j||^2)."""
    x = F.normalize(x, dim=-1)
    return torch.pdist(x, p=2).pow(2).mul(-2).exp().mean().log()


def directau_loss(adj: Adj, user_e, item_e, batch, layer_num: int, gamma: float):
    """DirectAU.cal_loss (models/general_cf/directau.py:38-48); embeddings are the layer MEAN (:33)."""
    ancs, poss = batch[0], batch[1]
    e = lightgcn_embeds(adj.torch_coo(user_e.dtype), torch.cat([user_e, item_e], 0), layer_num) / (layer_num + 1)
    ue, ie = _split(e, adj.n_user)
    a, p = ue[ancs], ie[poss]
    align = alignment(a, p)
    uniform = gamma * (uniformity(a) + uniformity(p)) / 2
    return align + uniform, {'align_loss': align, 'uniform_loss': uniform}


def simgcl_loss(adj: Adj, user_e, item_e, batch, layer_num: int, reg_weight: float, cl_weight: float,
                temperature: float, eps: float, uniforms1, uniforms2):
    """SimGCL.cal_loss (models/general_cf/simgcl.py:39-55): two perturbed views + one clean view."""
    ancs, poss, negs = batch
    a_t = adj.torch_coo(user_e.dtype)
    e0 = torch.cat([user_e, item_e], 0)
    u1, i1 = _split(simgcl_embeds(a_t, e0, layer_num, eps, uniforms1), adj.n_user)
    u2, i2 = _split(simgcl_embeds(a_t, e0, layer_num, eps, uniforms2), adj.n_user)
    u3, i3 = _split(simgcl_embeds(a_t, e0, layer_num, eps, None), adj.n_user)
    bsz = ancs.shape[0]
    bpr = bpr_loss_sum(u3[ancs], i3[poss], i3[negs]) / bsz
    cl = infonce_loss_sum(u1[ancs], u2[ancs], u2, temperature) + infonce_loss_sum(i1[poss], i2[poss], i2, temperature)
    cl = cl / bsz
    reg = reg_weight * reg_sumsq([user_e, item_e])
    cl = cl * cl_weight
    return bpr + reg + cl, {'bpr_loss': bpr, 'reg_loss': reg, 'cl_loss': cl}


def sgl_loss(adj: Adj, user_e, item_e, batch, layer_num: int, reg_weight: float, cl_weight: float,
             temperature: float, augmentation: str, keep_rate: float,
             edge_keeps=(None, None), node_keeps=(None, None)):
    """SGL.cal_loss (models/general_cf/sgl.py:45-65): two augmented views + clean view; three
    InfoNCE terms (anchors, positives, negatives; :57-59)."""
    ancs, poss, negs = batch
    e0 = torch.cat([user_e, item_e], 0)
    u1, i1 = _split(sgl_embeds(adj, e0, layer_num, augmentation, keep_rate, edge_keeps[0], node_keeps[0]), adj.n_user)
    u2, i2 = _split(sgl_embeds(adj, e0, layer_num, augmentation, keep_rate, edge_keeps[1], node_keeps[1]), adj.n_user)
    u3, i3 = _split(sgl_embeds(adj, e0, layer_num, augmentation, 1.0), adj.n_user)
    bsz = ancs.shape[0]
    bpr = bpr_loss_sum(u3[ancs], i3[poss], i3[negs]) / bsz
    cl = (infonce_loss_sum(u1[ancs], u2[ancs], u2, temperature)
          + infonce_loss_sum(i1[poss], i2[poss], i2, temperature)
          + infonce_loss_sum(i1[negs], i2[negs], i2, temperature))
    cl = cl / bsz
    reg = reg_weight * reg_sumsq([user_e, item_e])
    cl = cl * cl_weight
    return bpr + reg + cl, {'bpr_loss': bpr, 'reg_loss': reg, 'cl_loss': cl}


def ncl_loss(adj: Adj, user_e, item_e, batch, layer_num: int, high_order: int, reg_weight: float,
             proto_weight: float, struct_weight: float, temperature: float,
             user_centroids, user2cluster, item_centroids, item2cluster):
    """NCL.cal_loss (models/general_cf/ncl.py:70-86) with the k-means state injected
    (:26-28 runs it on detached E0, so centroids are constants)."""
    ancs, poss, negs = batch
    nu = adj.n_user
    a_t = adj.torch_coo(user_e.dtype)
    e, xs = ncl_embeds_list(a_t, torch.cat([user_e, item_e], 0), layer_num, high_order)
    ego, ctx = xs[0], xs[2 * high_order]
    bsz = ancs.shape[0]
    struct = (infonce_loss_sum(ctx[:nu][ancs], ego[:nu][ancs], ego[:nu], temperature)
              + infonce_loss_sum(ctx[nu:][poss], ego[nu:][poss], ego[nu:], temperature)) / bsz       # :51-58
    proto = (infonce_loss_sum(ego[:nu][ancs], user_centroids[user2cluster[ancs]], user_centroids, temperature)
             + infonce_loss_sum(ego[nu:][poss], item_centroids[item2cluster[poss]], item_centroids, temperature)) / bsz  # :60-68
    struct = struct * struct_weight
    proto = proto * proto_weight
    bpr = bpr_loss_sum(e[:nu][ancs], e[nu:][poss], e[nu:][negs]) / bsz
    reg = reg_sumsq([user_e, item_e]) * reg_weight
    return bpr + struct + proto + reg, {'bpr_loss': bpr, 'reg_loss': reg, 'struct_loss': struct, 'proto_loss': proto}


def hccf_loss(adj: Adj, user_e, item_e, user_w, item_w, batch, layer_num: int, reg_weight: float, cl_weight: float,
              temperature: float, keep_rate: float, mult: float, slope: float, edge_keeps=None, hyper_keeps=None):
    """HCCF.cal_loss (models/general_cf/hccf.py:65-88): BPR = -mean log sigmoid(diff) (:73-74);
    per layer spec-node InfoNCE between the *detached* gcn output and the hyper output on the
    unique anchors / positives (:76-81)."""
    ancs, poss, negs = batch
    nu = adj.n_user
    e, gcn_list, hyper_list = hccf_embeds(adj, user_e, item_e, user_w, item_w, layer_num, keep_rate, mult, slope,
                                          edge_keeps, hyper_keeps)
    diff = (e[:nu][ancs] * e[nu:][poss]).sum(-1) - (e[:nu][ancs] * e[nu:][negs]).sum(-1)
    bpr = -diff.sigmoid().log().mean()
    cl = 0
    ua, up = torch.unique(ancs), torch.unique(poss)
    for k in range(layer_num):
        g, h = gcn_list[k].detach(), hyper_list[k]
        cl = cl + infonce_spec_nodes_mean(g[:nu], h[:nu], ua, temperature) + infonce_spec_nodes_mean(g[nu:], h[nu:], up, temperature)
    reg = reg_sumsq([user_e, item_e, user_w, item_w]) * reg_weight
    cl = cl * cl_weight
    return bpr + reg + cl, {'bpr_loss': bpr, 'reg_loss': reg, 'cl_loss': cl}


# --------------------------------------------------------------------------------------
# SURVEY 8(f) row 4  LightGCL (models/general_cf/lightgcl.py)
# --------------------------------------------------------------------------------------

def lightgcl_adjacency(trn_rows: np.ndarray, trn_cols: np.ndarray, n_user: int, n_item: int) -> Adj:
    """The U x I matrix R / sqrt(rowD colD) of lightgcl.py:16-20 (float32 arithmetic throughout: the pickle is
    cast to float32 at data_handler_general_cf.py:32) laid out as the symmetric bipartite Adj, so that one
    propagation step [Z_u; Z_i] = A [E_u; E_i] is both ``_spmm(adj, E_i)`` and ``_spmm(adj^T, E_u)`` (:75-76)."""
    pair = np.unique(np.asarray(trn_rows, dtype=np.int64) * n_item + np.asarray(trn_cols, dtype=np.int64))
    ur, ic = pair // n_item, pair % n_item
    row_d = np.bincount(ur, minlength=n_user).astype(np.float32)
    col_d = np.bincount(ic, minlength=n_item).astype(np.float32)
    v = (np.float32(1.0) / np.power(row_d[ur] * col_d[ic], np.float32(0.5))).astype(np.float32)
    rows = np.concatenate([ur, ic + n_user])
    cols = np.concatenate([ic + n_user, ur])
    vals = np.concatenate([v, v])
    order = np.lexsort((cols, rows))
    return Adj(rows[order], cols[order], vals[order], n_user, n_item)


def lightgcl_embeds(adj: Adj, user_e, item_e, layer_num: int, ut, vt, u_mul_s, v_mul_s, edge_keeps=None, dropout: float = 0.0):
    """LightGCL.forward (lightgcl.py:70-95): E^(l) = A_drop E^(l-1) (no residual, :86-87), G_u^(l) = (U S)(V^T E_i^(l-1)),
    G_i^(l) = (V S)(U^T E_u^(l-1)) (:79-83); returns the layer sums E_u, E_i, G_u, G_i (:90-93).
    ``edge_keeps[l]``: keep mask of the directed entries at layer l+1 (the reference draws one F.dropout per direction,
    :75-76), kept values are divided by 1 - dropout."""
    nu = adj.n_user
    dt = user_e.dtype
    e_u, e_i = [user_e], [item_e]
    g_u, g_i = [user_e], [item_e]
    for layer in range(1, layer_num + 1):
        keep = None if edge_keeps is None else edge_keeps[layer - 1]
        a_t = edge_dropped(adj, keep, 1.0 - dropout, True, dt) if keep is not None else adj.torch_coo(dt)
        z = torch.sparse.mm(a_t, torch.cat([e_u[-1], e_i[-1]], 0))
        g_u.append(u_mul_s.to(dt) @ (vt.to(dt) @ e_i[-1]))
        g_i.append(v_mul_s.to(dt) @ (ut.to(dt) @ e_u[-1]))
        e_u.append(z[:nu])
        e_i.append(z[nu:])
    return sum(e_u), sum(e_i), sum(g_u), sum(g_i)


def lightgcl_loss(adj: Adj, user_e, item_e, ws, batch, layer_num: int, reg_weight: float, cl_weight: float, temp: float,
                  ut, vt, u_mul_s, v_mul_s, edge_keeps=None, dropout: float = 0.0):
    """LightGCL.cal_loss (lightgcl.py:97-124).  ``ws``: the W_contrastive matrices, which only enter reg_params."""
    ancs, poss, negs = batch
    eu, ei, gu, gi = lightgcl_embeds(adj, user_e, item_e, layer_num, ut, vt, u_mul_s, v_mul_s, edge_keeps, dropout)
    a, p, n = eu[ancs], ei[poss], ei[negs]
    bpr = -((a * p).sum(-1) - (a * n).sum(-1)).sigmoid().log().mean()                                   # :104-106
    neg_score = torch.log(torch.exp(gu[ancs] @ eu.T / temp).sum(1) + 1e-8).mean()                       # :112
    neg_score = neg_score + torch.log(torch.exp(gi[poss] @ ei.T / temp).sum(1) + 1e-8).mean()           # :113
    pos_score = (torch.clamp((gu[ancs] * eu[ancs]).sum(1) / temp, -5.0, 5.0)).mean() \
        + (torch.clamp((gi[poss] * ei[poss]).sum(1) / temp, -5.0, 5.0)).mean()                          # :114-115
    cl = (-pos_score + neg_score) * cl_weight
    reg = reg_sumsq([user_e, item_e] + list(ws)) * reg_weight
    return bpr + cl + reg, {'bpr_loss': bpr, 'reg_loss': reg, 'cl_loss': cl}


# --------------------------------------------------------------------------------------
# a17  k-means (models/aug_utils.py:142-157)
# --------------------------------------------------------------------------------------

def kmeans(embeds: torch.Tensor, init_centroids: torch.Tensor, iters: int = 1000):
    """Lloyd iterations from the given initial centroids (the reference draws them from
    ``t.rand([K, d])`` at :147); empty clusters collapse towards 0 via the 1e-6 guard (:156)."""
    cents = init_centroids.clone()
    k = cents.shape[0]
    idx = None
    for _ in range(iters):
        d2 = (embeds.unsqueeze(1) - cents.unsqueeze(0)).square().sum(-1)
        idx = d2.argmin(1)
        new = torch.zeros_like(cents).index_add_(0, idx, embeds)
        cnt = torch.zeros(k, 1, dtype=embeds.dtype).index_add_(0, idx, torch.ones(embeds.shape[0], 1, dtype=embeds.dtype))
        cents = new / (cnt + 1e-6)
    return cents, idx, cnt


# --------------------------------------------------------------------------------------
# a18  prediction + masking + top-k  (lightgcn.py:58-66, base_model.py:35-36, metrics.py:108)
# --------------------------------------------------------------------------------------

def full_predict(user_e_final: torch.Tensor, item_e_final: torch.Tensor, users: torch.Tensor,
                 train_mask: torch.Tensor) -> torch.Tensor:
    """S = E_u[users] E_i^T ; S*(1-M) - 1e8*M."""
    s = user_e_final[users] @ item_e_final.T
    m = train_mask.to(s.dtype)
    return s * (1 - m) - 1e8 * m


def topk_items(preds: torch.Tensor, k: int) -> torch.Tensor:
    return torch.topk(preds, k=k).indices


# --------------------------------------------------------------------------------------
# a20  Adam  (trainer/trainer.py:45-49 -> torch.optim.Adam, weight_decay = 0 in every in-scope YAML)
# --------------------------------------------------------------------------------------

def adam_update(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int,
                lr: float, beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8, weight_decay: float = 0.0):
    """One torch.optim.Adam step (non-amsgrad, L2 weight decay folded into the gradient).
    Returns the new (p, m, v); ``step`` is 1-based."""
    if weight_decay != 0.0:
        g = g + weight_decay * p
    m = beta1 * m + (1 - beta1) * g
    v = beta2 * v + (1 - beta2) * g * g
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = v.sqrt() / math.sqrt(bc2) + eps
    p = p - (lr / bc1) * m / denom
    return p, m, v


# --------------------------------------------------------------------------------------
# a21  negative sampling (data_utils/datasets_general_cf.py:13-20) -- host side, integer
# --------------------------------------------------------------------------------------

def sample_negatives(trn_rows: np.ndarray, trn_cols: np.ndarray, n_item: int, rng: np.random.RandomState) -> np.ndarray:
    """For every positive (u, i): draw uniform items until one is not a training positive of u."""
    pos = set(zip(trn_rows.tolist(), trn_cols.tolist()))
    out = np.zeros(len(trn_rows), dtype=np.int32)
    for k, u in enumerate(trn_rows.tolist()):
        while True:
            j = int(rng.randint(n_item))
            if (u, j) not in pos:
                break
        out[k] = j
    return out


# --------------------------------------------------------------------------------------
# whole training steps on CPU (used by bench.py cpu_baseline / --impl reference)
# --------------------------------------------------------------------------------------

def xavier_uniform(rows: int, cols: int, gen: torch.Generator, dtype=torch.float32) -> torch.Tensor:
    """nn.init.xavier_uniform_ (lightgcn.py:21-22): U(-a, a), a = sqrt(6/(fan_in+fan_out))."""
    a = math.sqrt(6.0 / (rows + cols))
    return (torch.rand(rows, cols, generator=gen, dtype=dtype) * 2 - 1) * a


class CpuTrainer:
    """Drives ``zero_grad -> cal_loss -> loss.item() -> backward -> Adam.step`` exactly as
    trainer/trainer.py:63-68 does, on CPU tensors, for the model restatements above.  The
    adjacency layout is the reference's COO by default (``csr=True`` gives the "tuned CPU"
    variant of BASELINE.md section 2)."""

    def __init__(self, model: str, adj: Adj, dim: int, hp: Dict, seed: int = 2023, csr: bool = False):
        self.model, self.adj, self.hp = model, adj, dict(hp)
        g = torch.Generator().manual_seed(seed)
        self.user_e = xavier_uniform(adj.n_user, dim, g).requires_grad_(True)
        self.item_e = xavier_uniform(adj.n_item, dim, g).requires_grad_(True)
        self.params = [self.user_e, self.item_e]
        self.opt = torch.optim.Adam(self.params, lr=hp.get('lr', 1e-3), weight_decay=0)
        self.gen = g
        if csr:
            self.adj = Adj(adj.rows, adj.cols, adj.vals, adj.n_user, adj.n_item, csr_layout=True)

    def step(self, batch) -> float:
        hp, adj = self.hp, self.adj
        self.opt.zero_grad()
        if self.model == 'lightgcn':
            keep = hp.get('keep_rate', 1.0)
            ek = None if keep == 1.0 else keep_mask_from_uniform(torch.rand(adj.nnz, generator=self.gen), keep).numpy()
            loss, _ = lightgcn_loss(adj, self.user_e, self.item_e, batch, hp['layer_num'], hp['reg_weight'], keep, ek)
        elif self.model == 'simgcl':
            shp = (adj.n, self.user_e.shape[1])
            u1 = [torch.rand(shp, generator=self.gen) for _ in range(hp['layer_num'])]
            u2 = [torch.rand(shp, generator=self.gen) for _ in range(hp['layer_num'])]
            loss, _ = simgcl_loss(adj, self.user_e, self.item_e, batch, hp['layer_num'], hp['reg_weight'],
                                  hp['cl_weight'], hp['temperature'], hp['eps'], u1, u2)
        elif self.model == 'sgl':
            keep = hp['keep_rate']
            eks = [keep_mask_from_uniform(torch.rand(adj.nnz, generator=self.gen), keep).numpy() for _ in range(2)]
            loss, _ = sgl_loss(adj, self.user_e, self.item_e, batch, hp['layer_num'], hp['reg_weight'], hp['cl_weight'],
                               hp['temperature'], 'edge_drop', keep, edge_keeps=eks)
        elif self.model == 'directau':
            loss, _ = directau_loss(adj, self.user_e, self.item_e, batch, hp['layer_num'], hp['gamma'])
        else:
            raise ValueError(self.model)
        val = loss.item()
        loss.backward()
        self.opt.step()
        return val
