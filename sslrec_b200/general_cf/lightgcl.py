"""LightGCL -- drop-in for models/general_cf/lightgcl.py (SURVEY.md section 8f row 4).

The reference keeps a U x I matrix R / sqrt(rowD colD) and propagates users and items with two scatter
``_spmm`` calls per layer (lightgcl.py:59-66,75-76).  Stacked as the symmetric bipartite matrix that pair
is one launch of the sm_90a SpMM, [Z_u; Z_i] = A [E_u; E_i], with the dropout of the stored values
(``_sparse_dropout``, :68-72) evaluated in-kernel per layer and direction.  The low-rank branch
(U S)(V^T E), (V S)(U^T E) (:79-83) is two skinny library GEMMs per side; the contrastive term's
log sum_j exp(G[b] . E_j / temp) over ALL users / items (:112-113) runs on the tensor-core contraction without the
[B, N] logits (engine.dense_logsumexp_mean).  Layers are tied together by torch autograd, as in HCCF."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import torch
from torch import nn

from .. import engine as E
from ..base_model import BaseModel
from ..config import configs
from ..graph import GraphPlan
from ..loss_utils import cal_bpr_loss, reg_params

init = nn.init.xavier_uniform_


class W_contrastive(nn.Module):
    """lightgcl.py:140-146: part of the checkpoint and of reg_params; the reference never calls it in cal_loss."""

    def __init__(self, d):
        super().__init__()
        self.W = nn.Parameter(init(torch.empty(d, d)))

    def forward(self, x):
        return x @ self.W


class LightGCL(BaseModel):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        # lightgcl.py:16 re-reads the training pickle; a handler built from arrays has no file and hands over the matrix it holds
        train_mat = data_handler._load_one_mat(data_handler.trn_file) if getattr(data_handler, 'trn_file', None) else data_handler.trn_mat
        train_mat = sp.coo_matrix((train_mat != 0).astype(np.float32))
        train_mat.sum_duplicates()
        # lightgcl.py:16-20 in float32 (the pickle is cast at data_handler_general_cf.py:32): R / sqrt(rowD colD)
        row_d = np.asarray(train_mat.sum(1)).squeeze().astype(np.float32)
        col_d = np.asarray(train_mat.sum(0)).squeeze().astype(np.float32)
        r, c = train_mat.row.astype(np.int64), train_mat.col.astype(np.int64)
        vals = (np.float32(1.0) / np.power(row_d[r] * col_d[c], np.float32(0.5))).astype(np.float32)
        self._ui = (r, c, vals)

        self.temp = configs['model']['temp']
        self.dropout = configs['model']['dropout']
        self.layer_num = configs['model']['layer_num']
        self.cl_weight = configs['model']['cl_weight']
        self.reg_weight = configs['model']['reg_weight']
        self.svd_q = configs['model']['svd_q']

        self._alloc_embeddings()                                                                   # lightgcl.py:33-34
        self.Ws = nn.ModuleList([W_contrastive(self.embedding_size) for _ in range(self.layer_num)])
        self.E_u = self.E_i = self.G_u = self.G_i = None
        self.ut = self.vt = self.u_mul_s = self.v_mul_s = None       # SvdDecomposition output (aug_utils.py:89-98), built on first use
        self.is_training = True
        self._init_runtime(data_handler)
        self._bip_plan = None

    # ---- one-time device structures --------------------------------------------------------------
    def _bipartite_plan(self) -> GraphPlan:
        dev = self.user_embeds.device
        if self._bip_plan is None or self._bip_plan.device != dev:
            if dev.type != 'cuda':
                raise RuntimeError('sslrec_b200 models run on CUDA only (move the model with .to("cuda")); there is no CPU path')
            r, c, v = self._ui
            rows = np.concatenate([r, c + self.user_num])
            cols = np.concatenate([c + self.user_num, r])
            self._bip_plan = GraphPlan(rows, cols, np.concatenate([v, v]), self.user_num + self.item_num, dev, side_split=self.user_num)
        return self._bip_plan

    def _svd(self):
        if self.ut is None:
            dev = self.user_embeds.device
            r, c, v = self._ui
            idx = torch.from_numpy(np.vstack([r, c])).to(dev)
            adj = torch.sparse_coo_tensor(idx, torch.from_numpy(v).to(dev), (self.user_num, self.item_num)).coalesce()
            if E.deterministic():
                # torch's CUDA sparse products behind svd_lowrank sum in an order that varies from run to run; its host
                # operators do not.  Once per model, before the first step
                svd_u, s, svd_v = (t.to(dev) for t in torch.svd_lowrank(adj.cpu(), q=self.svd_q))
            else:
                svd_u, s, svd_v = torch.svd_lowrank(adj, q=self.svd_q)                             # aug_utils.py:94
            self.ut, self.vt = svd_u.T.contiguous(), svd_v.T.contiguous()
            self.u_mul_s, self.v_mul_s = svd_u @ torch.diag(s), svd_v @ torch.diag(s)
        return self.ut, self.vt, self.u_mul_s, self.v_mul_s

    _FACTORS = ('ut', 'vt', 'u_mul_s', 'v_mul_s')

    def resume_state(self) -> dict:
        """The seed stream and the low-rank factors: recomputing them would give other factors and take other draws from
        torch's generator (``svd_lowrank``), so a restored model keeps the saved ones and ``_svd`` does not run again."""
        state = super().resume_state()
        if self.ut is not None:
            state['svd'] = {k: getattr(self, k).detach().cpu() for k in self._FACTORS}
        return state

    def load_resume_state(self, state: dict) -> None:
        super().load_resume_state(state)
        svd = state.get('svd')
        dev = self.user_embeds.device
        for k in self._FACTORS:
            setattr(self, k, None if svd is None else svd[k].to(dev))

    # ---- forward -----------------------------------------------------------------------------------
    def forward(self, test=False):
        if test and self.E_u is not None:
            return self.E_u, self.E_i
        plan = self._bipartite_plan()
        ut, vt, u_mul_s, v_mul_s = self._svd()
        keep = 1.0 - self.dropout
        view = E.ViewSpec() if keep == 1.0 else E.ViewSpec(edge_mode=1, keep=keep, scale=1.0 / keep, per_layer_edges=True,
                                                           seed=self._seeds.next())
        nu = self.user_num
        e_list = [torch.concat([self.user_embeds, self.item_embeds], dim=0)]
        g_u, g_i = [self.user_embeds], [self.item_embeds]
        for layer in range(1, self.layer_num + 1):
            prev = e_list[-1]
            z = E.spmm(plan, prev, view, layer)                              # Z_u, Z_i of lightgcl.py:75-76 in one launch
            g_u.append(u_mul_s @ (vt @ prev[nu:]))                           # :79-80
            g_i.append(v_mul_s @ (ut @ prev[:nu]))                           # :81-82
            e_list.append(z)                                                 # :86-87 (no residual)
        e = sum(e_list)
        self._mix_tables = e_list if self.neg.mixgcf else None     # train.mixgcf mixes the item rows of every layer
        self.G_u, self.G_i = sum(g_u), sum(g_i)
        self.E_u, self.E_i = e[:nu], e[nu:]
        return self.E_u, self.E_i

    def cal_loss(self, batch_data):
        self.is_training = True
        user_embeds, item_embeds = self.forward()
        ancs, poss, negs = batch_data
        draw = self._dns_candidates(ancs, negs)
        # -log sigmoid(a.p - a.n).mean() == softplus(a.n - a.p).mean()  (lightgcl.py:101-106)
        layers = lambda: [t[self.user_num:] for t in self._mix_tables]
        bpr_loss = self._bpr_term(user_embeds, item_embeds, layers, ancs, poss, negs, draw, cal_bpr_loss)[0] / ancs.shape[0]
        at = E.rows_at          # table[ids]; under train.deterministic with an ordered backward
        g_u, g_i = at(self.G_u, ancs), at(self.G_i, poss)
        neg_score = E.dense_logsumexp_mean(g_u, user_embeds, self.temp, 1e-8) + E.dense_logsumexp_mean(g_i, item_embeds, self.temp, 1e-8)
        pos_score = torch.clamp((g_u * at(user_embeds, ancs)).sum(1) / self.temp, -5.0, 5.0).mean() \
            + torch.clamp((g_i * at(item_embeds, poss)).sum(1) / self.temp, -5.0, 5.0).mean()
        cl_loss = -pos_score + neg_score
        reg_loss = reg_params(self) * self.reg_weight
        cl_loss = self.cl_weight * cl_loss
        loss = bpr_loss + cl_loss + reg_loss
        losses = {self.bpr_loss_name: bpr_loss, 'reg_loss': reg_loss, 'cl_loss': cl_loss}
        return loss, losses

    def _eval_tables(self):
        user_embeds, item_embeds = self.forward(test=True)
        self.is_training = False
        return user_embeds.detach(), item_embeds.detach()

    def full_predict(self, batch_data):
        return self._predict(*self._eval_tables(), batch_data)

    def predict_topk(self, batch_data, k, return_values=False):
        """``topk(full_predict(batch_data), k, return_values)`` without the [Bt, I] score matrix (same ids and values)."""
        return self._predict_topk(*self._eval_tables(), batch_data, k, return_values)
