"""LightGCN -- drop-in for models/general_cf/lightgcn.py (class name, ctor, forward, cal_loss,
full_predict, ``is_training`` / ``final_embeds`` cache semantics are the reference's)."""
from __future__ import annotations

import torch

from .. import engine as E
from ..aug_utils import EdgeDrop
from ..base_model import BaseModel
from ..config import configs
from ..loss_utils import cal_bpr_loss, reg_params


class LightGCN(BaseModel):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        self.adj = data_handler.torch_adj
        self.layer_num = configs['model']['layer_num']
        self.reg_weight = configs['model']['reg_weight']
        self.keep_rate = configs['model']['keep_rate']

        self._alloc_embeddings()                      # user_embeds, item_embeds  (lightgcn.py:21-22)

        self.edge_dropper = EdgeDrop()
        self.is_training = True
        self.final_embeds = None

        self._init_runtime(data_handler)

    def _table(self) -> torch.Tensor:
        return E.flat_table(self.user_embeds, self.item_embeds)

    def _propagate(self, views, n_layers=None, sum_layers=None, keep_layers=(), noise_eps=0.0, adj=None) -> E.PropState:
        """All augmented views, all layers and the layer sum: replaces the loop of t.spmm calls
        (lightgcn.py:28-29,38-41)."""
        shard = self.comm is not None and self.comm.shard_propagation
        prop = E.Propagation(self._plan(adj), views, self.layer_num if n_layers is None else n_layers,
                             sum_layers, keep_layers, noise_eps, comm=self.comm if shard else None, loss_comm=self.comm)
        st = E.propagate(prop, self.user_embeds, self.item_embeds, self._table())
        self._state = st
        return st

    def _edge_view(self, keep_rate, slot=0):
        inj = None if self._inject is None else self._inject.get('edge_masks', [None] * 4)[slot]
        return self.edge_dropper.view(keep_rate, self._seeds.next(), injected=inj)

    def forward(self, adj, keep_rate):
        if not self.is_training and self.final_embeds is not None:
            return self.final_embeds[:self.user_num], self.final_embeds[self.user_num:]
        view = self._edge_view(keep_rate) if self.is_training else E.ViewSpec()
        st = self._propagate([view], adj=adj)
        embeds = st.E.view(st.n, st.dim)
        self.final_embeds = embeds
        return embeds[:self.user_num], embeds[self.user_num:]

    def cal_loss(self, batch_data):
        self.is_training = True
        ancs, poss, negs = batch_data
        st = self._propagate([self._edge_view(self.keep_rate)])
        self.final_embeds = st.E.view(st.n, st.dim)
        bpr_loss = cal_bpr_loss(st.users(0), st.items(0), ancs, poss, negs) / ancs.shape[0]
        reg_loss = self.reg_weight * reg_params(self)
        loss = bpr_loss + reg_loss
        losses = {'bpr_loss': bpr_loss, 'reg_loss': reg_loss}
        return loss, losses

    def _exact_forward(self):
        """Optional key ``test.exact_order: true``: the evaluation forward pass in the arithmetic order of the reference's CPU run -- each layer
        by ``engine.spmm_exact`` (the row's entries in one sequential FMA chain, as ``t.spmm`` on the reference's adjacency), the layer sum as
        Python's ``sum(embeds_list)`` forms it, ((E0 + X1) + X2) + ... (lightgcn.py:38-42).  With ``ssl_predict_mask``'s sequential score chains
        ``full_predict`` then equals the reference's CPU ``full_predict`` bit for bit on the same parameters.  Same cache rule as ``forward``."""
        if not self.is_training and getattr(self, '_exact_embeds', None) is not None:
            embeds = self._exact_embeds
        else:
            if self.comm is not None and self.comm.shard_propagation:
                raise RuntimeError('test.exact_order is a single-GPU evaluation mode')
            with torch.no_grad():
                plan = self._plan()
                x = self._table().contiguous()
                embeds = x.clone()
                for _ in range(self.layer_num):
                    x = E.spmm_exact(plan, x)
                    embeds = embeds + x
            self._exact_embeds = self.final_embeds = embeds
        return embeds[:self.user_num], embeds[self.user_num:]

    def _eval_embeds(self, forward):
        """The embeddings ``full_predict`` scores with: the regular forward pass, or the exact-order one (``test.exact_order``)."""
        if configs.get('test', {}).get('exact_order', False):
            return self._exact_forward()
        return forward()

    def _eval_tables(self):
        """The (user, item) tables evaluation scores with, with full_predict's side effects (``is_training``, the cache)."""
        user_embeds, item_embeds = self._eval_embeds(lambda: self.forward(self.adj, 1.0))
        self.is_training = False
        return user_embeds, item_embeds

    def full_predict(self, batch_data):
        return self._predict(*self._eval_tables(), batch_data)

    def predict_topk(self, batch_data, k, return_values=False):
        """``topk(full_predict(batch_data), k, return_values)`` without the [Bt, I] score matrix (same ids and values)."""
        return self._predict_topk(*self._eval_tables(), batch_data, k, return_values)
