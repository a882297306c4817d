"""DirectAU -- drop-in for models/general_cf/directau.py (SURVEY.md section 8f row 4): LightGCN propagation with the
layer MEAN (:33) and the alignment / uniformity objective (:38-48).  Both losses normalise their rows, so the
training step reads the layer SUM the propagation kernel already writes (the 1 / (L + 1) cancels exactly) and the
mean is only formed for ``final_embeds`` / prediction."""
from __future__ import annotations

from .. import engine as E
from ..base_model import BaseModel
from ..config import configs
from ..loss_utils import alignment, uniformity


class DirectAU(BaseModel):
    bpr_negatives = False          # alignment / uniformity only: train.dns_candidates > 1 is refused

    def __init__(self, data_handler):
        super().__init__(data_handler)
        self.adj = data_handler.torch_adj
        self.layer_num = configs['model']['layer_num']
        self.gamma = configs['model']['gamma']
        self._alloc_embeddings()                                   # directau.py:19-20
        self.is_training = True
        self.final_embeds = None
        self._init_runtime(data_handler)

    def _propagate(self, adj=None) -> E.PropState:
        shard = self.comm is not None and self.comm.shard_propagation
        prop = E.Propagation(self._plan(adj), [E.ViewSpec()], self.layer_num, comm=self.comm if shard else None, loss_comm=None)
        st = E.propagate(prop, self.user_embeds, self.item_embeds, E.flat_table(self.user_embeds, self.item_embeds))
        self._state = st
        return st

    def forward(self, adj):
        if not self.is_training and self.final_embeds is not None:
            return self.final_embeds[:self.user_num], self.final_embeds[self.user_num:]
        st = self._propagate(adj)
        self.final_embeds = st.E.view(st.n, st.dim) / (self.layer_num + 1)          # directau.py:33
        return self.final_embeds[:self.user_num], self.final_embeds[self.user_num:]

    def cal_loss(self, batch_data):
        self.is_training = True
        ancs, poss, _ = batch_data
        st = self._propagate()
        self.final_embeds = st.E.view(st.n, st.dim) / (self.layer_num + 1)
        users, items = st.users(0), st.items(0)
        align_loss = alignment(users, items, ancs, poss)
        uniform_loss = self.gamma * (uniformity(users, ancs) + uniformity(items, poss)) / 2
        loss = align_loss + uniform_loss
        losses = {'align_loss': align_loss, 'uniform_loss': uniform_loss}
        return loss, losses

    def _eval_tables(self):
        user_embeds, item_embeds = self.forward(self.adj)
        self.is_training = False
        return user_embeds, item_embeds

    def full_predict(self, batch_data):
        return self._predict(*self._eval_tables(), batch_data)

    def predict_topk(self, batch_data, k, return_values=False):
        """``topk(full_predict(batch_data), k, return_values)`` without the [Bt, I] score matrix (same ids and values)."""
        return self._predict_topk(*self._eval_tables(), batch_data, k, return_values)
