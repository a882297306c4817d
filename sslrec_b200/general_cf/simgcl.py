"""SimGCL -- drop-in for models/general_cf/simgcl.py.  The two perturbed views and the clean view
are propagated together ([N, 3, d] interleaved; layer 1 is computed once and perturbed twice)."""
from __future__ import annotations

from .. import engine as E
from ..aug_utils import EmbedPerturb
from ..config import configs
from ..loss_utils import cal_bpr_loss, cal_infonce_loss, reg_params
from .lightgcn import LightGCN


class SimGCL(LightGCN):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        self.cl_weight = configs['model']['cl_weight']
        self.temperature = configs['model']['temperature']
        self.eps = configs['model']['eps']
        self.embed_perturb = EmbedPerturb(eps=self.eps)

    def _noise_view(self, slot):
        inj = None if self._inject is None else self._inject['noise_u'][slot]
        return self.embed_perturb.view(self._seeds.next(), injected=inj)

    def forward(self, adj, perturb=False):
        if not perturb:
            return super().forward(adj, 1.0)
        st = self._propagate([self._noise_view(0)], noise_eps=self.eps, adj=adj)      # simgcl.py:23-30
        embeds = st.E.view(st.n, st.dim)
        return embeds[:self.user_num], embeds[self.user_num:]

    def cal_loss(self, batch_data):
        self.is_training = True
        ancs, poss, negs = batch_data
        # views 0, 1: perturbed (simgcl.py:41-42); view 2: clean (simgcl.py:43).  Views 0 (InfoNCE anchors) and 2 (BPR) are
        # read at the batch rows only, so the last layer computes them there; view 1 is the InfoNCE table (every row)
        batch_rows = E.row_bitmap(self.user_num + self.item_num, self.user_embeds.device, (ancs, 0), (poss, self.user_num), (negs, self.user_num))
        v0, v2 = self._noise_view(0), E.ViewSpec()
        v0.row_bits = v2.row_bits = batch_rows
        st = self._propagate([v0, self._noise_view(1), v2], noise_eps=self.eps)
        bsz = ancs.shape[0]
        bpr_loss = cal_bpr_loss(st.users(2), st.items(2), ancs, poss, negs) / bsz
        cl_loss = cal_infonce_loss(st.users(0), st.users(1), st.users(1), self.temperature, idx=ancs) + \
            cal_infonce_loss(st.items(0), st.items(1), st.items(1), self.temperature, idx=poss)
        cl_loss = cl_loss / bsz
        reg_loss = self.reg_weight * reg_params(self)
        cl_loss = cl_loss * self.cl_weight
        loss = bpr_loss + reg_loss + cl_loss
        losses = {'bpr_loss': bpr_loss, 'reg_loss': reg_loss, 'cl_loss': cl_loss}
        return loss, losses

    def _eval_tables(self):
        user_embeds, item_embeds = self._eval_embeds(lambda: self.forward(self.adj, False))
        self.is_training = False
        return user_embeds, item_embeds
