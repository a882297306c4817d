"""SGL -- drop-in for models/general_cf/sgl.py (edge_drop and node_drop; the reference's
random_walk branch is unreachable code, sgl.py:30-32, and raises here with a clear message)."""
from __future__ import annotations

from .. import engine as E
from ..aug_utils import NodeDrop
from ..config import configs
from ..loss_utils import cal_bpr_loss, cal_infonce_loss, reg_params
from .lightgcn import LightGCN


class SGL(LightGCN):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        self.augmentation = configs['model']['augmentation']
        self.cl_weight = configs['model']['cl_weight']
        self.temperature = configs['model']['temperature']
        self.node_dropper = NodeDrop()
        if self.augmentation not in ('edge_drop', 'node_drop'):
            raise NotImplementedError("SGL augmentation '%s': the reference implements edge_drop and node_drop only "
                                      "(its random_walk branch fails with a NameError, sgl.py:31)" % self.augmentation)

    def _aug_view(self, keep_rate, slot):
        if keep_rate == 1.0:
            return E.ViewSpec()
        if self.augmentation == 'node_drop':
            inj = None if self._inject is None else self._inject['node_masks'][slot]
            return self.node_dropper.view(keep_rate, self._seeds.next(), injected=inj)
        return self._edge_view(keep_rate, slot)

    def forward(self, adj, keep_rate):
        if not self.is_training and self.final_embeds is not None:
            return self.final_embeds[:self.user_num], self.final_embeds[self.user_num:]
        st = self._propagate([self._aug_view(keep_rate, 0)], n_layers=configs['model']['layer_num'], adj=adj)
        embeds = st.E.view(st.n, st.dim)
        self.final_embeds = embeds
        return embeds[:self.user_num], embeds[self.user_num:]

    def cal_loss(self, batch_data):
        self.is_training = True
        keep_rate = configs['model']['keep_rate']
        ancs, poss, negs = batch_data
        # views 0, 1: augmented (sgl.py:48-49); view 2: keep_rate 1.0 (sgl.py:50).  View 0 is read at the batch rows only (InfoNCE
        # anchors); view 2 becomes final_embeds and view 1 is the InfoNCE table, so both are computed at every row
        v0 = self._aug_view(keep_rate, 0)
        v0.row_bits = E.row_bitmap(self.user_num + self.item_num, self.user_embeds.device, (ancs, 0), (poss, self.user_num), (negs, self.user_num))
        st = self._propagate([v0, self._aug_view(keep_rate, 1), E.ViewSpec()], n_layers=configs['model']['layer_num'])
        self.final_embeds = st.E[:, 2, :]
        bsz = ancs.shape[0]
        bpr_loss = cal_bpr_loss(st.users(2), st.items(2), ancs, poss, negs) / bsz
        cl_loss = cal_infonce_loss(st.users(0), st.users(1), st.users(1), self.temperature, idx=ancs) + \
            cal_infonce_loss(st.items(0), st.items(1), st.items(1), self.temperature, idx=poss) + \
            cal_infonce_loss(st.items(0), st.items(1), st.items(1), self.temperature, idx=negs)
        cl_loss = cl_loss / bsz
        reg_loss = self.reg_weight * reg_params(self)
        cl_loss = cl_loss * self.cl_weight
        loss = bpr_loss + reg_loss + cl_loss
        losses = {'bpr_loss': bpr_loss, 'reg_loss': reg_loss, 'cl_loss': cl_loss}
        return loss, losses
