"""NCL -- drop-in for models/general_cf/ncl.py: one propagation of max(L, 2*high_order) layers, the
layer sum over the first L+1 outputs, structure-contrast between layer 0 and layer 2*high_order,
prototype-contrast against k-means centroids (constants), BPR."""
from __future__ import annotations

import torch

from .. import engine as E
from ..config import configs
from ..kmeans import KMeansClustering
from ..loss_utils import cal_bpr_loss, cal_infonce_loss, reg_params
from .lightgcn import LightGCN


class NCL(LightGCN):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        self.proto_weight = configs['model']['proto_weight']
        self.struct_weight = configs['model']['struct_weight']
        self.temperature = configs['model']['temperature']
        self.layer_num = configs['model']['layer_num']
        self.high_order = configs['model']['high_order']
        self.kmeans = KMeansClustering(cluster_num=configs['model']['cluster_num'],
                                       embedding_size=configs['model']['embedding_size'])

    def _cluster(self):
        self.user_centroids, self.user2cluster, _ = self.kmeans(self.user_embeds.detach())     # ncl.py:26-28
        self.item_centroids, self.item2cluster, _ = self.kmeans(self.item_embeds.detach())

    def graph_pre_step(self, recluster: bool) -> None:
        """Run by graphed.GraphedStep before every step, outside the captured region: the re-clustering that the eager
        ``cal_loss`` does when the batch's k-means flag is set (and on the first step).  The results are copied IN PLACE into
        the buffers of the first clustering, so a captured step keeps reading the current centroids and assignments."""
        if hasattr(self, 'user2cluster') and not recluster:
            return
        first = not hasattr(self, 'user2cluster')
        old = None if first else (self.user_centroids, self.user2cluster, self.item_centroids, self.item2cluster)
        self._cluster()
        if old is not None:
            new = (self.user_centroids, self.user2cluster, self.item_centroids, self.item2cluster)
            for dst, src in zip(old, new):
                dst.copy_(src)
            self.user_centroids, self.user2cluster, self.item_centroids, self.item2cluster = old

    def _run(self):
        ctx_layer = self.high_order * 2
        iteration = max(self.layer_num, ctx_layer)                                              # ncl.py:36
        return self._propagate([E.ViewSpec()], n_layers=iteration, sum_layers=self.layer_num, keep_layers=(ctx_layer,))

    def forward(self, adj):
        """-> (summed embeddings [N, d], state); ``state.all_nodes(0, k).dense()`` is layer k."""
        if not self.is_training and getattr(self, '_eval_state', None) is not None:
            st = self._eval_state
        else:
            st = self._run()
        self._eval_state = st
        return st.E.view(st.n, st.dim), st

    def cal_loss(self, batch_data):
        self.is_training = True
        ancs, poss, negs, kmeans_flags = batch_data
        # ncl.py:73-74; driven by a graphed.GraphedStep the flag is decided on the host and graph_pre_step clusters
        if not getattr(self, '_graph_mode', False) and (not hasattr(self, 'user2cluster') or bool(torch.sum(kmeans_flags) != 0)):
            self._cluster()
        embeds, st = self.forward(self.adj)
        ctx = self.high_order * 2
        bsz = ancs.shape[0]
        # structure loss (ncl.py:51-58): context (layer 2*high_order) vs ego (layer 0), all ego rows as negatives
        struct_loss = (cal_infonce_loss(st.users(0, ctx), st.users(0, 0), st.users(0, 0), self.temperature, idx=ancs)
                       + cal_infonce_loss(st.items(0, ctx), st.items(0, 0), st.items(0, 0), self.temperature, idx=poss)) / bsz
        # prototype loss (ncl.py:60-68): ego vs its cluster centroid, all centroids as negatives
        uc, ic = E.Rows.constant(self.user_centroids), E.Rows.constant(self.item_centroids)
        proto_loss = (cal_infonce_loss(st.users(0, 0), uc, uc, self.temperature, idx=ancs, idx2=self.user2cluster[ancs])
                      + cal_infonce_loss(st.items(0, 0), ic, ic, self.temperature, idx=poss, idx2=self.item2cluster[poss])) / bsz
        struct_loss = struct_loss * self.struct_weight
        proto_loss = proto_loss * self.proto_weight
        bpr_loss = cal_bpr_loss(st.users(0), st.items(0), ancs, poss, negs) / bsz
        reg_loss = reg_params(self) * self.reg_weight
        loss = bpr_loss + struct_loss + proto_loss + reg_loss
        losses = {'bpr_loss': bpr_loss, 'reg_loss': reg_loss, 'struct_loss': struct_loss, 'proto_loss': proto_loss}
        return loss, losses

    def _eval_tables(self):
        if configs.get('test', {}).get('exact_order', False):        # the evaluation embeddings are the sum of the first layer_num + 1 outputs (ncl.py:40-41)
            user_embeds, item_embeds = self._exact_forward()
        else:
            embeds, _ = self.forward(self.adj)
            user_embeds, item_embeds = embeds[:self.user_num], embeds[self.user_num:]
        self.is_training = False
        return user_embeds, item_embeds
