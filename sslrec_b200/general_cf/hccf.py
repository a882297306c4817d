"""HCCF -- drop-in for models/general_cf/hccf.py.  The GCN half of every layer is the sm_90a SpMM
with a fresh, rescaled in-kernel edge mask (hccf.py:33,47); the two contrastive terms per layer and
side run through the fused InfoNCE kernels (loss_utils.py:42-51); the hyper-graph half
(E W, H^T X, H . : skinny [N_side, d] x [d, hyper_num] products with dropout and LeakyReLU, hccf.py:43-49,100-108)
and its backward run on the library's row-local / row-reducing kernels (csrc/hyper.cu: no cuBLAS, the dropout mask is
drawn in-kernel).  torch autograd only orders the nodes."""
from __future__ import annotations

import torch
from torch import nn

from .. import engine as E
from ..aug_utils import EdgeDrop
from ..base_model import BaseModel
from ..config import configs
from ..loss_utils import cal_bpr_loss, cal_infonce_loss_spec_nodes, reg_params

init = nn.init.xavier_uniform_


class HCCF(BaseModel):
    def __init__(self, data_handler):
        super().__init__(data_handler)
        model_config = configs['model']
        self.adj = data_handler.torch_adj
        self.layer_num = model_config['layer_num']
        self.reg_weight = model_config['reg_weight']
        self.cl_weight = model_config['cl_weight']
        self.hyper_num = model_config['hyper_num']
        self.mult = model_config['mult']
        self.keep_rate = model_config['keep_rate']
        self.temperature = model_config['temperature']

        self._alloc_embeddings()                                                            # hccf.py:27-28
        self.hgnn_layer = HGNNLayer(model_config['leaky'])
        self.user_hyper_embeds = nn.Parameter(init(torch.empty(self.embedding_size, self.hyper_num)))
        self.item_hyper_embeds = nn.Parameter(init(torch.empty(self.embedding_size, self.hyper_num)))
        self.edge_drop = EdgeDrop(resize_val=True)
        self._init_runtime(data_handler)

    # ---- pieces of one layer ---------------------------------------------------------------------
    def _gcn_layer(self, embeds, view, layer):
        return E.spmm(self._plan(), embeds, view, layer)

    def _hyper_drop(self, keep_rate, layer, side, seed) -> E.HyperDrop:
        """The dropout of one side's incidence at one layer (hccf.py:48-49): an in-kernel draw keyed by the step's seed and
        (layer, side), or the injected Bernoulli keeps of the parity tests."""
        if keep_rate == 1.0:
            return E.HyperDrop()
        mask = None
        if self._inject is not None and 'hyper_keeps' in self._inject:
            mask = self._inject['hyper_keeps'][layer][side]
        return E.HyperDrop(keep=float(keep_rate), seed=seed, stream=2 * layer + side, mask=mask)

    def forward(self, adj, keep_rate):
        """-> (sum over layers [N, d], per-layer SpMM outputs, per-layer hyper outputs)   (hccf.py:38-54)."""
        a_u = E.hyper_incidence(self.user_embeds, self.user_hyper_embeds, self.mult)          # H_user, H_item (:43-44)
        a_i = E.hyper_incidence(self.item_embeds, self.item_hyper_embeds, self.mult)
        inj = None if self._inject is None else self._inject.get('edge_masks_per_layer')
        view = self.edge_drop.view(keep_rate, self._seeds.next(), per_layer=True, injected=inj)   # a fresh rescaled mask per layer (:47)
        drop_seed = self._seeds.next()
        layers = [torch.concat([self.user_embeds, self.item_embeds], dim=0)]
        gcn_out, hyper_out = [], []
        for k in range(self.layer_num):
            gcn_out.append(self._gcn_layer(layers[-1], view, k + 1))
            hyper_out.append(E.hyper_layer(layers[-1], a_u, a_i, self.hgnn_layer.slope,                # :48-49
                                           self._hyper_drop(keep_rate, k, 0, drop_seed), self._hyper_drop(keep_rate, k, 1, drop_seed)))
            layers.append(gcn_out[-1] + hyper_out[-1])                                         # :52
        self._mix_tables = layers if self.neg.mixgcf else None     # train.mixgcf mixes the item rows of every layer
        return sum(layers), gcn_out, hyper_out

    def _contrast(self, gcn_out, hyper_out, ancs, poss):
        """sum over layers and sides of the spec-node InfoNCE between the DETACHED SpMM output and the hyper output on the
        batch's unique users / items (hccf.py:76-81).  Driven by a graphed.GraphedStep (``_graph_mode``), the de-duplication
        runs on the device and the term is bounded by the device count: no host sync, no data-dependent shape."""
        nu = self.user_num
        if getattr(self, '_graph_mode', False):
            picks = ((slice(0, nu), ancs), (slice(nu, None), poss))
            term = E.dense_infonce_spec_nodes_mean_dev
        else:
            picks = ((slice(0, nu), torch.unique(ancs)), (slice(nu, None), torch.unique(poss)))
            term = cal_infonce_loss_spec_nodes
        total = 0
        for g, h in zip(gcn_out, hyper_out):
            g = g.detach()
            for rows, nodes in picks:
                total = total + term(g[rows], h[rows], nodes, self.temperature)
        return total

    def cal_loss(self, batch_data):
        ancs, poss, negs = batch_data
        embeds, gcn_out, hyper_out = self.forward(self.adj, self.keep_rate)
        users, items = embeds[:self.user_num], embeds[self.user_num:]
        draw = self._dns_candidates(ancs, negs)
        # -log sigmoid(a.p - a.n).mean() == softplus(a.n - a.p).mean()  (hccf.py:70-74)
        layers = lambda: [t[self.user_num:] for t in self._mix_tables]
        bpr_loss = self._bpr_term(users, items, layers, ancs, poss, negs, draw, cal_bpr_loss)[0] / ancs.shape[0]
        terms = {self.bpr_loss_name: bpr_loss,
                 'reg_loss': reg_params(self) * self.reg_weight,
                 'cl_loss': self._contrast(gcn_out, hyper_out, ancs, poss) * self.cl_weight}
        return bpr_loss + terms['reg_loss'] + terms['cl_loss'], terms

    def _eval_tables(self):
        embeds, _, _ = self.forward(self.adj, 1.0)
        return embeds[:self.user_num], embeds[self.user_num:]

    def full_predict(self, batch_data):
        return self._predict(*self._eval_tables(), batch_data)

    def predict_topk(self, batch_data, k, return_values=False):
        """``topk(full_predict(batch_data), k, return_values)`` without the [Bt, I] score matrix (same ids and values)."""
        return self._predict_topk(*self._eval_tables(), batch_data, k, return_values)


class HGNNLayer(nn.Module):
    """hccf.py:100-108: act(adj @ act(adj.T @ embeds)); the drop-in model calls engine.hyper_layer for both sides at once; this
    module keeps the activation's slope and serves stand-alone callers through the same kernels (one side)."""

    def __init__(self, leaky):
        super().__init__()
        self.slope = float(leaky)
        self.act = nn.LeakyReLU(negative_slope=leaky)

    def forward(self, adj, embeds):
        # one side only: the second side of engine.hyper_layer is empty
        return E.hyper_layer(embeds, adj, adj.new_zeros((0, adj.shape[1])), self.slope, E.HyperDrop(), E.HyperDrop())
