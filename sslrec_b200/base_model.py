"""Plugin base class, mirror of models/base_model.py:6-47 (same constructor contract, same
``_mask_predict`` formula), plus the flat embedding table the kernels read without a concat."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
from torch import nn

from ._lib import check, lib
from .config import configs
from .graph import GraphPlan


class NegDraw(NamedTuple):
    """A step's candidates (``BaseModel._dns_candidates``): [B, M] int64, column 0 the loader's negatives; the seed they and
    MixGCF's weights were drawn with (None: no draw); the [B, M] logQ correction of the sampled softmax (None: uncorrected)."""
    cands: torch.Tensor
    seed: object
    bias: Optional[torch.Tensor]


class BaseModel(nn.Module):
    def __init__(self, data_handler):
        super().__init__()
        self.user_num = configs['data']['user_num']
        self.item_num = configs['data']['item_num']
        self.embedding_size = configs['model']['embedding_size']

    def forward(self):
        pass

    def cal_loss(self, batch_data):
        """-> (0-d loss tensor, dict of loss terms)   (base_model.py:23-33)"""
        pass

    def _mask_predict(self, full_preds, train_mask):
        return full_preds * (1 - train_mask) - 1e8 * train_mask          # base_model.py:35-36

    def full_predict(self, batch_data):
        pass

    # ---- flat table -------------------------------------------------------------------------
    def _alloc_embeddings(self):
        """``user_embeds`` / ``item_embeds`` (the checkpoint contract, SURVEY.md section 5) as adjacent
        views of ONE [N, d] storage, xavier-uniform per side in the reference's order
        (lightgcn.py:21-22) so the same torch seed gives the same initial weights."""
        # optional key model.init_on_device: draw the initial weights with the device generator (a 6 GB table -- BASELINE
        # config 4 -- takes tens of seconds and 6 GB of host memory per process on the CPU generator); same distribution,
        # different bits than the reference's CPU draw
        on_dev = configs['model'].get('init_on_device', False) and str(configs.get('device', 'cpu')).startswith('cuda')
        table = torch.empty(self.user_num + self.item_num, self.embedding_size, device=configs['device'] if on_dev else None)
        nn.init.xavier_uniform_(table[:self.user_num])
        nn.init.xavier_uniform_(table[self.user_num:])
        self.user_embeds = nn.Parameter(table[:self.user_num])
        self.item_embeds = nn.Parameter(table[self.user_num:])

    def _retie(self):
        u, i = self.user_embeds, self.item_embeds
        adjacent = (u.is_contiguous() and i.is_contiguous()
                    and u.untyped_storage().data_ptr() == i.untyped_storage().data_ptr()
                    and i.data_ptr() == u.data_ptr() + u.numel() * u.element_size())
        if not adjacent:
            table = torch.cat([u.data, i.data], 0)
            u.data = table[:self.user_num]
            i.data = table[self.user_num:]

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)        # .to(device) / .cuda() move the two views separately
        if hasattr(self, 'user_embeds') and hasattr(self, 'item_embeds'):
            self._retie()
        return out

    # ---- training checkpoint (Trainer.save_checkpoint / load_checkpoint) ---------------------------------
    def resume_state(self) -> dict:
        """What a resumed run needs besides ``state_dict()``: the position of the kernel seed stream.  Models with more
        non-parameter training state extend it.  Tensors are returned on the CPU."""
        return {'seeds': self._seeds.state_dict()}

    def load_resume_state(self, state: dict) -> None:
        self._seeds.load_state_dict(state['seeds'])

    # ---- runtime shared by the drop-in models ----------------------------------------------------
    def _init_runtime(self, data_handler):
        from . import engine as E
        self._trn_mat = getattr(data_handler, 'trn_mat', None)
        self._seeds = E.SeedStream(configs.get('train', {}).get('seed', 2023))
        self._plans = {}
        self._state = None
        self._inject = None        # tests: dict of injected masks / noise
        self.comm = None           # parallel.RowShard for row-sharded multi-GPU runs
        # optional: data_handler.plan_source(device, row_ranges, side_split) -> GraphPlan builds the CSR plan without a
        # torch sparse COO tensor (BASELINE config 4: 300 M stored entries are generated and sorted on the device)
        self._plan_source = getattr(data_handler, 'plan_source', None)
        # the negative-sampling keys (engine.NegSpec); the last step's outputs: ``dns_negs`` the selected negatives of
        # train.dns_candidates (like ``final_embeds``: last step only), ``mixgcf_picks`` / ``mixgcf_alpha`` ([B, L+1]) MixGCF's
        # picked items and mixing weights, ``_mix_seed`` the seed of the candidates and of MixGCF's weights
        self.neg = E.NegSpec.from_config()
        self.neg.check_model(self)
        self.dns_negs = self.mixgcf_picks = self.mixgcf_alpha = self._mix_seed = None
        self._mix_alpha_in = None      # tests: injected [B, L+1] mixing weights instead of the seeded draw
        self._pop = None               # engine.PopTables of train.neg_popularity, built once (``_pop_tables``)
        self._in_batch = None          # engine.InBatchWeights of train.ssm_in_batch, built once (``_in_batch_weights``)

    bpr_negatives = True           # the loss has a BPR term with sampled negatives (train.dns_candidates / mixgcf / ssm_temperature apply)
    # the keys of ``neg`` under their config names, read-only
    dns_candidates = property(lambda self: self.neg.candidates)
    mixgcf = property(lambda self: self.neg.mixgcf)
    ssm_temperature = property(lambda self: self.neg.ssm_temperature)
    neg_popularity = property(lambda self: self.neg.popularity)
    ssm_in_batch = property(lambda self: self.neg.in_batch)

    @property
    def bpr_loss_name(self) -> str:
        """The name ``cal_loss`` reports the BPR term under: 'ssm_loss' when train.ssm_temperature replaces it, else 'bpr_loss'."""
        return 'bpr_loss' if self.neg.ssm_temperature is None else 'ssm_loss'

    def _dns_candidates(self, ancs, negs) -> Optional[NegDraw]:
        """The batch's negative candidates as a ``NegDraw``, or None for the plain step (train.dns_candidates 1, neither
        train.mixgcf nor train.ssm_temperature).  Their seed, kept as ``_mix_seed``, is the last one the step draws, so a DNS
        step draws every seed of the plain step in the same order; MixGCF keys its mixing weights by the same seed, and with
        M = 1 its candidates are the loader's negatives (no draw).  The sampled softmax loss with M = 1 takes the loader's
        negatives without drawing a seed.  With train.neg_popularity the candidates come from the popularity draw on the same seed, and
        with the sampled softmax the draw also returns their logQ correction.  train.ssm_in_batch draws nothing: None."""
        from . import engine as E
        neg = self.neg
        if neg.candidates == 1 and not neg.mixgcf:
            if neg.ssm_temperature is None or neg.in_batch:
                return None
            seed = None
        else:
            seed = self._mix_seed = self._seeds.next()
        if neg.candidates == 1:
            cands, bias = E._i64(negs, ancs.device).view(-1, 1), None
        else:
            rowptr, cols = self._train_csr(ancs.device)
            pop = None if neg.popularity is None else self._pop_tables(ancs.device)
            want_bias = pop is not None and neg.ssm_temperature is not None
            out = E.neg_candidates(ancs, negs, neg.candidates, rowptr, cols, self.item_num, seed, pop=pop, want_bias=want_bias)
            cands, bias = out if want_bias else (out, None)
        return NegDraw(cands, seed, bias)

    def _pop_tables(self, device):
        """The alias table and logQ tables of train.neg_popularity (``engine.PopTables``) on ``device``, built once from the
        training CSR ``_train_csr`` uploads: a pure function of (training matrix, beta), so checkpoints do not store it."""
        from . import engine as E
        if self._pop is None or self._pop.table.device != device:
            import numpy as np
            import scipy.sparse as sp
            m = sp.csr_matrix(self._trn_mat)
            m.sort_indices()
            self._pop = E.PopTables(m.indptr.astype(np.int64), m.indices.astype(np.int64), self.item_num, self.neg.popularity, device)
        return self._pop

    def _in_batch_weights(self, device):
        """The column weights of train.ssm_in_batch (``engine.InBatchWeights``) on ``device``, built once from the training CSR:
        a pure function of the training matrix, so checkpoints do not store it."""
        from . import engine as E
        if self._in_batch is None or self._in_batch.v.device != device:
            import numpy as np
            import scipy.sparse as sp
            m = sp.csr_matrix(self._trn_mat)
            m.sort_indices()
            self._in_batch = E.InBatchWeights.of_matrix(m.indptr.astype(np.int64), m.indices.astype(np.int64), self.item_num, device)
        return self._in_batch

    def _bpr_term(self, users, items, item_layers, ancs, poss, negs, draw, bpr):
        """The batch's BPR sum and the negatives every other term of ``cal_loss`` reads: the plain term (``draw`` None); with DNS
        the term on the selected candidates of ``draw`` (which the other terms then read too); with MixGCF
        ``engine.mixgcf_bpr_sum`` and with train.ssm_temperature ``engine.ssm_loss_sum`` on them (the other terms keep the
        loader's negatives); with train.ssm_in_batch ``engine.ssm_in_batch_sum`` over the batch's own items.  ``users`` /
        ``items`` are the summed table as Rows or [n, d] tensors; ``item_layers()`` lists the item rows of its layers 0 .. L
        (called with MixGCF only).  ``bpr``: the ``cal_bpr_loss`` the plain and DNS terms call
        (a model passes its module's, so a restatement can stand in for it)."""
        from . import engine as E
        rows = isinstance(users, E.Rows)
        if self.neg.in_batch:          # no draw: every pair against the batch's positives and loader negatives
            return E.ssm_in_batch_sum(users, items, ancs, poss, negs, self.neg.ssm_temperature, self._in_batch_weights(ancs.device)), negs
        if draw is not None:
            if self.neg.mixgcf:
                loss, self.mixgcf_picks, self.mixgcf_alpha = E.mixgcf_bpr_sum(users, items, item_layers(), ancs, poss, draw.cands,
                                                                              draw.seed, self._mix_alpha_in)
                return loss, negs
            if self.neg.ssm_temperature is not None:
                logq = {} if draw.bias is None else dict(bias=draw.bias)      # uniform candidates: the uncorrected term
                return E.ssm_loss_sum(users, items, ancs, poss, draw.cands, self.neg.ssm_temperature, **logq), negs
            negs = self._dns_select(users if rows else users.detach(), items if rows else items.detach(), ancs, draw.cands)
        if rows:
            return bpr(users, items, ancs, poss, negs), negs
        at = E.rows_at          # table[ids]; under train.deterministic with an ordered backward
        return bpr(at(users, ancs), at(items, poss), at(items, negs)), negs

    def _dns_select(self, users, items, ancs, cands) -> torch.Tensor:
        """The highest-scored candidate of every pair on the rows the BPR term reads (``engine.hard_negatives``), kept as ``dns_negs``."""
        from . import engine as E
        self.dns_negs = E.hard_negatives(users, items, ancs, cands)
        return self.dns_negs

    def _plan(self, adj=None) -> GraphPlan:
        """CSR plan of an adjacency tensor, built once per (tensor, device)."""
        adj = self.adj if adj is None else adj
        dev = self.user_embeds.device
        sharded = self.comm is not None and self.comm.shard_propagation
        need_rev = self._inject is not None
        # keyed by the tensor's storage (an id() can be reused after the tensor is freed; the entry also holds a reference)
        key = (None if adj is None else (adj._values().data_ptr(), adj._nnz()), str(dev), sharded, need_rev)
        if key not in self._plans:
            if dev.type != 'cuda':
                raise RuntimeError('sslrec_b200 models run on CUDA only (move the model with .to("cuda")); there is no CPU path')
            if adj is None:
                if self._plan_source is None:
                    raise RuntimeError('the data handler provides neither torch_adj nor plan_source')
                plan = self._plan_source(dev, self.comm.ranges if sharded else None, self.user_num)
            elif sharded:
                plan = self.comm.make_plan(adj, dev, side_split=self.user_num)
            else:
                plan = GraphPlan.from_torch_adj(adj, dev, need_rev=need_rev, side_split=self.user_num)
            self._plans[key] = (plan, adj)
        return self._plans[key][0]

    def shard_to(self, comm) -> None:
        """Attach a parallel.RowShard.  When it row-shards the propagation, the flat [N, d] parameter table moves into a
        shared table (every rank maps every peer's replica) so the sharded Adam can store the rows it updates straight
        into the peers' replicas; rank 0's values are broadcast so all replicas start identical."""
        from . import engine as E
        if comm is not None and E.deterministic():
            raise RuntimeError('train.deterministic is single-GPU: a row-sharded model sums its partials across GPUs in an order of its own')
        if comm is not None:
            self.neg.refuse_multi_gpu(sharded=True)
        self.comm = comm
        self._plans.clear()
        if comm is None or not comm.shard_propagation:
            return
        dev = self.user_embeds.device
        tb = comm.table('params', (self.user_num + self.item_num, self.embedding_size), dev)
        with torch.no_grad():
            tb.t[:self.user_num].copy_(self.user_embeds.data)
            tb.t[self.user_num:].copy_(self.item_embeds.data)
            comm.dist.broadcast(tb.t, src=0)
        self.user_embeds.data = tb.t[:self.user_num]
        self.item_embeds.data = tb.t[self.user_num:]
        comm.barrier()
        # what the sharded optimizer needs per parameter: the owned row range and the peers' base addresses of that parameter
        row_bytes = 4 * self.embedding_size
        targets = [tb.mc_ptr] if tb.mc_ptr else list(tb.peer_ptrs)      # one multicast store (it also rewrites our copy with the same value) or one store per peer
        self.row_shards = {
            id(self.user_embeds): (comm.u0, comm.u1, targets, comm.user_bounds),
            id(self.item_embeds): (comm.i0 - self.user_num, comm.i1 - self.user_num, [p + self.user_num * row_bytes for p in targets], comm.item_bounds),
        }

    def _train_csr(self, device):
        """Training interactions as a device CSR (int32), built once: the mask of ``_mask_predict`` without the
        dense [Bt, I] float64 rows the reference ships per eval batch (datasets_general_cf.py:64-68)."""
        if getattr(self, '_trn_csr_dev', None) is None or self._trn_csr_dev[0].device != device:
            import numpy as np
            import scipy.sparse as sp
            m = sp.csr_matrix(self._trn_mat)
            m.sort_indices()
            self._trn_csr_dev = (torch.from_numpy(m.indptr.astype(np.int32)).to(device), torch.from_numpy(m.indices.astype(np.int32)).to(device))
        return self._trn_csr_dev

    def _predict(self, user_embeds, item_embeds, batch_data):
        """E_u[users] E_i^T with the training positives masked to -1e8 (lightgcn.py:61-65, base_model.py:35-36) in
        one kernel; no [Bt, I] temporaries besides the result.  ``train_mask``: the reference's dense [Bt, I] 0/1
        tensor, or None = no masking, or the string 'train' = mask the user's training items from the device CSR."""
        pck_users, mask, rowptr, cols = self._eval_batch(batch_data, user_embeds.device)
        n_b = pck_users.shape[0]
        preds = torch.empty(n_b, self.item_num, device=user_embeds.device, dtype=torch.float32)
        with torch.cuda.device(preds.device):
            check(lib.ssl_predict_mask(user_embeds.data_ptr(), user_embeds.stride(0), item_embeds.data_ptr(), item_embeds.stride(0),
                                       pck_users.data_ptr(), n_b, self.item_num, self.embedding_size,
                                       None if mask is None else mask.data_ptr(), None if rowptr is None else rowptr.data_ptr(),
                                       None if cols is None else cols.data_ptr(), preds.data_ptr(),
                                       torch.cuda.current_stream(preds.device).cuda_stream), 'ssl_predict_mask')
        return preds

    def _eval_batch(self, batch_data, device):
        """An evaluation batch -> (users int64, dense mask | None, CSR rowptr | None, CSR cols | None)."""
        # [users] alone (a lean AllRankTstData batch driven by the reference's Metric.eval, metrics.py:94-101) = mask from the device CSR
        pck_users, train_mask = (batch_data[0], 'train') if len(batch_data) == 1 else batch_data
        pck_users = pck_users.long().contiguous()
        mask, rowptr, cols = None, None, None
        if isinstance(train_mask, str):
            if train_mask != 'train' or getattr(self, '_trn_mat', None) is None:
                raise ValueError("train_mask must be a tensor, None or 'train' (needs data_handler.trn_mat)")
            rowptr, cols = self._train_csr(device)
        elif train_mask is not None:
            mask = train_mask.long().contiguous()
        return pck_users, mask, rowptr, cols

    def _predict_topk(self, user_embeds, item_embeds, batch_data, k, return_values=False):
        """``trainer.topk(self._predict(user_embeds, item_embeds, batch_data), k, return_values)`` -- the same ids and values bit for
        bit -- ranked on the device without the [Bt, I] score matrix: only the call's workspace and the [Bt, k] outputs are allocated."""
        dev = user_embeds.device
        pck_users, mask, rowptr, cols = self._eval_batch(batch_data, dev)
        n_b = pck_users.shape[0]
        ws_bytes = C.c_int64(0)
        check(lib.ssl_predict_topk_workspace(n_b, self.item_num, k, C.byref(ws_bytes)), 'ssl_predict_topk_workspace')
        ws = torch.empty(ws_bytes.value, device=dev, dtype=torch.uint8)
        idx = torch.empty(n_b, k, device=dev, dtype=torch.int64)
        val = torch.empty(n_b, k, device=dev, dtype=torch.float32) if return_values else None
        with torch.cuda.device(dev):
            check(lib.ssl_predict_topk(user_embeds.data_ptr(), user_embeds.stride(0), item_embeds.data_ptr(), item_embeds.stride(0),
                                       pck_users.data_ptr(), n_b, self.item_num, self.embedding_size,
                                       None if mask is None else mask.data_ptr(), None if rowptr is None else rowptr.data_ptr(),
                                       None if cols is None else cols.data_ptr(), k, ws.data_ptr(), ws_bytes.value, idx.data_ptr(),
                                       None if val is None else val.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), 'ssl_predict_topk')
        return (idx, val) if return_values else idx
