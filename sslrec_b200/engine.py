"""Host-side orchestration of the sm_90a kernels: multi-view K-layer propagation (forward and
the transposed backward), and the autograd plumbing that lets ``cal_loss`` read like the
reference's while every gradient is accumulated in place by the kernels.

Gradient plumbing ("sinks").  ``propagate()`` returns a :class:`PropState` holding the
interleaved embeddings ``E [N, V, d]`` (not autograd tensors) and a 0-d ``token`` that *is* an
autograd output of the propagation node.  Loss functions take row references into a state
(:class:`Rows`), depend on its token, and in their backward add their gradient rows straight into
the state's sink buffers (``G_sum``, ``G_layer[k]``, ``G_e0``) with the kernels' atomics; they
hand autograd only a zero for the token.  Autograd's ordering then guarantees the propagation
node's backward runs after every loss wrote its rows; it walks the layers with the transposed
SpMM (same CSR, mask key swapped) and returns d user_embeds / d item_embeds.  No [N, V, d]
gradient is ever materialised per loss term or added by torch.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import functools
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import PropArgs, check, lib
from .graph import GraphPlan

LOG2E = 1.4426950408889634
# InfoNCE contraction on the wgmma tensor cores (3xFP16 or 3xTF32, fp32-grade accuracy) when the dim allows; set to False
# to force the FP32-FMA kernel (tests compare the two)
USE_TENSOR_CORES = True
# ssl_softmax_gemm_f16x3 accepts unit rows scaled by |alpha| <= 16 and offsets in [0, 16] (csrc/f16x3.cuh): every InfoNCE
# temperature >= 0.0902 and the uniformity term.  Raw rows (LightGCL) and larger offsets keep the 3xTF32 kernel.
F16X3_MAX_OFFSET = 16.0
# a forward with column weights (ssm_in_batch_sum) keeps 3xFP16 only while no E' can fall below the flush threshold: up to this
# offset plus half the binades of its weights' range (csrc/f16x3.cuh's kF16NoFlushOffset; include/sslrec_b200.h, a28)
F16X3_NO_FLUSH_OFFSET = 13.5
LIVE_ROWS, LIVE_COLS = 1, 2     # SSL_LIVE_ROWS / SSL_LIVE_COLS: which operand of a *_live contraction the device count bounds
NUM_SM = 132          # H100 SXM; grids of the contraction are sized in resident-CTA slots (kNumSM in csrc/common.cuh)


def f16x3_applies(offset: float) -> bool:
    """True when the 3xFP16 contraction's operand bound holds for a term with this offset (rows normalised by the engine)."""
    return 0.0 <= offset <= F16X3_MAX_OFFSET


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f'sslrec_b200: {what} must live on a CUDA device (got {t.device}); there is no CPU path')
    if t.dtype != torch.float32:
        raise RuntimeError(f'sslrec_b200: {what} must be float32')


def ceil_to(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class KernelTimer:
    """Optional CUDA-event brackets around the dominant kernels (bench.py's roofline numbers are
    measured live with these, on the launching stream).  Off unless ``engine.TIMER`` is set."""

    def __init__(self):
        self.records = []          # (name, meta, start_event, end_event)

    def launches(self):
        """[(name, meta, milliseconds)] -- call after a device synchronize."""
        return [(name, meta, a.elapsed_time(b)) for name, meta, a, b in self.records]

    def summary(self):
        out = {}
        for name, meta, ms in self.launches():
            e = out.setdefault(name, dict(ms=0.0, launches=0, meta=meta))
            e['ms'] += ms
            e['launches'] += 1
        return out


TIMER: Optional[KernelTimer] = None


class _timed:
    def __init__(self, name, meta=None):
        self.name, self.meta = name, meta

    def __enter__(self):
        if TIMER is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.a.record()

    def __exit__(self, *exc):
        if TIMER is not None:
            b = torch.cuda.Event(enable_timing=True)
            b.record()
            TIMER.records.append((self.name, self.meta, self.a, b))
        return False


# ------------------------------------------------------------------------------------------------
# view specifications
# ------------------------------------------------------------------------------------------------

@dataclass
class ViewSpec:
    """One augmented view of the propagation (mirrors the reference augmentors).

    edge_mode   0 none | 1 in-kernel RNG keep test | 2 injected CSR-order uint8 mask(s)
    edge_masks  mode 2: one tensor (same mask for every layer: lightgcn.py:36-37, sgl.py:27-28) or a
                list with one tensor per layer (hccf.py:47)
    per_layer_edges  mode 1: redraw the mask at every layer (HCCF) instead of once per forward
    scale       multiplier of kept values (1/keep for EdgeDrop(resize_val=True))
    noise_mode  0 none | 1 in-kernel RNG | 2 injected per-layer [N, d] uniforms (``noise_u``)
    node_mode   0 none | 1 RNG | 2 injected [N] uint8 mask (``node_mask``): NodeDrop on E0
    """
    edge_mode: int = 0
    keep: float = 1.0
    scale: float = 1.0
    edge_masks: object = None
    per_layer_edges: bool = False
    noise_mode: int = 0
    noise_u: Optional[Sequence[torch.Tensor]] = None
    node_mode: int = 0
    node_keep: float = 1.0
    node_mask: Optional[torch.Tensor] = None
    seed: int = 0
    row_bits: Optional[torch.Tensor] = None   # ``row_bitmap``: the losses read this view of the layer sum at these rows only

    def edge_mask_for(self, layer: int) -> Optional[torch.Tensor]:
        if self.edge_mode != 2:
            return None
        if isinstance(self.edge_masks, (list, tuple)):
            return self.edge_masks[layer - 1]
        return self.edge_masks


def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    z = x
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return z ^ (z >> 31)


class DevSeed(int):
    """A kernel seed whose current value also lives in a device word (``ptr``): launches pass the pointer, so a step captured
    in a CUDA graph reads whatever the host wrote there before the replay."""
    ptr: int = 0


class SeedStream:
    """Per-model stream of 64-bit kernel seeds derived from the training seed (``train.seed``).

    Device mode (CUDA-graph capture, ``graphed.GraphedStep``): ``begin_step`` draws the next ``n`` seeds of the SAME sequence,
    copies them into a device buffer, and ``next()`` hands them out in order as :class:`DevSeed` (value + address) -- the eager
    and the graphed step therefore draw identical masks / noise."""

    def __init__(self, seed: int):
        self.state = splitmix64(int(seed) & 0xFFFFFFFFFFFFFFFF)
        self.count = 0                   # seeds handed out so far (graphed.GraphedStep counts a step's draws with it)
        self._dev = None                 # (device int64 buffer, pinned host staging buffer)
        self._step_vals: List[int] = []
        self._cursor = 0

    def _advance(self) -> int:
        self.state = splitmix64(self.state)
        return self.state

    def next(self) -> int:
        self.count += 1
        if self._dev is None:
            return self._advance()
        if self._cursor >= len(self._step_vals):
            raise RuntimeError('more seeds drawn in this step than begin_step() provided (the step is not the captured one)')
        v = DevSeed(self._step_vals[self._cursor])
        v.ptr = self._dev[0].data_ptr() + 8 * self._cursor
        self._cursor += 1
        return v

    def enable_device(self, device, capacity: int = 64, ring: int = 16) -> None:
        # a ring of pinned staging rows: the host runs ahead of the GPU, so a row is rewritten only after its copy has executed
        self._dev = (torch.zeros(capacity, dtype=torch.int64, device=device), torch.zeros(ring, capacity, dtype=torch.int64).pin_memory())
        self._ring_events = [None] * ring
        self._ring_pos = 0

    def disable_device(self) -> None:
        self._dev, self._step_vals, self._cursor = None, [], 0

    @contextlib.contextmanager
    def host_draws(self):
        """Seeds drawn outside a training step (an evaluation between graph replays) come from the host sequence, as in the
        eager loop: without this they would be read from the device buffer of the last step, which they do not belong to."""
        dev, self._dev = self._dev, None
        try:
            yield
        finally:
            self._dev = dev

    def state_dict(self) -> dict:
        """The position in the sequence as two plain ints (never a DevSeed): what a training checkpoint stores."""
        return {'state': int(self.state), 'count': int(self.count)}

    def load_state_dict(self, sd: dict) -> None:
        self.state, self.count = int(sd['state']), int(sd['count'])

    def begin_step(self, n: int) -> None:
        """Draw this step's ``n`` seeds and enqueue their host -> device copy on the current stream."""
        dev, ring = self._dev
        if n > dev.numel():
            raise RuntimeError('seed buffer too small')
        self._step_vals = [self._advance() for _ in range(n)]
        self._cursor = 0
        if n == 0:
            return
        k = self._ring_pos
        self._ring_pos = (k + 1) % ring.shape[0]
        if self._ring_events[k] is not None:
            self._ring_events[k].synchronize()
        host = ring[k]
        host[:n] = torch.tensor([v - (1 << 64) if v >= (1 << 63) else v for v in self._step_vals], dtype=torch.int64)     # same 64 bits, signed
        dev[:n].copy_(host[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev.device))
        self._ring_events[k] = ev


# ------------------------------------------------------------------------------------------------
# propagation
# ------------------------------------------------------------------------------------------------

class Rows:
    """Reference to the rows [off, off+n) of view ``v`` of a [*, V, d] (or [*, d]) fp32 tensor, plus
    where their gradient goes: a sink created zeroed on first use, either of the same shape or -- ``grad_views`` = 1, a
    view-linear propagation (``Propagation.view_linear``) -- one [*, 1, d] sink that every view's gradient is added to."""

    def __init__(self, base: torch.Tensor, v: int, n_views: int, off: int, n: int, dim: int,
                 sink_get=None, token: Optional[torch.Tensor] = None, comm=None, grad_views: Optional[int] = None,
                 restricted: bool = False):
        self.base, self.v, self.n_views, self.off, self.n, self.dim = base, v, n_views, off, n, dim
        self.restricted = restricted    # the view was computed at its marked rows only: gather it by index, never whole
        self.sink_get, self.token = sink_get, token
        self.comm = comm          # RowShard: as a *table* operand only the rank's own rows are contracted
        self.grad_views = n_views if grad_views is None else grad_views
        if self.grad_views not in (1, n_views):
            raise ValueError('a sink holds every view or one summed view')

    def sub(self, lo: int, hi: int) -> 'Rows':
        """The same reference restricted to global rows [lo, hi) of the underlying tensor."""
        return Rows(self.base, self.v, self.n_views, lo, hi - lo, self.dim, self.sink_get, self.token, grad_views=self.grad_views,
                    restricted=self.restricted)

    def require_whole(self, what: str) -> None:
        if self.restricted:
            raise RuntimeError(f'sslrec_b200: view {self.v} of this layer sum was computed at the rows its ViewSpec.row_bits marks '
                               f'only; {what} reads every row')

    @property
    def stride(self) -> int:
        return self.n_views * self.dim

    @property
    def grad_stride(self) -> int:
        """Row stride of the gradient sink (elements): ``stride``, or ``dim`` when the views share one sink."""
        return self.grad_views * self.dim

    @property
    def _grad_v(self) -> int:
        return self.v if self.grad_views == self.n_views else 0

    @property
    def ptr(self) -> int:
        return self.base.data_ptr() + 4 * ((self.off * self.n_views + self.v) * self.dim)

    def grad_ptr(self) -> Optional[int]:
        if self.sink_get is None:
            return None
        g = self.sink_get()
        return g.data_ptr() + 4 * ((self.off * self.grad_views + self._grad_v) * self.dim)

    def grad_dense(self) -> torch.Tensor:
        """A strided torch view of the referenced rows' gradient in the sink."""
        g = self.sink_get().view(-1, self.grad_views, self.dim)
        return g[self.off:self.off + self.n, self._grad_v, :]

    def dense(self) -> torch.Tensor:
        """A strided torch view of the referenced rows (for inspection / tests)."""
        self.require_whole('Rows.dense()')
        return self._view()

    def _view(self) -> torch.Tensor:
        return self.base.view(-1, self.n_views, self.dim)[self.off:self.off + self.n, self.v, :]

    def take(self, idx: torch.Tensor) -> torch.Tensor:
        """The rows at ``idx`` as a contiguous [len(idx), dim] tensor (a restricted view holds them: its marked rows are the batch's)."""
        return self._view().index_select(0, idx)

    @staticmethod
    def constant(t: torch.Tensor) -> 'Rows':
        _require_cuda(t, 'constant rows')
        t = t.contiguous()
        return Rows(t, 0, 1, 0, t.shape[0], t.shape[1])


class PropState:
    """Result of one multi-view propagation (see module docstring)."""

    def __init__(self, prop: 'Propagation', e0: torch.Tensor, n_user: int):
        self.prop, self.e0, self.n_user = prop, e0, n_user
        self.n, self.dim, self.n_views = e0.shape[0], e0.shape[1], len(prop.views)
        self.E: Optional[torch.Tensor] = None
        self.layers: Dict[int, torch.Tensor] = {}
        self.token: Optional[torch.Tensor] = None
        self._g_sum = None
        self._g_layers: Dict[int, torch.Tensor] = {}
        self._g_e0 = None
        self.reg_pending: Optional[torch.Tensor] = None     # upstream gradient of sum ||E0||^2 (device scalar), folded into the last backward launch
        self.grad_views = 1 if prop.view_linear else self.n_views     # views of the E / layer sinks (1: every view's gradient summed)
        self.restricted_views = set()    # views of E computed at their row_bits rows only (Propagation.forward)

    # ---- sinks -------------------------------------------------------------------------------
    def _sink(self, like: torch.Tensor) -> torch.Tensor:
        return torch.zeros(like.shape[0], self.grad_views, self.dim, device=like.device, dtype=torch.float32)

    def g_sum(self) -> torch.Tensor:
        if self._g_sum is None:
            self._g_sum = self._sink(self.E)
        return self._g_sum

    def g_layer(self, k: int) -> torch.Tensor:
        if k == 0:
            return self.g_e0()
        if k not in self._g_layers:
            self._g_layers[k] = self._sink(self.layers[k])
        return self._g_layers[k]

    def g_e0(self) -> torch.Tensor:
        if self._g_e0 is None:
            self._g_e0 = torch.zeros_like(self.e0)
        return self._g_e0

    # ---- row references ------------------------------------------------------------------------
    def _rows(self, which, v: int, off: int, n: int) -> Rows:
        comm = self.prop.loss_comm
        if which == 'sum':
            return Rows(self.E, v, self.n_views, off, n, self.dim, self.g_sum, self.token, comm, self.grad_views,
                        restricted=v in self.restricted_views)
        k = int(which)
        if k == 0:           # layer 0 is E0 itself (ncl.py:75)
            return Rows(self.e0, 0, 1, off, n, self.dim, self.g_e0, self.token, comm)
        return Rows(self.layers[k], v, self.n_views, off, n, self.dim, lambda: self.g_layer(k), self.token, comm, self.grad_views)

    def users(self, v: int = 0, which='sum') -> Rows:
        return self._rows(which, v, 0, self.n_user)

    def items(self, v: int = 0, which='sum') -> Rows:
        return self._rows(which, v, self.n_user, self.n - self.n_user)

    def all_nodes(self, v: int = 0, which='sum') -> Rows:
        return self._rows(which, v, 0, self.n)


class Propagation:
    """K-layer LightGCN-family propagation of several augmented views in one pass per layer.

    E_v = sum_{k=0..sum_layers} X_k^(v),  X_0^(v) = nodedrop_v(E0),  X_k^(v) = perturb_v(A_v X_{k-1}^(v)).
    ``n_layers`` may exceed ``sum_layers`` (NCL runs max(L, 2*high_order) layers, ncl.py:36) and
    ``keep_layers`` lists layer outputs that losses read (and send gradients to).
    """

    def __init__(self, plan: GraphPlan, views: Sequence[ViewSpec], n_layers: int, sum_layers: Optional[int] = None,
                 keep_layers: Sequence[int] = (), noise_eps: float = 0.0, comm=None, loss_comm=None):
        self.plan, self.views = plan, list(views)
        self.n_layers = int(n_layers)
        self.sum_layers = self.n_layers if sum_layers is None else int(sum_layers)
        self.keep_layers = set(int(k) for k in keep_layers)
        self.noise_eps = float(noise_eps)
        self.comm = comm       # parallel.RowShard with shard_propagation: layer outputs live in shared tables, rows are
                               # exchanged by the kernel's peer stores (or an all-gather) after every launch
        self.loss_comm = loss_comm if loss_comm is not None else comm    # shards the InfoNCE table rows
        if not 1 <= len(self.views) <= _lib.MAX_VIEWS:
            raise ValueError('1..%d views' % _lib.MAX_VIEWS)
        if self.sum_layers > self.n_layers or self.sum_layers + 1 > _lib.MAX_SUM_SRC + 1:
            raise ValueError('sum_layers out of range')
        self.any_node = any(v.node_mode != 0 for v in self.views)
        # view-linear: every view's layers are the same linear map Â (no edge mask, no node drop).  The views then differ only
        # by the SimGCL perturbation eps sign(x) û, whose derivative is zero, so the transposed recursions of all views can be
        # summed before they run -- one [N, 1, d] sink and one-view backward launches instead of V of each
        self.view_linear = all(v.edge_mode == 0 and v.node_mode == 0 for v in self.views)

    # ---- argument block ------------------------------------------------------------------------
    def _args(self, dim: int, layer: int, transpose: bool) -> PropArgs:
        a = PropArgs()
        a.dim, a.n_views, a.transpose = dim, len(self.views), int(transpose)
        a.noise_eps = self.noise_eps
        a.noise_stream_id = layer
        per_layer = any(v.per_layer_edges for v in self.views)
        a.edge_stream_id = layer if per_layer else 0
        for i, v in enumerate(self.views):
            a.edge_mode[i] = v.edge_mode
            a.edge_keep[i] = v.keep
            a.edge_scale[i] = v.scale
            a.seed[i] = int(v.seed)
            a.seed_ptr[i] = getattr(v.seed, 'ptr', 0) or None
            m = v.edge_mask_for(layer)
            a.edge_mask[i] = _ptr(m)
            if not transpose:
                a.noise_mode[i] = v.noise_mode
                if v.noise_mode == 2:
                    a.noise_u[i] = _ptr(v.noise_u[layer - 1])
        return a

    def _launch(self, a: PropArgs, ref: torch.Tensor):
        name = 'prop_bwd' if a.transpose else 'prop_fwd'
        meta = None
        if TIMER is not None:
            shared = a.in_views == 1 and not any(a.edge_mode[i] for i in range(a.n_views))
            gather = 1 if shared else a.n_views
            restricted = [i for i in range(a.n_views) if a.row_bits[i]]
            if restricted and not shared and not torch.cuda.is_current_stream_capturing():
                # a restricted view gathers the stored entries of its marked rows only (host read: timed runs only)
                gather -= sum(1.0 - self._marked_entry_fraction(self.views[i].row_bits) for i in restricted)
            meta = dict(views=a.n_views, gather_views=gather, restricted_views=len(restricted), dim=a.dim, residual=bool(a.residual), reg_src2=bool(a.reg_src2),
                        x_out=bool(a.x_out), sum_out=bool(a.sum_out), reduce_views=bool(a.reduce_views),
                        sum_src=[a.sum_src_views[i] for i in range(a.n_sum_src)], reg_src=bool(a.reg_src),
                        nnz=self.plan.nnz, rows=self.plan.n_rows)
        with torch.cuda.device(ref.device), _timed(name, meta):
            check(lib.ssl_propagate_layer(self.plan.handle, C.byref(a), _stream(ref)), 'ssl_propagate_layer')

    def _marked_entry_fraction(self, bits: torch.Tensor) -> float:
        """Share of the plan's stored entries that lie in the rows a row bitmap marks."""
        plan = self.plan
        deg = getattr(plan, '_deg_dev', None)
        if deg is None or deg.device != bits.device:
            deg = torch.from_numpy(plan.h_rowptr.astype('int64')).diff().to(bits.device)
            plan._deg_dev = deg
        rows = torch.arange(deg.numel(), device=bits.device)
        marked = (bits.to(torch.int64)[rows >> 5] >> (rows & 31)) & 1
        return float((deg * marked).sum().item()) / max(1, plan.nnz)

    def _node_drop(self, x: torch.Tensor, out: torch.Tensor, backward: bool):
        V = len(self.views)
        mode = (C.c_int32 * V)(*[v.node_mode for v in self.views])
        keep = (C.c_float * V)(*[v.node_keep for v in self.views])
        masks = (C.c_void_p * V)(*[_ptr(v.node_mask) for v in self.views])
        seeds = (C.c_uint64 * V)(*[int(v.seed) for v in self.views])
        seed_ptrs = (C.c_void_p * V)(*[(getattr(v.seed, 'ptr', 0) or None) for v in self.views])
        n = out.shape[0] if backward else x.shape[0]
        with torch.cuda.device(x.device):
            # the table is full height on every rank (a row-sharded plan shards the SpMM, not NodeDrop): the RNG is keyed by
            # the global row, so the offset of row 0 is 0 whatever the plan owns
            check(lib.ssl_node_drop_dev(x.data_ptr(), out.data_ptr(), n, x.shape[-1], V, int(backward), mode, keep, masks, seeds, seed_ptrs,
                                        0, _stream(x)), 'ssl_node_drop')

    # ---- output tables ---------------------------------------------------------------------------
    def _out(self, key, shape, ref: torch.Tensor):
        """A full-height output table: plain memory on one GPU, a persistent shared table (parallel.SharedTable) when the
        propagation is row-sharded.  Returns (tensor, shared table or None)."""
        if self.comm is None:
            return torch.empty(shape, device=ref.device, dtype=torch.float32), None
        tb = self.comm.table(key, shape, ref.device)
        return tb.t, tb

    @staticmethod
    def _set_peers(a: PropArgs, field: str, tb) -> None:
        """Where the launch stores its rows besides (or instead of) this GPU's table: the multicast address of the shared table
        when there is one -- the ONLY store target then, the switch delivers the row to every copy including ours -- else
        the peers' mapped copies."""
        if tb is None:
            return
        if tb.mc_ptr:
            setattr(a, field[:-len('_peers')], tb.mc_ptr)          # x_out / sum_out = the multicast address
            return
        if not tb.peer_ptrs:
            return
        a.n_peers = len(tb.peer_ptrs)
        arr = getattr(a, field)
        for q, ptr in enumerate(tb.peer_ptrs):
            arr[q] = ptr

    def _exchange(self, tables) -> None:
        """Complete the tables a launch wrote (owned rows -> every rank)."""
        tables = [tb for tb in tables if tb is not None]
        if self.comm is None or not tables:
            return
        with _timed('prop_exchange', dict(tables=len(tables))):
            if self.comm.transport == 'symm':
                self.comm.barrier()                      # the rows travelled with the kernel's stores
            else:
                for tb in tables:
                    self.comm.sync_rows(tb)

    # ---- forward -------------------------------------------------------------------------------
    def forward(self, e0: torch.Tensor, n_user: int) -> PropState:
        """e0: the full [N, d] table (every rank holds all of it; rows are sharded for compute)."""
        _require_cuda(e0, 'embedding table')
        if not e0.is_contiguous():
            raise RuntimeError('embedding table must be contiguous')
        if self.sum_layers == 0:
            raise ValueError('sum_layers must be >= 1')
        st = PropState(self, e0, n_user)
        N, d, V = e0.shape[0], e0.shape[1], len(self.views)
        if self.plan.n != N:
            raise RuntimeError(f'plan is for {self.plan.n} nodes, the table has {N} rows')
        opts = dict(device=e0.device, dtype=torch.float32)
        if self.any_node:
            x0 = torch.empty(N, V, d, **opts)
            self._node_drop(e0, x0, backward=False)
            x_prev, in_views = x0, V
            srcs = [(x0, V)]
        else:
            x_prev, in_views = e0, 1
            srcs = [(e0, 1)]
        st.x0 = x_prev
        for k in range(1, self.n_layers + 1):
            a = self._args(d, k, transpose=False)
            a.in_views = in_views
            a.x_in = x_prev.data_ptr()
            need_out = (k < self.n_layers) or (k in self.keep_layers)
            x_out = x_tb = e_tb = None
            if need_out:
                x_out, x_tb = self._out(('x', k), (N, V, d), e0)
                a.x_out = x_out.data_ptr()
                self._set_peers(a, 'x_out_peers', x_tb)
            if k == self.sum_layers:
                st.E, e_tb = self._out('E', (N, V, d), e0)
                a.sum_out = st.E.data_ptr()
                if not need_out and self.comm is None:
                    # views the losses read at batch rows only: gathered and written at the marked rows (the kernel accepts a
                    # restriction only for a launch that writes sum_out alone; a row-sharded launch computes every row)
                    for i, v in enumerate(self.views):
                        if v.row_bits is not None:
                            a.row_bits[i] = v.row_bits.data_ptr()
                            st.restricted_views.add(i)
                self._set_peers(a, 'sum_out_peers', e_tb)
                a.n_sum_src = len(srcs)
                for i, (s, sv) in enumerate(srcs):
                    a.sum_src[i] = s.data_ptr()
                    a.sum_src_views[i] = sv
            self._launch(a, e0)
            self._exchange([x_tb, e_tb])
            if x_out is not None:
                if k in self.keep_layers:
                    st.layers[k] = x_out
                if k < self.sum_layers:
                    srcs.append((x_out, V))
                x_prev, in_views = x_out, V
        return st

    # ---- backward ------------------------------------------------------------------------------
    def backward(self, st: PropState) -> torch.Tensor:
        """Consumes the sinks of ``st``; returns dE0 [N, d].  Row-sharded: only the rows this rank owns are computed
        (the others are zero) -- the sharded Adam updates exactly those and stores them to the peers.

        View-linear: the sinks hold sum_v G^v, and D_{k-1} = Â^T D_k + sum_v G^v_{k-1} runs as one view."""
        e0 = st.e0
        N, d, V = st.n, st.dim, st.grad_views
        opts = dict(device=e0.device, dtype=torch.float32)
        L, S = self.n_layers, self.sum_layers

        def residual(k: int) -> Optional[torch.Tensor]:
            parts = []
            if k <= S and st._g_sum is not None:
                parts.append(st._g_sum)
            if k >= 1 and k in st._g_layers:
                parts.append(st._g_layers[k])
            if not parts:
                return None
            return parts[0] if len(parts) == 1 else parts[0] + parts[1]

        # D_k = total gradient w.r.t. X_k; start at the deepest layer that received any gradient
        top = L
        while top >= 1 and residual(top) is None:
            top -= 1
        # regulariser gradient 2 g E0 (loss_utils.py:20-24): read straight from E0 by the last launch's epilogue when that
        # launch exists (no [N, d] sink to zero, fill and re-read); otherwise materialised into the E0 sink
        fold_reg = st.reg_pending is not None and not self.any_node and top >= 1
        if st.reg_pending is not None and not fold_reg:
            with torch.cuda.device(e0.device):
                check(lib.ssl_axpy(e0.data_ptr(), st.g_e0().data_ptr(), e0.numel(), st.reg_pending.data_ptr(), 2.0, _stream(e0)), 'ssl_axpy')
        g_e0 = st._g_e0
        if top == 0:
            d0 = residual(0)     # only X_0 got gradient (through the layer sum)
            if d0 is None:
                return g_e0 if g_e0 is not None else torch.zeros_like(e0)
            out = d0.sum(1) if not self.any_node else self._node_bwd(d0, g_e0, e0)
            if g_e0 is not None and not self.any_node:
                out = out + g_e0
            return out
        D = residual(top)
        for k in range(top, 0, -1):           # D_{k-1} = A_v^T D_k + residual(k-1)
            a = self._args(d, k, transpose=True)
            a.n_views = a.in_views = V
            a.x_in = D.data_ptr()
            res = residual(k - 1)
            if res is not None:
                a.residual = res.data_ptr()
            last = (k == 1)
            if last and not self.any_node:
                out = torch.empty(N, d, **opts) if self.comm is None else torch.zeros(N, d, **opts)
                a.sum_out, a.reduce_views = out.data_ptr(), 1
                if fold_reg:
                    a.reg_src, a.reg_coef, a.reg_coef_dev = e0.data_ptr(), 2.0, st.reg_pending.data_ptr()
                    a.reg_src2 = _ptr(g_e0)
                elif g_e0 is not None:
                    a.reg_src, a.reg_coef = g_e0.data_ptr(), 1.0
                self._launch(a, e0)
                return out
            x_out, x_tb = self._out(('d', k % 2), (N, V, d), e0)
            a.x_out = x_out.data_ptr()
            self._set_peers(a, 'x_out_peers', x_tb)
            self._launch(a, e0)
            self._exchange([x_tb])
            D = x_out
        return self._node_bwd(D, g_e0, e0)

    def _node_bwd(self, d0: torch.Tensor, g_e0: Optional[torch.Tensor], e0: torch.Tensor) -> torch.Tensor:
        out = g_e0.clone() if g_e0 is not None else torch.zeros_like(e0)
        self._node_drop(d0, out, backward=True)
        return out


class _PropFn(torch.autograd.Function):
    """Autograd node of a propagation: inputs are the two embedding parameters, the only autograd
    output is the 0-d token; E lives in the PropState."""

    @staticmethod
    def forward(ctx, user_e, item_e, prop: Propagation, e0: torch.Tensor, holder: dict):
        st = prop.forward(e0, user_e.shape[0])
        ctx.st = st
        holder['state'] = st
        return torch.zeros((), device=e0.device, dtype=torch.float32)

    @staticmethod
    def backward(ctx, g_token):
        st = ctx.st
        de0 = st.prop.backward(st)
        nu = st.n_user
        # token -> grad_fn -> ctx -> state -> token is a reference cycle through the autograd node: break it now instead of leaving
        # it to the cyclic collector (it would keep the step's tables, and the parameters' gradient accumulators, alive until then)
        st.token = None
        ctx.st = None
        return de0[:nu], de0[nu:], None, None, None


def propagate(prop: Propagation, user_e: torch.Tensor, item_e: torch.Tensor, e0: Optional[torch.Tensor] = None) -> PropState:
    """Run the propagation.  ``e0`` is the flat [N, d] table the two parameters are views of (built by
    a concat when they are not)."""
    if e0 is None:
        e0 = flat_table(user_e, item_e)
    if torch.is_grad_enabled() and (user_e.requires_grad or item_e.requires_grad):
        holder: dict = {}
        token = _PropFn.apply(user_e, item_e, prop, e0, holder)
        st = holder['state']
        st.token = token
        return st
    return prop.forward(e0.detach(), user_e.shape[0])


class _SpmmFn(torch.autograd.Function):
    """Single masked propagation layer on a dense autograd tensor: Y = A_m X, dX = A_m^T dY (the same
    kernel with transpose = 1).  Used where layers are interleaved with other autograd ops (HCCF)."""

    @staticmethod
    def forward(ctx, x, plan, view, layer):
        ctx.pack = (plan, view, layer)
        return _spmm_once(plan, x.detach(), view, layer, False)

    @staticmethod
    def backward(ctx, g):
        plan, view, layer = ctx.pack
        return _spmm_once(plan, g, view, layer, True), None, None, None


def _spmm_once(plan: GraphPlan, x: torch.Tensor, view: ViewSpec, layer: int, transpose: bool) -> torch.Tensor:
    _require_cuda(x, 'spmm input')
    if plan.n_rows != plan.n:
        raise RuntimeError('engine.spmm needs a plan that owns every row (HCCF / LightGCL do not row-shard the propagation)')
    x = x.contiguous()
    prop = Propagation(plan, [view], max(1, layer))
    a = prop._args(x.shape[1], layer, transpose)
    out = torch.empty(plan.n_rows, 1, x.shape[1], device=x.device, dtype=torch.float32)
    a.in_views, a.x_in, a.x_out = 1, x.data_ptr(), out.data_ptr()
    a.noise_mode[0] = 0
    prop._launch(a, x)
    return out.view(plan.n_rows, x.shape[1])


def spmm(plan: GraphPlan, x: torch.Tensor, view: Optional[ViewSpec] = None, layer: int = 1) -> torch.Tensor:
    """t.spmm(adj, embeds) (lightgcn.py:29 / hccf.py:36) with an optional in-kernel edge mask."""
    return _SpmmFn.apply(x, plan, view if view is not None else ViewSpec(), layer)


def spmm_exact(plan: GraphPlan, x: torch.Tensor) -> torch.Tensor:
    """Y = A X in the accumulation order of the reference's CPU ``t.spmm`` (lightgcn.py:29): every output element one sequential fp32 FMA
    chain over the CSR row in ascending column order, rows never split (``ssl_spmm_exact``; the opt-in evaluation mode ``test.exact_order``).
    No autograd, not for training: a hub row is as slow as its length."""
    _require_cuda(x, 'spmm input')
    if plan.n_rows != plan.n:
        raise RuntimeError('engine.spmm_exact needs a plan that owns every row (single GPU)')
    if x.dim() != 2 or x.shape[0] != plan.n or x.stride(1) != 1:
        raise RuntimeError('engine.spmm_exact: x must be [N, d] with unit column stride')
    y = torch.empty(plan.n_rows, x.shape[1], device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        check(lib.ssl_spmm_exact(plan.rowptr_dev().data_ptr(), plan.colidx.data_ptr(), plan.vals.data_ptr(), plan.n_rows, x.data_ptr(), x.stride(0),
                                 x.shape[1], y.data_ptr(), y.stride(0), _stream(x)), 'ssl_spmm_exact')
    return y


def flat_table(user_e: torch.Tensor, item_e: torch.Tensor) -> torch.Tensor:
    """[N, d] table of both sides without a copy when the parameters are adjacent views of one
    storage (FlatEmbeddings), else a concat (lightgcn.py:34)."""
    ud, idt = user_e.detach(), item_e.detach()
    if (ud.is_contiguous() and idt.is_contiguous() and ud.untyped_storage().data_ptr() == idt.untyped_storage().data_ptr()
            and idt.data_ptr() == ud.data_ptr() + ud.numel() * 4 and ud.shape[1] == idt.shape[1]):
        return torch.as_strided(ud, (ud.shape[0] + idt.shape[0], ud.shape[1]), (ud.shape[1], 1))
    return torch.cat([ud, idt], 0)


# ------------------------------------------------------------------------------------------------
# losses
# ------------------------------------------------------------------------------------------------

def _i64(t: torch.Tensor, device) -> torch.Tensor:
    if t.dtype != torch.int64 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.int64).contiguous()
    return t


# ---- train.deterministic: batch rows added into their sinks in a fixed order ------------------------------------------

DETERMINISTIC: Optional[bool] = None     # tests set it; None = the optional key train.deterministic of the config


def deterministic() -> bool:
    """The one switch of the ordered mode (optional key ``train.deterministic``, INTEGRATION §2).  On: every loss backward whose
    ids can repeat has its loss kernel write each position's contribution c_p into a stage (identity ids, one add per element)
    and adds the stage into the sink with ``ssl_scatter_rows_ordered`` (sink[r] + ((c_p1 + c_p2) + ...), positions in order),
    instead of adding c_p with float atomics in whatever order the warps run; ``rows_at`` gathers with the same ordered
    backward.  A training step is then a pure function of (parameters, optimizer state, batch, seeds).  Single GPU only."""
    if DETERMINISTIC is not None:
        return bool(DETERMINISTIC)
    from .config import configs
    return bool(configs.get('train', {}).get('deterministic', False))


def _memo(t: torch.Tensor, name: str, fn):
    """fn(t), kept on ``t`` while its contents are unchanged (``_version``): an index list is argsorted once per step however
    many terms scatter by it.  Values computed inside a CUDA-graph capture are kept apart from eager ones, so the graph
    recomputes at every replay what it captured."""
    stamp = (t._version, torch.cuda.is_current_stream_capturing())
    memo = getattr(t, '_ssl_memo', None)
    if memo is None or memo[0] != stamp:
        memo = t._ssl_memo = (stamp, {})
    if name not in memo[1]:
        memo[1][name] = fn(t)
    return memo[1][name]


def _stage(n: int, d: int, dev) -> torch.Tensor:
    """[n, d] stage of per-position contributions.  Filled with -0.0, the exact additive identity (+0.0 + -0.0 is +0.0), so
    the one add a loss kernel makes to each element leaves exactly its c_p there."""
    return torch.full((n, d), -0.0, device=dev, dtype=torch.float32)


def scatter_rows_ordered(stage: torch.Tensor, ids: torch.Tensor, sink_ptr: int, sink_stride: int) -> None:
    """sink row ids[p] += stage[p] for every position p, in the order of ``ssl_scatter_rows_ordered`` (positions with a negative
    id skipped).  ``stage`` [P, d] contiguous fp32, ``ids`` [P] int64 on its device; the sink is addressed as sink_ptr + 4 *
    (row * sink_stride + k)."""
    order = _memo(ids, 'order', lambda t: torch.argsort(t, stable=True))
    with torch.cuda.device(stage.device):
        check(lib.ssl_scatter_rows_ordered(stage.data_ptr(), ids.data_ptr(), order.data_ptr(), ids.numel(), stage.shape[1], sink_ptr,
                                           sink_stride, _stream(stage)), 'ssl_scatter_rows_ordered')


def _scatter_blocks(stage: torch.Tensor, parts) -> None:
    """Scatter consecutive blocks of ``stage``, one per part (ids, sink pointer, sink stride).  Two parts that address the same
    sink (SimGCL's view-linear sinks make an InfoNCE term's e1 and e2 the same rows) are ONE scatter over their concatenated
    positions; otherwise one scatter per part, in order."""
    if len(parts) == 2 and parts[0][1:] == parts[1][1:]:
        ids = parts[0][0] if parts[0][0] is parts[1][0] else None
        both = _memo(ids, 'twice', lambda t: torch.cat([t, t])) if ids is not None else torch.cat([parts[0][0], parts[1][0]])
        parts = [(both,) + tuple(parts[0][1:])]
    row = 0
    for ids, ptr, stride in parts:
        scatter_rows_ordered(stage[row:row + ids.numel()], ids, ptr, stride)
        row += ids.numel()


class _RowsAtFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, ids):
        ctx.shape, ctx.ids = table.shape, ids
        return table.index_select(0, ids)

    @staticmethod
    def backward(ctx, g):
        sink = torch.zeros(ctx.shape, device=g.device, dtype=torch.float32)
        scatter_rows_ordered(g.contiguous(), ctx.ids, sink.data_ptr(), sink.stride(0))          # c_p = g[p]
        return sink, None


def rows_at(table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """``table[ids]`` (the batch gathers of hccf.py:94 and lightgcl.py:117-121).  Under ``deterministic()`` its backward adds
    the gathered rows' gradients into a zeroed table gradient with the ordered scatter instead of torch's index backward."""
    if not deterministic():
        return table[ids]
    _require_cuda(table, 'gathered table')
    return _RowsAtFn.apply(table, _i64(ids, table.device))


def _tokens(*rows: Rows) -> List[torch.Tensor]:
    seen, out = set(), []
    for r in rows:
        if r is not None and r.token is not None and id(r.token) not in seen:
            seen.add(id(r.token))
            out.append(r.token)
    return out


def _bpr_fwd(users: Rows, items: Rows, ancs, poss, negs):
    dev = users.base.device
    B = ancs.numel()
    loss_b = torch.empty(B, device=dev)
    coef = torch.empty(B, device=dev)
    out = torch.empty((), device=dev)
    with torch.cuda.device(dev):
        s = _stream(users.base)
        check(lib.ssl_bpr_fwd(users.ptr, users.stride, items.ptr, items.stride, ancs.data_ptr(), poss.data_ptr(),
                              negs.data_ptr(), B, users.dim, loss_b.data_ptr(), coef.data_ptr(), s), 'ssl_bpr_fwd')
        check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0, out.data_ptr(), s), 'ssl_sum')
    return out, coef


def _bpr_bwd(users: Rows, items: Rows, ancs, poss, negs, coef, g, distinct: bool = False):
    """``distinct``: the caller's ids never repeat (every sink element gets one add), so the atomic kernel is order-fixed as it is."""
    g = g.contiguous()
    if not distinct and deterministic():
        # the kernel on the gathered rows with identity ids computes the same c_p into stages; users are positions ancs[0..B),
        # items poss[0..B) then negs[0..B) as positions B..2B of one scatter
        B, d = ancs.numel(), users.dim
        item_ids = torch.cat([poss, negs])
        u, i = users.take(ancs), items.take(item_ids)
        su, si = _stage(B, d, g.device), _stage(2 * B, d, g.device)
        ar = torch.arange(B, device=g.device)
        with torch.cuda.device(g.device):
            check(lib.ssl_bpr_bwd(u.data_ptr(), d, i.data_ptr(), d, ar.data_ptr(), ar.data_ptr(), (ar + B).data_ptr(), B, d, coef.data_ptr(),
                                  g.data_ptr(), 1.0, su.data_ptr(), d, si.data_ptr(), d, _stream(g)), 'ssl_bpr_bwd')
        scatter_rows_ordered(su, ancs, users.grad_ptr(), users.grad_stride)
        scatter_rows_ordered(si, item_ids, items.grad_ptr(), items.grad_stride)
        return
    with torch.cuda.device(g.device):
        check(lib.ssl_bpr_bwd(users.ptr, users.stride, items.ptr, items.stride, ancs.data_ptr(), poss.data_ptr(),
                              negs.data_ptr(), ancs.numel(), users.dim, coef.data_ptr(), g.data_ptr(), 1.0,
                              users.grad_ptr(), users.grad_stride, items.grad_ptr(), items.grad_stride, _stream(g)), 'ssl_bpr_bwd')


class _BprFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, users: Rows, items: Rows, ancs, poss, negs, *tokens):
        out, coef = _bpr_fwd(users, items, ancs, poss, negs)
        ctx.pack = (users, items, ancs, poss, negs, coef, len(tokens))
        return out

    @staticmethod
    def backward(ctx, g):
        users, items, ancs, poss, negs, coef, nt = ctx.pack
        _bpr_bwd(users, items, ancs, poss, negs, coef, g)
        zero = torch.zeros((), device=g.device)
        return (None,) * 5 + (zero,) * nt


def bpr_loss_sum(users: Rows, items: Rows, ancs, poss, negs) -> torch.Tensor:
    """sum_b softplus(a.n - a.p) over gathered rows (lightgcn.py:48-52 + loss_utils.py:7-10)."""
    dev = users.base.device
    ancs, poss, negs = _i64(ancs, dev), _i64(poss, dev), _i64(negs, dev)
    return _BprFn.apply(users, items, ancs, poss, negs, *_tokens(users, items))


# cached: every eager step asks again for the same few shapes, and the search over splits costs up to tens of
# microseconds of host time per call, on a step whose rate follows the host's enqueue on some hosts (r09 §7)
@functools.lru_cache(maxsize=1024)
def choose_split(n_rtiles: int, n_ctiles: int, slots: int = 2 * NUM_SM, prefer_few: bool = False) -> int:
    """Number of chunks the streamed operand is cut into: n_rtiles * n_split CTAs on ``slots`` resident-CTA slots (2 per SM for
    the FFMA kernel at dim <= 64, 1 per SM for the tensor-core kernel), every CTA keeping >= 4 tiles.

    ``prefer_few`` (the persistent tensor-core kernel, one CTA per SM looping over n_rtiles * n_split units): minimise
    rounds(s) * (tiles_per_unit(s) + c)  with c = 5 tile-times of per-unit overhead (R fragment load, pipeline restart,
    O write-out), fitted to an n_split sweep of that kernel at the amazon forward shape on an H100 (profiles/r04_nce_tc.md;
    the sweep of the 3xFP16 kernel in profiles/r07_nce_f16x3.md fits the same c); fewer, longer units than the pure
    wave-efficiency rule picks.  The split only changes how the work is cut, never the
    result beyond summation order.
    Otherwise: the split with the best wave efficiency (FFMA kernel)."""
    max_split = max(1, min(n_ctiles // 4 if n_ctiles >= 4 else 1, 64))
    if prefer_few:
        best, best_cost = 1, None
        for s in range(1, max_split + 1):
            cost = math.ceil(n_rtiles * s / slots) * (math.ceil(n_ctiles / s) + 5.0)
            if best_cost is None or cost < best_cost - 1e-9:
                best, best_cost = s, cost
        return best
    effs = []
    for s in range(1, max_split + 1):
        ctas = n_rtiles * s
        effs.append((ctas / (math.ceil(ctas / slots) * slots), s))
    return max(effs, key=lambda t: (round(t[0], 9), -t[1]))[1]


def contraction_kind(d: int, offset: float, raw: bool = False, colscale_range: Optional[float] = None) -> str:
    """The InfoNCE contraction kernel for rows of width ``d`` at ``offset``: 'ffma' (FP32 FMA, any d), 'tf32x3' (3xTF32 on the
    tensor cores: raw rows, which the 3xFP16 operand bound does not cover, and offsets above F16X3_MAX_OFFSET) or 'f16x3'.
    ``colscale_range``: max / min of the column weights of a weighted forward (``ssm_in_batch_sum``); 3xFP16 takes it only
    while offset + (1 + log2(range)) / 2 <= F16X3_NO_FLUSH_OFFSET, where no E' reaches the flush rule (the bound is derived in
    include/sslrec_b200.h, a28); past it an E' below 2^-14 keeps 2^-11 of its digits, so 3xTF32 runs it."""
    if not USE_TENSOR_CORES or d not in (32, 64):
        return 'ffma'
    if raw or not f16x3_applies(offset):
        return 'tf32x3'
    if colscale_range is not None and offset + 0.5 * (1.0 + math.log2(colscale_range)) > F16X3_NO_FLUSH_OFFSET:
        return 'tf32x3'
    return 'f16x3'


@dataclass
class Operand:
    """One side of the contraction: ``n`` rows, ``hat`` [npad, d] (normalised, scaled, zero-padded) and ``rinv`` [max(n, 1)]
    (None for raw rows), plus the copies the ``kind`` kernel reads (None: hat and rinv only): the FFMA kernel's K-major tile
    copy ``t`` [npad / 64, d, 64], the tensor-core kernels' hi / lo split [npad, d] (fp16 for 3xFP16) and 3xTF32's
    transposed split ``thi`` / ``tlo`` [d, npad]."""
    kind: Optional[str]
    n: int
    npad: int
    hat: torch.Tensor
    rinv: Optional[torch.Tensor]
    t: Optional[torch.Tensor] = None
    hi: Optional[torch.Tensor] = None
    lo: Optional[torch.Tensor] = None
    thi: Optional[torch.Tensor] = None
    tlo: Optional[torch.Tensor] = None


def _operand(rows: Rows, idx, norm_mode: int, alpha: float, s: int, kind: Optional[str] = None, streamed: bool = False,
             npad: Optional[int] = None) -> Operand:
    """rows[idx] (every row when ``idx`` is None) normalised by ``norm_mode`` (3: raw rows) and scaled by ``alpha``, with the
    copies the ``kind`` kernel reads of its resident operand R or, ``streamed``, also of its streamed operand C (3xFP16 reads
    its hi / lo parts in both roles).  ``npad`` defaults to ceil64(n)."""
    n, d, dev = (rows.n if idx is None else idx.numel()), rows.dim, rows.base.device
    npad = ceil_to(n, 64) if npad is None else npad
    f = dict(device=dev, dtype=torch.float32)
    op = Operand(kind, n, npad, torch.empty(npad, d, **f), None if norm_mode == 3 else torch.empty(max(n, 1), **f))
    if kind == 'f16x3':
        op.hi, op.lo = torch.empty(npad, d, device=dev, dtype=torch.float16), torch.empty(npad, d, device=dev, dtype=torch.float16)
        check(lib.ssl_rows_normalize_f16x3(rows.ptr, rows.stride, _ptr(idx), n, d, norm_mode, alpha, op.hat.data_ptr(),
                                           op.rinv.data_ptr(), op.hi.data_ptr(), op.lo.data_ptr(), s), 'ssl_rows_normalize_f16x3')
        return op
    if kind == 'tf32x3':
        op.hi, op.lo = torch.empty(npad, d, **f), torch.empty(npad, d, **f)
        if streamed:
            op.thi, op.tlo = torch.empty(d, npad, **f), torch.empty(d, npad, **f)
    elif kind == 'ffma' and streamed:
        op.t = torch.empty(npad // 64, d, 64, **f)
    check(lib.ssl_rows_normalize(rows.ptr, rows.stride, _ptr(idx), n, d, norm_mode, alpha, op.hat.data_ptr(), _ptr(op.t),
                                 _ptr(op.rinv), _ptr(op.hi), _ptr(op.lo), _ptr(op.thi), _ptr(op.tlo), 0 if kind is None else npad, s),
          'ssl_rows_normalize')
    return op


def _n_split(R: Operand, C: Operand) -> int:
    """choose_split for a contraction of R against C on their kernel: the tensor-core kernels are persistent, one CTA per SM."""
    tc = R.kind != 'ffma'
    return choose_split((R.n + 127) // 128, C.npad // 64, slots=NUM_SM if tc else 2 * NUM_SM, prefer_few=tc)


_GEMM_ENTRY = dict(ffma='ssl_softmax_gemm', tf32x3='ssl_softmax_gemm_tf32x3', f16x3='ssl_softmax_gemm_f16x3')


def _contract(R: Operand, C: Operand, colscale, offset: float, n_split: int, rowsum_part, o_part, s: int, live=None,
              live_role: int = LIVE_ROWS, bwd: Optional[bool] = None):
    """One launch of the contraction of R against C on their kernel, timed as the forward role (R = anchors) or, with
    ``colscale``, the backward role (R = table, C = anchors).  ``live``: the device count that bounds the ``live_role`` side.
    ``bwd`` names the role where ``colscale`` does not tell it: the weighted forward of ``ssm_in_batch_sum`` passes False."""
    name = _GEMM_ENTRY[R.kind] + ('' if live is None else '_live')
    if R.kind == 'ffma':
        ops = (R.hat.data_ptr(), R.n, C.hat.data_ptr(), C.t.data_ptr(), C.n)
    elif R.kind == 'tf32x3':
        ops = (R.hi.data_ptr(), R.lo.data_ptr(), R.n, C.hi.data_ptr(), C.lo.data_ptr(), C.thi.data_ptr(), C.tlo.data_ptr(), C.npad, C.n)
    else:
        ops = (R.hi.data_ptr(), R.lo.data_ptr(), R.n, C.hi.data_ptr(), C.lo.data_ptr(), C.n)
    tail = () if live is None else (live.data_ptr(), live_role)
    d, bwd = R.hat.shape[1], (colscale is not None) if bwd is None else bwd
    meta = dict(B=C.n, n=R.n) if bwd else dict(B=R.n, n=C.n)
    with _timed('nce_gemm_bwd' if bwd else 'nce_gemm_fwd', dict(meta, dim=d, tc=R.kind != 'ffma')):
        check(getattr(lib, name)(*ops, d, _ptr(colscale), offset, n_split, _ptr(rowsum_part), o_part.data_ptr(), *tail, s),
              f'{name}({"bwd" if bwd else "fwd"})')


def _nce_fwd(e1: Rows, e2: Rows, table: Rows, idx, idx2, tau, norm_mode, mean, deno_eps, live=None, distinct=False):
    """``live``: optional int64 DEVICE scalar; only the first ``*live`` of the ``idx`` rows are anchors (a padded list of
    capacity idx.numel(), see ``dense_infonce_spec_nodes_mean_dev``).  Shapes and n_split then depend on the capacity only.
    ``distinct``: the ids of ``idx`` never repeat (see ``_bpr_bwd``)."""
    dev = table.base.device
    table.require_whole('an InfoNCE table operand')
    d, B = table.dim, idx.numel()
    f = dict(device=dev, dtype=torch.float32)
    comm = table.comm
    full_table, npad = table, None
    if live is not None and (comm is not None or not mean):
        raise RuntimeError('a device-bounded InfoNCE term is a mean on one GPU')
    if comm is not None:                  # contract only this rank's rows of the table; partials are all-reduced
        lo, hi = comm.side_range(table.off, table.n)
        table = table.sub(lo, hi)
        npad = max(64, ceil_to(table.n, 64))
    off = LOG2E / tau
    kind = contraction_kind(d, off)
    rowsum, obar, loss_b, out = torch.empty(B, **f), torch.empty(B, d, **f), torch.empty(B, **f), torch.empty((), **f)
    with torch.cuda.device(dev):
        s = _stream(table.base)
        # anchors and table are R and C here and C and R in the backward: both get the copies of either role
        a = _operand(e1, idx, norm_mode, off, s, kind, streamed=True)
        p = _operand(e2, idx2, norm_mode, 1.0, s)
        t = _operand(table, None, norm_mode, 1.0, s, kind, streamed=True, npad=npad)
        n_split = _n_split(a, t)
        rs_part, o_part = torch.zeros(n_split, B, **f), torch.zeros(n_split, B, d, **f)
        _contract(a, t, None, off, n_split, rs_part, o_part, s, live, LIVE_ROWS)
        if comm is not None:
            red = torch.cat([o_part.sum(0), rs_part.sum(0).unsqueeze(1)], 1)         # [B, d+1]
            comm.allreduce_sum(red)
            o_part, rs_part, n_split = red[:, :d].contiguous().unsqueeze(0), red[:, d].contiguous().unsqueeze(0), 1
        check(lib.ssl_nce_finalize(rs_part.data_ptr(), o_part.data_ptr(), n_split, B, d, a.hat.data_ptr(), p.hat.data_ptr(),
                                   tau, deno_eps * math.exp(-1.0 / tau), rowsum.data_ptr(), obar.data_ptr(),
                                   loss_b.data_ptr(), s), 'ssl_nce_finalize')
        if live is not None:          # (1 / live) sum_{b < live} loss_b: the padding rows' values are never read
            check(lib.ssl_sum_live(loss_b.data_ptr(), B, live.data_ptr(), 1.0, out.data_ptr(), s), 'ssl_sum_live')
        else:
            check(lib.ssl_sum(loss_b.data_ptr(), B, (1.0 / B) if mean else 1.0, out.data_ptr(), s), 'ssl_sum')
    return out, (e1, e2, table, idx, tau, mean, a, p, t, rowsum, obar, full_table, comm, live, distinct)


def _nce_bwd_rows_ordered(saved, g, g1, g2, scale, s):
    """The row gradients of an InfoNCE term under ``deterministic()``: the row kernel with identity ids into a stage of one block
    per sink ([g1 positions; g2 positions]), then the ordered scatter.  Count-bounded (``live``): positions b >= *live get id -1."""
    e1, e2, _, idx, tau, _, a, p, _, _, obar, _, _, live, _ = saved
    B, d = idx.numel(), a.hat.shape[1]
    sinks = [(ptr, rows.grad_stride) for ptr, rows in ((g1, e1), (g2, e2)) if ptr is not None]
    stage = _stage(len(sinks) * B, d, g.device)
    s1 = stage.data_ptr() if g1 is not None else None
    s2 = stage[B if g1 is not None else 0:].data_ptr() if g2 is not None else None
    ar = torch.arange(B, device=g.device)
    if live is not None:
        check(lib.ssl_nce_bwd_rows_live(a.hat.data_ptr(), p.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), p.rinv.data_ptr(),
                                        ar.data_ptr(), B, live.data_ptr(), d, tau, g.data_ptr(), 1.0, s1, d, s2, d, s), 'ssl_nce_bwd_rows_live')
        ids = torch.where(ar < live, idx, -1)
    else:
        check(lib.ssl_nce_bwd_rows(a.hat.data_ptr(), p.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), p.rinv.data_ptr(),
                                   ar.data_ptr(), B, d, tau, g.data_ptr(), scale, s1, d, s2, d, s), 'ssl_nce_bwd_rows')
        ids = idx
    _scatter_blocks(stage, [(ids, ptr, stride) for ptr, stride in sinks])


def _nce_bwd(saved, g):
    e1, e2, table, idx, tau, mean, a, p, t, rowsum, obar, full_table, comm, live, distinct = saved
    dev, d = g.device, table.dim
    B, n = idx.numel(), table.n
    g = g.contiguous()
    scale = (1.0 / B) if mean else 1.0
    f = dict(device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        s = _stream(g)
        g1, g2, gt = e1.grad_ptr(), e2.grad_ptr(), table.grad_ptr()
        gt_stride, local_dt = table.grad_stride, None
        if comm is not None and gt is not None:
            # own rows' dense gradient goes to a compact block that is all-gathered and added to the sink
            local_dt = torch.zeros(comm.side_block(full_table.n), d, **f)
            gt, gt_stride = local_dt.data_ptr(), d
        if (g1 is not None or g2 is not None) and not distinct and deterministic():
            _nce_bwd_rows_ordered(saved, g, g1, g2, scale, s)
        elif live is not None and (g1 is not None or g2 is not None):        # rows b < live only, mean over live
            check(lib.ssl_nce_bwd_rows_live(a.hat.data_ptr(), p.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), p.rinv.data_ptr(),
                                            idx.data_ptr(), B, live.data_ptr(), d, tau, g.data_ptr(), 1.0, g1, e1.grad_stride, g2, e2.grad_stride, s),
                  'ssl_nce_bwd_rows_live')
        elif g1 is not None or g2 is not None:
            check(lib.ssl_nce_bwd_rows(a.hat.data_ptr(), p.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), p.rinv.data_ptr(),
                                       idx.data_ptr(), B, d, tau, g.data_ptr(), scale, g1, e1.grad_stride, g2, e2.grad_stride, s),
                  'ssl_nce_bwd_rows')
        if gt is not None and n > 0:
            colscale = torch.zeros(a.npad, **f)   # padded tail is read (then masked) by the tile loads
            if live is not None:          # 0 past the live anchors
                check(lib.ssl_nce_colscale_live(rowsum.data_ptr(), B, live.data_ptr(), g.data_ptr(), 1.0, colscale.data_ptr(), s),
                      'ssl_nce_colscale_live')
            else:
                check(lib.ssl_nce_colscale(rowsum.data_ptr(), B, g.data_ptr(), scale, colscale.data_ptr(), s), 'ssl_nce_colscale')
            n_split = _n_split(t, a)
            dt_part = torch.empty(n_split, n, d, **f)
            _contract(t, a, colscale, LOG2E / tau, n_split, None, dt_part, s, live, LIVE_COLS)
            check(lib.ssl_nce_bwd_table(dt_part.data_ptr(), n_split, t.hat.data_ptr(), t.rinv.data_ptr(), n, d, gt,
                                        gt_stride, 1, s), 'ssl_nce_bwd_table')
        if local_dt is not None:
            dense = comm.allgather_side(local_dt, full_table.n)
            full_table.grad_dense().add_(dense)


class _InfoNceFn(torch.autograd.Function):
    """One InfoNCE term: rows e1[idx], e2[idx2] against all rows of ``table`` (loss_utils.py:30-39,
    and :42-51 with norm_mode 1 / mean reduction / deno_eps)."""

    @staticmethod
    def forward(ctx, e1: Rows, e2: Rows, table: Rows, idx, idx2, tau, norm_mode, mean, deno_eps, *tokens):
        out, ctx.saved_pack = _nce_fwd(e1, e2, table, idx, idx2, tau, norm_mode, mean, deno_eps)
        ctx.nt = len(tokens)
        return out

    @staticmethod
    def backward(ctx, g):
        _nce_bwd(ctx.saved_pack, g)
        zero = torch.zeros((), device=g.device)
        return (None,) * 9 + (zero,) * ctx.nt


def infonce_loss_sum(e1: Rows, e2: Rows, table: Rows, idx, temp: float, idx2=None) -> torch.Tensor:
    """cal_infonce_loss on row references: sum_b [-(e1^.e2^)/temp + log sum_j exp(e1^.table^_j/temp)]."""
    dev = table.base.device
    idx = _i64(idx, dev)
    idx2 = idx if idx2 is None else _i64(idx2, dev)
    return _InfoNceFn.apply(e1, e2, table, idx, idx2, float(temp), 0, False, 0.0, *_tokens(e1, e2, table))


# ---- LightGCL: log-sum-exp of raw (un-normalised) rows against a raw table (lightgcl.py:112-113) -------------

class _DenseLseFn(torch.autograd.Function):
    """mean_b log(sum_j exp(a_b . t_j / temp) + eps) for dense a [B, d], t [n, d] (both receive gradients), without the
    [B, n] logits: forward = the contraction with R = a log2e / temp, C = t; backward w.r.t. a is its O output, w.r.t. t
    the swapped contraction.  No running max, as in the reference."""

    @staticmethod
    def forward(ctx, a, t, temp, eps):
        _require_cuda(a, 'anchors')
        _require_cuda(t, 'table')
        a, t = a.detach().contiguous().float(), t.detach().contiguous().float()
        (B, d), n = a.shape, t.shape[0]
        kind = contraction_kind(d, 0.0, raw=True)
        f = dict(device=a.device, dtype=torch.float32)
        rowsum, obar, loss_b, out = torch.empty(B, **f), torch.empty(B, d, **f), torch.empty(B, **f), torch.empty((), **f)
        with torch.cuda.device(a.device):
            s = _stream(a)
            # raw rows (norm_mode 3) with the copies of either role: a and t swap roles in the backward
            A = _operand(Rows.constant(a), None, 3, LOG2E / temp, s, kind, streamed=True, npad=max(64, ceil_to(B, 64)))
            T = _operand(Rows.constant(t), None, 3, 1.0, s, kind, streamed=True, npad=max(64, ceil_to(n, 64)))
            n_split = _n_split(A, T)
            rs_part, o_part = torch.zeros(n_split, B, **f), torch.zeros(n_split, B, d, **f)
            _contract(A, T, None, 0.0, n_split, rs_part, o_part, s)
            check(lib.ssl_lse_finalize(rs_part.data_ptr(), o_part.data_ptr(), n_split, B, d, eps, rowsum.data_ptr(), obar.data_ptr(),
                                       loss_b.data_ptr(), s), 'ssl_lse_finalize')
            check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0 / B, out.data_ptr(), s), 'ssl_sum')
        ctx.pack = (A, T, B, n, d, temp, rowsum, obar)
        return out

    @staticmethod
    def backward(ctx, g):
        A, T, B, n, d, temp, rowsum, obar = ctx.pack
        g = g.contiguous()
        ga = gt = None
        if ctx.needs_input_grad[0]:
            ga = obar * (g * (1.0 / (B * temp)))                 # d/da_b = softmax-weighted table average / (B temp)
        if ctx.needs_input_grad[1]:
            f = dict(device=g.device, dtype=torch.float32)
            colscale = torch.zeros(A.npad, **f)
            n_split = _n_split(T, A)
            dt_part = torch.empty(n_split, n, d, **f)
            with torch.cuda.device(g.device):
                s = _stream(g)
                check(lib.ssl_nce_colscale(rowsum.data_ptr(), B, g.data_ptr(), 1.0 / B, colscale.data_ptr(), s), 'ssl_nce_colscale')
                _contract(T, A, colscale, 0.0, n_split, None, dt_part, s)
            gt = dt_part[0] if n_split == 1 else dt_part.sum(0)
        return ga, gt, None, None


def dense_logsumexp_mean(a: torch.Tensor, table: torch.Tensor, temp: float, eps: float = 1e-8) -> torch.Tensor:
    return _DenseLseFn.apply(a, table, float(temp), float(eps))


# ---- DirectAU: alignment / uniformity on unit rows (loss_utils.py:75-86) -----------------------------------

def _align_fwd(x: Rows, y: Rows, ix, iy):
    """alignment(x, y, alpha=2) = mean_b |x^_b - y^_b|^2 (loss_utils.py:75-79)."""
    dev, d, B = x.base.device, x.dim, ix.numel()
    loss_b, out = torch.empty(B, device=dev), torch.empty((), device=dev)
    with torch.cuda.device(dev):
        s = _stream(x.base)
        # F.normalize (norm_mode 2): hat and rinv, the FFMA kernel's resident operand
        xo, yo = _operand(x, ix, 2, 1.0, s, 'ffma'), _operand(y, iy, 2, 1.0, s, 'ffma')
        xh, yh, rx, ry = xo.hat, yo.hat, xo.rinv, yo.rinv
        check(lib.ssl_align_fwd(xh.data_ptr(), yh.data_ptr(), B, d, loss_b.data_ptr(), s), 'ssl_align_fwd')
        check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0 / B, out.data_ptr(), s), 'ssl_sum')
    return out, (x, y, ix, iy, xh, yh, rx, ry)


def _align_bwd(pack, g, distinct: bool = False):
    """``distinct``: see ``_bpr_bwd``.  Ordered: x's and y's positions are one block each of a stage (one scatter when they
    address the same sink)."""
    x, y, ix, iy, xh, yh, rx, ry = pack
    B, d = ix.numel(), x.dim
    g = g.contiguous()
    c = 2.0 / B                                                # d/dx^ mean |x^ - y^|^2 = 2 (x^ - y^) / B
    sides = [(rows, idx, a, b, ri) for (rows, idx, a, b, ri) in ((x, ix, xh, yh, rx), (y, iy, yh, xh, ry)) if rows.grad_ptr() is not None]
    ordered = not distinct and deterministic()
    stage = _stage(len(sides) * B, d, g.device) if ordered else None
    with torch.cuda.device(g.device):
        s = _stream(g)
        for k, (rows, idx, a, b, ri) in enumerate(sides):
            out, stride, ids = (stage[k * B:].data_ptr(), d, None) if ordered else (rows.grad_ptr(), rows.grad_stride, idx.data_ptr())
            check(lib.ssl_unit_rows_bwd(a.data_ptr(), ri.data_ptr(), ids, B, d, a.data_ptr(), c, b.data_ptr(), -c,
                                        g.data_ptr(), 1.0, out, stride, s), 'ssl_unit_rows_bwd(align)')
    if ordered:
        _scatter_blocks(stage, [(idx, rows.grad_ptr(), rows.grad_stride) for rows, idx, _, _, _ in sides])


def _uniform_fwd(x: Rows, ix):
    """uniformity(x) = log mean_{i<j} exp(-2 |x^_i - x^_j|^2) (loss_utils.py:82-86): from 256 rows on, the B x B pair sum
    runs on the InfoNCE contraction kernel (R = 4 log2e x^, C = x^), never materialising pdist's B(B-1)/2 vector."""
    dev, d, B = x.base.device, x.dim, ix.numel()
    if B < 2:
        raise ValueError('uniformity needs at least 2 rows')
    f = dict(device=dev, dtype=torch.float32)
    pair_sum, w, total = torch.empty(B, **f), torch.empty(B, d, **f), torch.empty((), **f)
    with torch.cuda.device(dev):
        s = _stream(x.base)
        if B < 256:
            # The contraction's pair_sum_i = rowsum_i - e_ii cancels when the off-diagonal sum is small next to e_ii = 1
            # (B = 2-3, near-antipodal rows).  Below 256 rows the pairs are summed directly from x^_i - x^_j instead.
            c = _operand(x, ix, 2, 1.0, s, 'ffma')
            check(lib.ssl_uniform_pairs(c.hat.data_ptr(), B, d, pair_sum.data_ptr(), w.data_ptr(), s), 'ssl_uniform_pairs')
        else:
            # from 256 rows on the pair sum is >> e_ii, so removing e_ii loses little and an fp32-grade contraction suffices
            off = 4.0 * LOG2E
            kind = contraction_kind(d, off)
            r = _operand(x, ix, 2, off, s, kind)
            c = _operand(x, ix, 2, 1.0, s, kind, streamed=True)
            n_split = _n_split(r, c)
            rs_part, o_part = torch.zeros(n_split, B, **f), torch.zeros(n_split, B, d, **f)
            _contract(r, c, None, off, n_split, rs_part, o_part, s)
            check(lib.ssl_uniform_finalize(rs_part.data_ptr(), o_part.data_ptr(), n_split, B, d, r.hat.data_ptr(), c.hat.data_ptr(), off,
                                           pair_sum.data_ptr(), w.data_ptr(), s), 'ssl_uniform_finalize')
        check(lib.ssl_sum(pair_sum.data_ptr(), B, 1.0, total.data_ptr(), s), 'ssl_sum')
    out = torch.log(total / float(B * (B - 1)))                 # total counts every unordered pair twice
    return out, (x, ix, c.hat, c.rinv, w, total)


def _uniform_bwd(pack, g, distinct: bool = False):
    """``distinct``: see ``_bpr_bwd``."""
    x, ix, c, rinv, w, total = pack
    gp = x.grad_ptr()
    if gp is None:
        return
    coef = (g * 8.0 / total).contiguous()                       # d total / d x^_i = 8 sum_{j != i} e_ij x^_j
    ordered = not distinct and deterministic()
    stage = _stage(ix.numel(), x.dim, g.device) if ordered else None
    out, stride, ids = (stage.data_ptr(), x.dim, None) if ordered else (gp, x.grad_stride, ix.data_ptr())
    with torch.cuda.device(g.device):
        check(lib.ssl_unit_rows_bwd(c.data_ptr(), rinv.data_ptr(), ids, ix.numel(), x.dim, w.data_ptr(), 1.0, None, 0.0,
                                    coef.data_ptr(), 1.0, out, stride, _stream(g)), 'ssl_unit_rows_bwd(uniformity)')
    if ordered:
        scatter_rows_ordered(stage, ix, gp, x.grad_stride)


class _AlignFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Rows, y: Rows, ix, iy, *tokens):
        out, ctx.pack = _align_fwd(x, y, ix, iy)
        ctx.nt = len(tokens)
        return out

    @staticmethod
    def backward(ctx, g):
        _align_bwd(ctx.pack, g)
        return (None,) * 4 + (torch.zeros((), device=g.device),) * ctx.nt


class _UniformFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Rows, ix, *tokens):
        out, ctx.pack = _uniform_fwd(x, ix)
        ctx.nt = len(tokens)
        return out

    @staticmethod
    def backward(ctx, g):
        _uniform_bwd(ctx.pack, g)
        return (None,) * 2 + (torch.zeros((), device=g.device),) * ctx.nt


def alignment_mean(x: Rows, y: Rows, ix, iy) -> torch.Tensor:
    dev = x.base.device
    return _AlignFn.apply(x, y, _i64(ix, dev), _i64(iy, dev), *_tokens(x, y))


def uniformity_log_mean(x: Rows, ix) -> torch.Tensor:
    return _UniformFn.apply(x, _i64(ix, x.base.device), *_tokens(x))


class _DenseAlignFn(torch.autograd.Function):
    """alignment on plain dense [B, d] tensors (the reference's signature)."""

    @staticmethod
    def forward(ctx, x, y):
        ar = torch.arange(x.shape[0], device=x.device)
        rx, sx = _dense_rows(x, True)
        ry, sy = _dense_rows(y, True)
        out, ctx.pack = _align_fwd(rx, ry, ar, ar)
        ctx.sinks = (sx, sy)
        return out

    @staticmethod
    def backward(ctx, g):
        _align_bwd(ctx.pack, g, distinct=True)
        return ctx.sinks[0](), ctx.sinks[1]()


class _DenseUniformFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        rx, ctx.sink = _dense_rows(x, True)
        out, ctx.pack = _uniform_fwd(rx, torch.arange(x.shape[0], device=x.device))
        return out

    @staticmethod
    def backward(ctx, g):
        _uniform_bwd(ctx.pack, g, distinct=True)
        return ctx.sink()


# ---- the same kernels behind plain dense tensors (reference signatures; gradients are returned
# ---- as ordinary dense tensors -- used by HCCF, whose hyper-graph branch lives in torch autograd)

class _LocalSink:
    def __init__(self, like: torch.Tensor):
        self.like, self.buf = like, None

    def __call__(self):
        if self.buf is None:
            self.buf = torch.zeros_like(self.like)
        return self.buf


def _dense_rows(t: torch.Tensor, with_grad: bool):
    _require_cuda(t, 'loss input')
    t = t.detach().contiguous()
    sink = _LocalSink(t) if with_grad else None
    return Rows(t, 0, 1, 0, t.shape[0], t.shape[1], sink), sink


class _DenseBprFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anc, pos, neg):
        B = anc.shape[0]
        ar = torch.arange(B, device=anc.device)
        items = torch.cat([pos.detach(), neg.detach()], 0)
        users, su = _dense_rows(anc, True)
        items_r, si = _dense_rows(items, True)
        out, coef = _bpr_fwd(users, items_r, ar, ar, ar + B)
        ctx.pack = (users, items_r, ar, coef, su, si, B)
        return out

    @staticmethod
    def backward(ctx, g):
        users, items_r, ar, coef, su, si, B = ctx.pack
        _bpr_bwd(users, items_r, ar, ar, ar + B, coef, g, distinct=True)
        gi = si()
        return su(), gi[:B], gi[B:]


class _DenseInfoNceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e1, e2, table, idx, idx2, tau, norm_mode, mean, deno_eps, shared_table, distinct, live=None):
        ctx.n_inputs = 11 if live is None else 12
        r1, s1 = _dense_rows(e1, ctx.needs_input_grad[0])
        if shared_table:                      # e2 rows are rows of the table itself (spec_nodes)
            rt, st_ = _dense_rows(table, ctx.needs_input_grad[2])
            r2, s2 = rt, st_
        else:
            r2, s2 = _dense_rows(e2, ctx.needs_input_grad[1])
            rt, st_ = _dense_rows(table, ctx.needs_input_grad[2])
        out, ctx.saved_pack = _nce_fwd(r1, r2, rt, idx, idx2, tau, norm_mode, mean, deno_eps, live, distinct)
        ctx.sinks = (s1, s2, st_, shared_table)
        return out

    @staticmethod
    def backward(ctx, g):
        _nce_bwd(ctx.saved_pack, g)
        s1, s2, st_, shared = ctx.sinks
        g1 = s1() if s1 is not None else None
        g2 = None if shared else (s2() if s2 is not None else None)
        gt = st_() if st_ is not None else None
        return (g1, g2, gt) + (None,) * (ctx.n_inputs - 3)


def dense_bpr_loss_sum(anc, pos, neg):
    return _DenseBprFn.apply(anc, pos, neg)


def dense_infonce_loss_sum(e1, e2, all2, temp):
    """cal_infonce_loss(embeds1 [B,d], embeds2 [B,d], all_embeds2 [N,d], temp) -- loss_utils.py:30-39."""
    B = e1.shape[0]
    ar = torch.arange(B, device=e1.device)
    return _DenseInfoNceFn.apply(e1, e2, all2, ar, ar, float(temp), 0, False, 0.0, False, True)


def dense_infonce_spec_nodes_mean(embeds1, embeds2, nodes, temp):
    """cal_infonce_loss_spec_nodes(embeds1 [N,d], embeds2 [N,d], nodes, temp) -- loss_utils.py:42-51."""
    nodes = _i64(nodes, embeds2.device)
    return _DenseInfoNceFn.apply(embeds1, embeds2, embeds2, nodes, nodes, float(temp), 1, True, 1e-8, True, False)


def unique_ids(idx: torch.Tensor, n_range: int):
    """torch.unique(idx, sorted=True) without a host sync or a data-dependent shape: -> (out int64 [n], count int64 device
    scalar); out[:count] are the distinct ids ascending, out[count:] repeat the largest one.  Every id must be in [0, n_range)."""
    dev = idx.device
    idx = _i64(idx, dev).contiguous()
    words = C.c_int64()
    check(lib.ssl_unique_ids_scratch(int(n_range), C.byref(words)), 'ssl_unique_ids_scratch')
    scratch = torch.empty(words.value, dtype=torch.int32, device=dev)
    out = torch.empty_like(idx)
    count = torch.empty((), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssl_unique_ids(idx.data_ptr(), idx.numel(), int(n_range), scratch.data_ptr(), words.value, out.data_ptr(),
                                 count.data_ptr(), _stream(idx)), 'ssl_unique_ids')
    return out, count


def row_bitmap(n_rows: int, device, *index_lists) -> torch.Tensor:
    """uint32 bitmap over [0, n_rows) marking every id of ``index_lists`` (pairs (ids, offset): marks ids + offset), built on
    ``device`` with no host read (``ssl_row_bitmap``): ``ViewSpec.row_bits`` of a view the losses read at batch rows only."""
    dev = torch.device(device)
    idx = torch.cat([_i64(ids, dev).reshape(-1) + int(off) for ids, off in index_lists])
    n_words = (int(n_rows) + 31) // 32
    bits = torch.empty(n_words, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssl_row_bitmap(idx.data_ptr(), idx.numel(), int(n_rows), bits.data_ptr(), n_words, _stream(idx)), 'ssl_row_bitmap')
    return bits


def dense_infonce_spec_nodes_mean_dev(embeds1, embeds2, ids, temp):
    """The graph-safe form of ``dense_infonce_spec_nodes_mean(embeds1, embeds2, torch.unique(ids), temp)``: the unique ids are
    found on the device (``unique_ids``), the term runs over the padded list at capacity ids.numel() and every piece is bounded
    by the device count -- no host read, no data-dependent shape, so a CUDA graph can capture it."""
    nodes, count = unique_ids(ids, embeds2.shape[0])
    return _DenseInfoNceFn.apply(embeds1, embeds2, embeds2, nodes, nodes, float(temp), 1, True, 1e-8, True, False, count)


# ---- negative sampling of the BPR models (optional keys train.dns_candidates, mixgcf, ssm_temperature, neg_popularity) -------

_SHARED_SEED = 'data-parallel ranks share the seed, so their candidate draws would coincide'
# why each key is single-GPU: (for a row-sharded model, for data-parallel gradient sync)
_SINGLE_GPU = {
    'dns_candidates': ('a row-sharded model does not select hard negatives', _SHARED_SEED),
    'mixgcf': ('a row-sharded model does not mix negatives', 'data-parallel ranks share the seed, so their mixing weights would coincide'),
    'ssm_temperature': ('a row-sharded model does not score sampled candidates', _SHARED_SEED),
    'neg_popularity': ('a row-sharded model does not draw candidates', _SHARED_SEED),
    'ssm_in_batch': ("a row-sharded model does not contract the batch's items",
                     'each rank would contract only its share of the batch, so N ranks would not equal one step at N times the batch'),
}


@dataclass(frozen=True)
class NegSpec:
    """The negative-sampling keys of the train section (INTEGRATION §2); the only reader of them.
    ``candidates`` (train.dns_candidates): M, the candidates per BPR pair, an integer in [1, 256]; 1 (the default) is the plain
    step, >= 2 trains each pair on the highest-scored of M (``neg_candidates``, ``hard_negatives``).
    ``mixgcf`` (train.mixgcf): True replaces the BPR term's negative by MixGCF's mixed negative (``mixgcf_bpr_sum``).
    ``ssm_temperature`` (train.ssm_temperature): tau, a finite number > 0 (int or float, not a bool), replaces the BPR term by
    the sampled softmax loss on cosine scores over tau (``ssm_loss_sum``).
    ``popularity`` (train.neg_popularity): beta, a number in [0, 1] (int or float, not a bool); the candidates 1 .. M-1 are then
    drawn in proportion to (deg_i + 1)^beta (``pop_tables``), and the sampled softmax takes their logQ correction.
    ``in_batch`` (train.ssm_in_batch): True scores every pair of the sampled softmax against the batch's 2B items (its
    positives and loader negatives) with the weights of ``in_batch_weights`` instead of drawn candidates (``ssm_in_batch_sum``).
    The two numbers are None when absent or null (the default)."""
    candidates: int = 1
    mixgcf: bool = False
    ssm_temperature: Optional[float] = None
    popularity: Optional[float] = None
    in_batch: bool = False

    @classmethod
    def from_config(cls) -> 'NegSpec':
        """The keys of ``configs['train']``, each checked on its own: ValueError outside its domain (tau's is checked in fp32)."""
        from .config import configs
        t = configs.get('train', {})
        m = t.get('dns_candidates', 1)
        if isinstance(m, bool) or not isinstance(m, int) or not 1 <= m <= _lib.MAX_CANDIDATES:
            raise ValueError(f'train.dns_candidates must be an integer in [1, {_lib.MAX_CANDIDATES}], got {m!r}')
        on = t.get('mixgcf', False)
        if not isinstance(on, bool):
            raise ValueError(f'train.mixgcf must be true or false, got {on!r}')
        tau = t.get('ssm_temperature')
        if tau is not None and (isinstance(tau, bool) or not isinstance(tau, (int, float)) or not 0.0 < C.c_float(tau).value < math.inf):
            raise ValueError(f'train.ssm_temperature must be a finite number > 0 or null, got {tau!r}')
        beta = t.get('neg_popularity')
        if beta is not None and (isinstance(beta, bool) or not isinstance(beta, (int, float)) or not 0.0 <= beta <= 1.0):
            raise ValueError(f'train.neg_popularity must be a number in [0, 1] or null, got {beta!r}')
        ib = t.get('ssm_in_batch', False)
        if not isinstance(ib, bool):
            raise ValueError(f'train.ssm_in_batch must be true or false, got {ib!r}')
        return cls(m, on, None if tau is None else float(tau), None if beta is None else float(beta), ib)

    def record(self) -> dict:
        """The keys that are set, under their config names and in the order above: what a training checkpoint records.  A key
        is set when M > 1, MixGCF is on or a number is given, so a run without any of them keeps the record it had before."""
        rec = {}
        if self.candidates > 1:
            rec['dns_candidates'] = self.candidates
        if self.mixgcf:
            rec['mixgcf'] = True
        if self.ssm_temperature is not None:
            rec['ssm_temperature'] = self.ssm_temperature
        if self.popularity is not None:
            rec['neg_popularity'] = self.popularity
        if self.in_batch:
            rec['ssm_in_batch'] = True
        return rec

    def refuse_multi_gpu(self, sharded: bool) -> None:
        """Raise ValueError naming the first set key (train.ssm_in_batch before the others, whose reasons it does not share):
        every key is single-GPU, for a row-sharded model (``sharded``) and for data-parallel gradient sync alike."""
        key = 'ssm_in_batch' if self.in_batch else next(iter(self.record()), None)
        if key is not None:
            raise ValueError(f'train.{key} is single-GPU: {_SINGLE_GPU[key][0 if sharded else 1]}')

    def check_model(self, model) -> None:
        """The rules that involve the model or two keys, in this order: a model without a BPR term (``bpr_negatives`` False)
        takes none of the keys; MixGCF mixes at most MIXGCF_MAX_LAYERS layers; the sampled softmax and MixGCF both replace the
        BPR term; the popularity draw needs M >= 2; the in-batch softmax needs the sampled softmax and draws no candidates."""
        key = next(iter(self.record()), None)
        if key is not None and not model.bpr_negatives:
            raise ValueError(f'train.{key}: {type(model).__name__} trains without negatives')
        if self.mixgcf and getattr(model, 'layer_num', 0) + 1 > MIXGCF_MAX_LAYERS:
            raise ValueError(f'train.mixgcf mixes at most {MIXGCF_MAX_LAYERS} layers (layer_num + 1), got {model.layer_num + 1}')
        if self.ssm_temperature is not None and self.mixgcf:
            raise ValueError('train.ssm_temperature and train.mixgcf both replace the BPR term: set one of them')
        if self.popularity is not None and self.candidates < 2:
            raise ValueError('train.neg_popularity draws the candidates of train.dns_candidates, which must then be >= 2, '
                             f'got {self.candidates}')
        if self.in_batch and self.ssm_temperature is None:
            raise ValueError('train.ssm_in_batch is a form of the sampled softmax: it needs train.ssm_temperature')
        if self.in_batch and self.candidates > 1:
            raise ValueError("train.ssm_in_batch scores the batch's own items, so the candidates of train.dns_candidates would be "
                             f'drawn and never read: it must be 1, got {self.candidates}')


def neg_candidates(users, negs, m: int, trn_rowptr: torch.Tensor, trn_cols: torch.Tensor, n_item: int, seed, pop=None,
                   want_bias: bool = False):
    """[B, m] int64 negative candidates of the pairs (users[b], ., negs[b]) (``ssl_neg_candidates``): column 0 is ``negs``, the
    others are drawn uniformly over the items, rejecting the user's training positives (int32 CSR, sorted rows).  A
    :class:`DevSeed` passes its device word, so a captured step draws with the seed written there before each replay.

    ``pop``: a :class:`PopTables` of the same training CSR draws columns 1 .. m-1 in proportion to the item weights instead
    (``ssl_neg_candidates_pop``, train.neg_popularity); ``want_bias`` then also returns the [B, m] fp32 logQ correction
    ln(M q_j(c_j)) of every candidate (include/sslrec_b200.h, a27) as ``(cands, bias)``."""
    dev = trn_cols.device
    users, negs = _i64(users, dev), _i64(negs, dev)
    if negs.numel() != users.numel():
        raise RuntimeError('sslrec_b200: one negative per user')
    if want_bias and pop is None:
        raise RuntimeError('sslrec_b200: the logQ correction needs popularity tables')
    cands = torch.empty(users.numel(), int(m), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        if pop is None:
            check(lib.ssl_neg_candidates(users.data_ptr(), negs.data_ptr(), users.numel(), int(m), trn_rowptr.data_ptr(),
                                         trn_cols.data_ptr(), int(n_item), int(seed), getattr(seed, 'ptr', 0) or None, cands.data_ptr(),
                                         _stream(cands)), 'ssl_neg_candidates')
            return cands
        if pop.n_item != int(n_item) or pop.table.device != dev:
            raise RuntimeError('sslrec_b200: the popularity tables belong to another item set or device')
        bias = torch.empty(users.numel(), int(m), dtype=torch.float32, device=dev) if want_bias else None
        check(lib.ssl_neg_candidates_pop(users.data_ptr(), negs.data_ptr(), users.numel(), int(m), trn_rowptr.data_ptr(),
                                         trn_cols.data_ptr(), int(n_item), pop.table.data_ptr(), pop.lp.data_ptr(), pop.lz_pop.data_ptr(),
                                         pop.lz_uni.data_ptr(), float(np.float32(math.log(int(m)))), int(seed),
                                         getattr(seed, 'ptr', 0) or None, cands.data_ptr(), _ptr(bias), _stream(cands)),
              'ssl_neg_candidates_pop')
    return (cands, bias) if want_bias else cands


# ---- popularity-proportional candidates (optional key train.neg_popularity) --------------------------------------------------

def pop_tables(indptr, indices, n_item: int, beta: float) -> dict:
    """The host tables of the popularity draw (include/sslrec_b200.h, a27) from a training CSR with sorted, distinct columns per
    row (numpy, float64 and exact integers; a pure function of its arguments):

    ``V`` [n_item] int64: V_i >= 1, the largest-remainder rounding of x_i = n_item 2^32 w_i / sum w, w_i = (deg_i + 1)^beta,
    deg_i the count of item i in ``indices`` (x_i = (w_i * n_item 2^32) / fsum(w) in float64; the units short of n_item 2^32
    after the floors go to the largest remainders x_i - floor(x_i), ties to the lower item; a surplus from float64 rounding
    comes off the smallest remainders the same way), so sum V = n_item 2^32 exactly.
    ``table`` [n_item, 2] uint32 {thr, alias}: Walker / Vose on V in integers with column capacity 2^32.  Columns start as
    ``small`` (V < 2^32) and ``large`` (V >= 2^32) stacks in ascending item order; while both are non-empty the top small item
    s fills its column's share thr = r_s and its alias is the top large item l, whose rest r_l -= 2^32 - r_s moves it to small
    when below 2^32.  Every item left over then has r = 2^32 exactly: its column is itself alone (alias = itself, thr = 0).
    ``lp`` [n_item], ``lz_pop`` / ``lz_uni`` [n_user] float32: log(V_i / T), log((T - sum_{i in P_u} V_i) / T) and
    log(n_item - deg_u), T = n_item 2^32, in float64 rounded once; 0 for a user who has every item."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    n = int(n_item)
    if n < 1 or n >= 1 << 31:
        raise ValueError(f'pop_tables: n_item {n} outside [1, 2^31)')
    K = 1 << 32
    T = n * K
    deg = np.bincount(indices, minlength=n).astype(np.float64)
    w = (deg + 1.0) ** float(beta)
    x = (w * float(T)) / math.fsum(w.tolist())
    fl = np.floor(x)
    V = fl.astype(np.int64)
    short = T - int(V.sum())
    rem = x - fl
    if short > 0:          # the largest remainders, ties to the lower item (a stable sort of -rem); more than n: whole rounds
        V += short // n
        V[np.argsort(-rem, kind='stable')[:short % n]] += 1
    elif short < 0:
        V[np.argsort(rem, kind='stable')[:-short]] -= 1
    if int(V.sum()) != T or int(V.min()) < 1:
        raise ValueError('pop_tables: the weights do not round to positive integers summing to n_item 2^32')
    thr = np.zeros(n, dtype=np.uint32)
    alias = np.arange(n, dtype=np.uint32)
    r = V.tolist()
    small = [i for i in range(n) if r[i] < K][::-1]          # stacks: the top (last element) is the lowest item
    large = [i for i in range(n) if r[i] >= K][::-1]
    while small and large:
        s, l = small.pop(), large.pop()
        thr[s] = r[s]
        alias[s] = l
        r[l] -= K - r[s]
        (small if r[l] < K else large).append(l)
    if small:                                                # impossible with sum V = n 2^32; kept as a guard
        raise ValueError('pop_tables: the alias construction did not close')
    with np.errstate(divide='ignore'):
        lp = np.log(V.astype(np.float64) / float(T))
        # sum of V over each user's row, in integers (np.add.reduceat misreads empty rows)
        cs = np.concatenate([[0], np.cumsum(V[indices])])
        left = T - (cs[indptr[1:]] - cs[indptr[:-1]])
        lz_pop = np.where(left > 0, np.log(np.maximum(left, 1).astype(np.float64) / float(T)), 0.0)
        free = n - np.diff(indptr)
        lz_uni = np.where(free > 0, np.log(np.maximum(free, 1).astype(np.float64)), 0.0)
    return {'V': V, 'table': np.stack([thr, alias], 1), 'lp': lp.astype(np.float32), 'lz_pop': lz_pop.astype(np.float32),
            'lz_uni': lz_uni.astype(np.float32)}


class PopTables:
    """``pop_tables`` on a device: the alias table (int32 [n_item, 2], the uint32 bits of {thr, alias}) and the fp32 ``lp``,
    ``lz_pop`` and ``lz_uni`` that ``neg_candidates(pop=...)`` reads."""

    def __init__(self, indptr, indices, n_item: int, beta: float, device):
        h = pop_tables(indptr, indices, n_item, beta)
        self.n_item, self.beta = int(n_item), float(beta)
        self.table = torch.from_numpy(np.ascontiguousarray(h['table']).view(np.int32)).to(device)
        self.lp, self.lz_pop, self.lz_uni = (torch.from_numpy(h[k]).to(device) for k in ('lp', 'lz_pop', 'lz_uni'))


def _score_table(t):
    """Rows or a [n, d] fp32 tensor with unit column stride -> (pointer of row 0, row stride, dim)."""
    if isinstance(t, Rows):
        return t.ptr, t.stride, t.dim
    _require_cuda(t, 'score table')
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError('sslrec_b200: a score table must be [n, d] with unit column stride')
    return t.data_ptr(), t.stride(0), t.shape[1]


def hard_negatives(users, items, ancs, cands: torch.Tensor) -> torch.Tensor:
    """[B] int64: for every pair b the candidate cands[b, j] whose score users[ancs[b]] . items[cands[b, j]] is largest
    (``ssl_neg_select``: one sequential fp32 FMA chain per score, ties to the lowest j, NaN never wins).  ``users`` / ``items``
    are :class:`Rows` (a restricted view must mark every candidate row) or [n, d] tensors; no gradient flows through it."""
    u_ptr, u_stride, d = _score_table(users)
    i_ptr, i_stride, d_i = _score_table(items)
    if d_i != d:
        raise RuntimeError('sslrec_b200: user and item rows differ in width')
    dev = cands.device
    ancs, cands = _i64(ancs, dev), _i64(cands, dev)
    B, m = cands.shape
    if ancs.numel() != B:
        raise RuntimeError('sslrec_b200: one anchor per row of candidates')
    out = torch.empty(B, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssl_neg_select(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), cands.data_ptr(), B, m, d, out.data_ptr(), _stream(out)),
              'ssl_neg_select')
    return out


# ---- MixGCF negatives (optional key train.mixgcf) ----------------------------------------------------------------------------

MIXGCF_MAX_LAYERS = 8


def _mix_grad_target(op, plain_grads: dict):
    """Where an operand's gradient goes: a Rows' sink, or the zeroed gradient of a plain tensor (one per distinct tensor)."""
    if isinstance(op, Rows):
        return op.grad_ptr(), op.grad_stride
    k, t = op
    if k not in plain_grads:
        plain_grads[k] = torch.zeros(t.shape, device=t.device, dtype=torch.float32)
    return plain_grads[k].data_ptr(), t.shape[1]


def _mix_table(op):
    return _score_table(op if isinstance(op, Rows) else op[1])


def _scatter_grouped(parts) -> None:
    """Ordered scatter of (stage, ids, sink pointer, sink stride) parts.  Parts that address the same sink (pointer and stride) are
    ONE scatter over their concatenated positions, in part order; the groups run in the order of their first part."""
    groups: Dict[tuple, list] = {}
    for stage, ids, ptr, stride in parts:
        groups.setdefault((ptr, stride), []).append((stage, ids))
    for (ptr, stride), ps in groups.items():
        if len(ps) == 1:
            scatter_rows_ordered(ps[0][0], ps[0][1], ptr, stride)
        else:
            scatter_rows_ordered(torch.cat([s for s, _ in ps]), torch.cat([i for _, i in ps]), ptr, stride)


class _MixgcfFn(torch.autograd.Function):
    """MixGCF's BPR term (``ssl_mixgcf_bpr_fwd`` / ``_bwd``).  Operands are Rows (gradients into their sinks, autograd sees their
    tokens) or (index, tensor) of the plain tensors passed after ``pack`` (gradients into zeroed tensors returned to autograd)."""

    @staticmethod
    def forward(ctx, pack, *inputs):
        ops, ancs, poss, cands, seed, alpha_in, n_plain = pack
        users, items, layers = ops[0], ops[1], ops[2:]
        u_ptr, u_stride, d = _mix_table(users)
        i_ptr, i_stride, d_i = _mix_table(items)
        tabs = [_mix_table(op) for op in layers]
        if d_i != d or any(t[2] != d for t in tabs):
            raise RuntimeError('sslrec_b200: the user, item and layer rows of a MixGCF term differ in width')
        dev = cands.device
        B, m = cands.shape
        L1 = len(layers)
        f = dict(device=dev, dtype=torch.float32)
        loss_b, coef, out = torch.empty(B, **f), torch.empty(B, **f), torch.empty((), **f)
        picks = torch.empty(B, L1, dtype=torch.int64, device=dev)
        alpha, nhat = torch.empty(B, L1, **f), torch.empty(B, d, **f)
        lp = (C.c_void_p * L1)(*[t[0] for t in tabs])
        ls = (C.c_int64 * L1)(*[t[1] for t in tabs])
        with torch.cuda.device(dev), _timed('mixgcf_fwd', dict(B=B, M=m, layers=L1, dim=d)):
            s = _stream(cands)
            check(lib.ssl_mixgcf_bpr_fwd(u_ptr, u_stride, i_ptr, i_stride, lp, ls, L1, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(),
                                         B, m, d, int(seed), getattr(seed, 'ptr', 0) or None, _ptr(alpha_in), loss_b.data_ptr(),
                                         coef.data_ptr(), picks.data_ptr(), alpha.data_ptr(), nhat.data_ptr(), s), 'ssl_mixgcf_bpr_fwd')
            check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0, out.data_ptr(), s), 'ssl_sum')
        ctx.pack = (ops, ancs, poss, picks, alpha, nhat, coef, n_plain, len(inputs) - n_plain)
        ctx.mark_non_differentiable(picks, alpha)
        return out, picks, alpha

    @staticmethod
    def backward(ctx, g, _g_picks, _g_alpha):
        ops, ancs, poss, picks, alpha, nhat, coef, n_plain, n_tokens = ctx.pack
        g = g.contiguous()
        users, items, layers = ops[0], ops[1], ops[2:]
        B, L1 = picks.shape
        d = nhat.shape[1]
        plain_grads: dict = {}
        targets = [_mix_grad_target(op, plain_grads) for op in ops]
        if any(p is None for p, _ in targets):
            raise RuntimeError('sslrec_b200: every operand of a MixGCF term must take a gradient')
        (gu, gu_s), (gi, gi_s), gl = targets[0], targets[1], targets[2:]
        dev = g.device
        with torch.cuda.device(dev), _timed('mixgcf_bwd', dict(B=B, layers=L1, dim=d)):
            s = _stream(g)
            if deterministic():
                # identity ids on gathered rows into -0.0 stages (positions: csrc/mixgcf.cuh), then the ordered scatters
                ug = _gather_rows(users, ancs)
                pg = _gather_rows(items, poss)
                ar = torch.arange(B, device=dev)
                ids = (ar + B).unsqueeze(1).expand(B, L1).contiguous()
                stage = _stage((2 + 2 * L1) * B, d, dev)
                su, si = stage[:B], stage[B:2 * B]
                sl = [stage[(2 + 2 * l) * B:(4 + 2 * l) * B] for l in range(L1)]
                lp = (C.c_void_p * L1)(*[t.data_ptr() for t in sl])
                ls = (C.c_int64 * L1)(*([d] * L1))
                check(lib.ssl_mixgcf_bpr_bwd(ug.data_ptr(), d, pg.data_ptr(), d, ar.data_ptr(), ar.data_ptr(), ids.data_ptr(), B, L1, d,
                                             nhat.data_ptr(), alpha.data_ptr(), coef.data_ptr(), g.data_ptr(), 1.0, su.data_ptr(), d,
                                             si.data_ptr(), d, lp, ls, s), 'ssl_mixgcf_bpr_bwd')
                parts = [(su, ancs, gu, gu_s), (si, poss, gi, gi_s)]
                parts += [(sl[l], torch.cat([poss, picks[:, l]]), p, st) for l, (p, st) in enumerate(gl)]
                _scatter_grouped(parts)
            else:
                u_ptr, u_stride, _ = _mix_table(users)
                i_ptr, i_stride, _ = _mix_table(items)
                lp = (C.c_void_p * L1)(*[p for p, _ in gl])
                ls = (C.c_int64 * L1)(*[st for _, st in gl])
                check(lib.ssl_mixgcf_bpr_bwd(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), picks.data_ptr(), B, L1, d,
                                             nhat.data_ptr(), alpha.data_ptr(), coef.data_ptr(), g.data_ptr(), 1.0, gu, gu_s, gi, gi_s,
                                             lp, ls, s), 'ssl_mixgcf_bpr_bwd')
        zero = torch.zeros((), device=dev)
        return (None,) + tuple(plain_grads[k] for k in range(n_plain)) + (zero,) * n_tokens


def _gather_rows(op, ids: torch.Tensor) -> torch.Tensor:
    """The rows ``ids`` of a MixGCF operand as a contiguous [len(ids), d] tensor."""
    return op.take(ids) if isinstance(op, Rows) else op[1].index_select(0, ids)


def mixgcf_bpr_sum(users, items, item_layers, ancs, poss, cands: torch.Tensor, seed, alpha=None):
    """MixGCF's BPR term summed over the batch (``ssl_mixgcf_bpr_fwd``; formula in include/sslrec_b200.h, a25) -> (loss, picks
    [B, L+1] int64, alpha [B, L+1] fp32).  ``users`` / ``items`` are the summed table the BPR term reads, ``item_layers`` the item
    rows of its layers 0 .. L (layer 0 = E0), ``cands`` [B, M] the candidates (column 0 the loader's negative).  Each table is a
    :class:`Rows` (gradient into its sink) or a [n, d] fp32 tensor (gradient through autograd, like ``rows_at``); under
    ``deterministic()`` every batch row's gradient is added in position order.  The alpha draw is keyed by ``seed`` (a
    :class:`DevSeed` passes its device word); ``alpha`` [B, L+1] fp32 injects the mixing weights instead."""
    layers = list(item_layers)
    if not 1 <= len(layers) <= MIXGCF_MAX_LAYERS:
        raise ValueError(f'MixGCF mixes 1 .. {MIXGCF_MAX_LAYERS} layers, got {len(layers)}')
    dev = cands.device
    ancs, poss, cands = _i64(ancs, dev), _i64(poss, dev), _i64(cands, dev)
    if cands.dim() != 2 or ancs.numel() != cands.shape[0] or poss.numel() != cands.shape[0]:
        raise RuntimeError('sslrec_b200: one anchor, one positive and one row of candidates per pair')
    if alpha is not None:
        alpha = alpha.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(alpha.shape) != (cands.shape[0], len(layers)):
            raise RuntimeError('sslrec_b200: injected alpha must be [B, L+1]')
    ops, plain = _mix_operands([users, items] + layers)
    pack = (ops, ancs, poss, cands, seed, alpha, len(plain))
    return _MixgcfFn.apply(pack, *plain, *_tokens(*[op for op in ops if isinstance(op, Rows)]))


def _mix_operands(tables):
    """-> (ops, plain): each table as an operand of ``_MixgcfFn`` / ``_SsmFn`` -- a Rows as it is, a plain tensor as (index,
    detached tensor) into ``plain``, the distinct plain tensors (one gradient per distinct tensor)."""
    plain: List[torch.Tensor] = []
    ops = []
    for t in tables:
        if isinstance(t, Rows):
            ops.append(t)
            continue
        k = next((i for i, q in enumerate(plain) if q is t), None)
        if k is None:
            plain.append(t)
            k = len(plain) - 1
        ops.append((k, t.detach()))
    return ops, plain


# ---- sampled softmax loss (optional key train.ssm_temperature) ---------------------------------------------------------------

class _SsmFn(torch.autograd.Function):
    """The sampled softmax term (``ssl_ssm_fwd`` / ``_bwd``).  Operands as in ``_MixgcfFn``: Rows (gradients into their sinks,
    autograd sees their tokens) or (index, tensor) of the plain tensors passed after ``pack``."""

    @staticmethod
    def forward(ctx, pack, *inputs):
        ops, ancs, poss, cands, tau, bias, n_plain = pack
        users, items = ops
        u_ptr, u_stride, d = _mix_table(users)
        i_ptr, i_stride, d_i = _mix_table(items)
        if d_i != d:
            raise RuntimeError('sslrec_b200: the user and item rows of a sampled softmax term differ in width')
        dev = cands.device
        B, m = cands.shape
        f = dict(device=dev, dtype=torch.float32)
        loss_b, out = torch.empty(B, **f), torch.empty((), **f)
        s, w, nrm = torch.empty(B, m + 1, **f), torch.empty(B, m + 1, **f), torch.empty(B, m + 2, **f)
        with torch.cuda.device(dev), _timed('ssm_fwd', dict(B=B, M=m, dim=d)):
            st = _stream(cands)
            if bias is None:
                check(lib.ssl_ssm_fwd(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, m, d, tau,
                                      loss_b.data_ptr(), s.data_ptr(), w.data_ptr(), nrm.data_ptr(), st), 'ssl_ssm_fwd')
            else:          # the logQ-corrected softmax; s stays raw, so the backward below is the same
                check(lib.ssl_ssm_fwd_logq(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, m, d,
                                           tau, loss_b.data_ptr(), s.data_ptr(), w.data_ptr(), nrm.data_ptr(), bias.data_ptr(), st),
                      'ssl_ssm_fwd_logq')
            check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0, out.data_ptr(), st), 'ssl_sum')
        ctx.pack = (ops, ancs, poss, cands, tau, s, w, nrm, n_plain, len(inputs) - n_plain)
        return out

    @staticmethod
    def backward(ctx, g):
        ops, ancs, poss, cands, tau, s, w, nrm, n_plain, n_tokens = ctx.pack
        g = g.contiguous()
        users, items = ops
        B, m = cands.shape
        d = _mix_table(users)[2]
        plain_grads: dict = {}
        targets = [_mix_grad_target(op, plain_grads) for op in ops]
        if any(p is None for p, _ in targets):
            raise RuntimeError('sslrec_b200: every operand of a sampled softmax term must take a gradient')
        (gu, gu_s), (gi, gi_s) = targets
        dev = g.device
        with torch.cuda.device(dev), _timed('ssm_bwd', dict(B=B, M=m, dim=d)):
            st = _stream(g)
            if deterministic():
                # identity ids on gathered rows into a -0.0 stage (positions: csrc/ssm.cuh), then the ordered scatters
                item_ids = torch.cat([poss, cands.view(-1)])
                ug, ig = _gather_rows(users, ancs), _gather_rows(items, item_ids)
                ar = torch.arange(B, device=dev)
                ci = torch.arange(B, B * (m + 1), device=dev)
                stage = _stage(B * (m + 2), d, dev)
                su, si = stage[:B], stage[B:]
                check(lib.ssl_ssm_bwd(ug.data_ptr(), d, ig.data_ptr(), d, ar.data_ptr(), ar.data_ptr(), ci.data_ptr(), B, m, d, tau,
                                      s.data_ptr(), w.data_ptr(), nrm.data_ptr(), g.data_ptr(), 1.0, su.data_ptr(), d, si.data_ptr(), d,
                                      st), 'ssl_ssm_bwd')
                _scatter_grouped([(su, ancs, gu, gu_s), (si, item_ids, gi, gi_s)])
            else:
                u_ptr, u_stride, _ = _mix_table(users)
                i_ptr, i_stride, _ = _mix_table(items)
                check(lib.ssl_ssm_bwd(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, m, d, tau,
                                      s.data_ptr(), w.data_ptr(), nrm.data_ptr(), g.data_ptr(), 1.0, gu, gu_s, gi, gi_s, st), 'ssl_ssm_bwd')
        zero = torch.zeros((), device=dev)
        return (None,) + tuple(plain_grads[k] for k in range(n_plain)) + (zero,) * n_tokens


def ssm_loss_sum(users, items, ancs, poss, cands: torch.Tensor, temp: float, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The sampled softmax loss summed over the batch (``ssl_ssm_fwd``; formula in include/sslrec_b200.h, a26): for every pair
    lse_q(s_q) - s_0 over the positive (q = 0) and the candidates ``cands`` [B, M] (column 0 the loader's negative), with
    s_q = cos(users[ancs[b]], items[c_q]) / temp.  ``users`` / ``items`` are each a :class:`Rows` (gradient into its sink; a
    restricted view must mark every candidate row) or a [n, d] fp32 tensor (gradient through autograd, like ``rows_at``); under
    ``deterministic()`` every batch row's gradient is added in position order.

    ``bias``: the [B, M] fp32 logQ correction of the candidates (``neg_candidates(pop=..., want_bias=True)``): the softmax then
    runs on s_q - bias[b, q-1] for the candidates (``ssl_ssm_fwd_logq``); no gradient flows into it."""
    dev = cands.device
    ancs, poss, cands = _i64(ancs, dev), _i64(poss, dev), _i64(cands, dev)
    if cands.dim() != 2 or ancs.numel() != cands.shape[0] or poss.numel() != cands.shape[0]:
        raise RuntimeError('sslrec_b200: one anchor, one positive and one row of candidates per pair')
    if bias is not None:
        _require_cuda(bias, 'logQ bias')
        if bias.dtype != torch.float32 or bias.shape != cands.shape:
            raise RuntimeError('sslrec_b200: the logQ bias must be fp32 and shaped like the candidates')
        bias = bias.detach().contiguous()
    ops, plain = _mix_operands([users, items])
    pack = (ops, ancs, poss, cands, float(temp), bias, len(plain))
    return _SsmFn.apply(pack, *plain, *_tokens(*[op for op in ops if isinstance(op, Rows)]))


# ---- in-batch negatives for the sampled softmax (optional key train.ssm_in_batch) -------------------------------------------

def in_batch_weights(indptr, indices, n_item: int) -> np.ndarray:
    """v [n_item] float64, the column weights of the in-batch softmax (include/sslrec_b200.h, a28), from a training CSR with
    distinct columns per row: v_i = 1 / (p_i + r_i) (0 when p_i + r_i = 0), where

        p_i = deg_i / |E|                                                 a positive slot holds i (uniform over the edges)
        r_i = sum_u (deg_u / |E|) [i not in P_u] / (n_item - deg_u)       a negative slot holds i (uniform over u's non-positives)

    r_i is computed in O(|E|) as (T - sum_{u holding i} a_u) / |E|, a_u = deg_u / (n_item - deg_u) (0 for a user who holds
    every item: no loader can serve it a negative), T = sum_u a_u.  B (p_i + r_i) is the expected count of i among the 2B
    columns of a batch of B pairs, so sum_c v[id_c] / B f(id_c) is an unbiased estimate of sum_i f(i) over the catalogue
    (Hansen-Hurwitz; the logQ correction of Yi et al. with the loaders' exact proposal).  It holds for the marginal law of
    the columns: a pair's own two columns follow its user's law, and nothing corrects for that.  Columns that are training
    positives of the pair's user are kept.  A pure function of the training matrix; ``InBatchWeights`` rounds it to fp32 once."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    n = int(n_item)
    if n < 1:
        raise ValueError(f'in_batch_weights: n_item {n} < 1')
    n_edge = int(indices.size)
    v = np.zeros(n, dtype=np.float64)
    if n_edge == 0:
        return v
    deg_u = np.diff(indptr).astype(np.float64)
    free = n - deg_u
    a = np.where(free > 0, deg_u / np.maximum(free, 1.0), 0.0)
    held = np.bincount(indices, weights=np.repeat(a, np.diff(indptr)), minlength=n)
    r = np.maximum(math.fsum(a.tolist()) - held, 0.0) / n_edge
    p = np.bincount(indices, minlength=n).astype(np.float64) / n_edge
    q = p + r
    np.divide(1.0, q, out=v, where=q > 0)
    return v


class InBatchWeights:
    """``in_batch_weights`` on a device: ``v`` fp32 [n_item] (rounded once); ``range``, max v / min v over the items with
    v > 0, which bounds the weights of any batch's columns and picks the forward's kernel (``contraction_kind``) on the host;
    and ``vmin``, the smallest v > 0, which bounds the smallest term of the forward (``in_batch_binades``)."""

    def __init__(self, v, device):
        v32 = np.asarray(v).astype(np.float32)
        live = v32[v32 > 0].astype(np.float64)
        if v32.ndim != 1 or not np.all(np.isfinite(v32)) or live.size == 0 or (v32 < 0).any():
            raise ValueError('in-batch weights must be a finite, non-negative [n_item] vector with a positive entry')
        self.n_item, self.range, self.vmin = int(v32.size), float(live.max() / live.min()), float(live.min())
        self.v = torch.from_numpy(v32).to(device)

    @classmethod
    def of_matrix(cls, indptr, indices, n_item: int, device) -> 'InBatchWeights':
        return cls(in_batch_weights(indptr, indices, n_item), device)


# the forward's terms w_c 2^(S - offset) stay normal fp32 numbers, which ex2.approx.ftz does not flush, while they span at most
# this many binades below 1 (include/sslrec_b200.h, a28: 126, less one binade for the rounding of S - offset)
IN_BATCH_MAX_BINADES = 125.0


def in_batch_binades(B: int, temp: float, vmin: float) -> float:
    """2 log2(e) / temp + max(0, log2(B / vmin)): how many binades below 1 the smallest term of the in-batch forward can lie
    (a column opposite its row, the smallest weight vmin / B); the term is refused past IN_BATCH_MAX_BINADES."""
    return 2.0 * LOG2E / float(temp) + max(0.0, math.log2(B / vmin))


def _in_batch_rows(op) -> Rows:
    """An operand of ``_mix_operands`` as the Rows the operand builder gathers from."""
    return op if isinstance(op, Rows) else Rows.constant(op[1])


class _SsmInBatchFn(torch.autograd.Function):
    """The in-batch sampled softmax (include/sslrec_b200.h, a28) on the InfoNCE contraction.  Operands as in ``_SsmFn``."""

    @staticmethod
    def forward(ctx, pack, *inputs):
        ops, ancs, poss, negs, tau, weights, n_plain = pack
        users, items = (_in_batch_rows(op) for op in ops)
        d = users.dim
        if items.dim != d:
            raise RuntimeError('sslrec_b200: the user and item rows of an in-batch softmax term differ in width')
        dev, B = ancs.device, ancs.numel()
        f = dict(device=dev, dtype=torch.float32)
        cols = torch.cat([poss, negs])
        off = LOG2E / tau
        kind = contraction_kind(d, off, colscale_range=weights.range)
        rowsum, obar, loss_b, out = torch.empty(B, **f), torch.empty(B, d, **f), torch.empty(B, **f), torch.empty((), **f)
        with torch.cuda.device(dev):
            s = _stream(ancs)
            # users are R here and C in the backward, the columns the other way round: both get the copies of either role
            a = _operand(users, ancs, 0, off, s, kind, streamed=True)
            t = _operand(items, cols, 0, 1.0, s, kind, streamed=True)
            w = torch.zeros(t.npad, **f)              # the padded tail is read (then masked) by the tile loads
            torch.div(weights.v.index_select(0, cols), B, out=w[:2 * B])
            n_split = _n_split(a, t)
            rs_part, o_part = torch.zeros(n_split, B, **f), torch.zeros(n_split, B, d, **f)
            _contract(a, t, w, off, n_split, rs_part, o_part, s, bwd=False)
            # rows 0 .. B-1 of the columns are the positives' p^
            check(lib.ssl_nce_finalize(rs_part.data_ptr(), o_part.data_ptr(), n_split, B, d, a.hat.data_ptr(), t.hat.data_ptr(), tau,
                                       0.0, rowsum.data_ptr(), obar.data_ptr(), loss_b.data_ptr(), s), 'ssl_nce_finalize')
            check(lib.ssl_sum(loss_b.data_ptr(), B, 1.0, out.data_ptr(), s), 'ssl_sum')
        ctx.pack = (ops, ancs, poss, cols, tau, a, t, w, rowsum, obar, n_plain, len(inputs) - n_plain)
        return out

    @staticmethod
    def backward(ctx, g):
        ops, ancs, poss, cols, tau, a, t, w, rowsum, obar, n_plain, n_tokens = ctx.pack
        g = g.contiguous()
        plain_grads: dict = {}
        targets = [_mix_grad_target(op, plain_grads) for op in ops]
        if any(p is None for p, _ in targets):
            raise RuntimeError('sslrec_b200: every operand of an in-batch softmax term must take a gradient')
        (gu, gu_s), (gi, gi_s) = targets
        dev, B, d = g.device, ancs.numel(), a.hat.shape[1]
        f = dict(device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            s = _stream(g)
            colscale = torch.zeros(a.npad, **f)
            check(lib.ssl_nce_colscale(rowsum.data_ptr(), B, g.data_ptr(), 1.0, colscale.data_ptr(), s), 'ssl_nce_colscale')
            n_split = _n_split(t, a)
            dt_part = torch.empty(n_split, 2 * B, d, **f)
            _contract(t, a, colscale, LOG2E / tau, n_split, None, dt_part, s, bwd=True)
            rows = (a.hat.data_ptr(), t.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), t.rinv.data_ptr())
            if deterministic():
                # identity ids into one -0.0 stage: users (positions ancs), the positives' row term (poss), the columns (cols)
                stage = _stage(4 * B, d, dev)
                ar = torch.arange(B, device=dev)
                check(lib.ssl_nce_bwd_rows(*rows, ar.data_ptr(), B, d, tau, g.data_ptr(), 1.0, stage.data_ptr(), d,
                                           stage[B:].data_ptr(), d, s), 'ssl_nce_bwd_rows')
                check(lib.ssl_nce_bwd_cols(dt_part.data_ptr(), n_split, t.hat.data_ptr(), t.rinv.data_ptr(), w.data_ptr(), None, 2 * B, d,
                                           stage[2 * B:].data_ptr(), d, s), 'ssl_nce_bwd_cols')
                _scatter_grouped([(stage[:B], ancs, gu, gu_s), (stage[B:], torch.cat([poss, cols]), gi, gi_s)])
            else:
                check(lib.ssl_nce_bwd_rows(*rows, ancs.data_ptr(), B, d, tau, g.data_ptr(), 1.0, gu, gu_s, None, 0, s), 'ssl_nce_bwd_rows')
                check(lib.ssl_nce_bwd_rows(*rows, poss.data_ptr(), B, d, tau, g.data_ptr(), 1.0, None, 0, gi, gi_s, s), 'ssl_nce_bwd_rows')
                check(lib.ssl_nce_bwd_cols(dt_part.data_ptr(), n_split, t.hat.data_ptr(), t.rinv.data_ptr(), w.data_ptr(), cols.data_ptr(),
                                           2 * B, d, gi, gi_s, s), 'ssl_nce_bwd_cols')
        zero = torch.zeros((), device=dev)
        return (None,) + tuple(plain_grads[k] for k in range(n_plain)) + (zero,) * n_tokens


def ssm_in_batch_sum(users, items, ancs, poss, negs, temp: float, weights: InBatchWeights) -> torch.Tensor:
    """The in-batch sampled softmax summed over the batch (formula in include/sslrec_b200.h, a28): for every pair
    ln(sum_c w_c exp(s_bc)) - s_bb over the 2B columns [poss; negs], s_bc = cos(users[ancs[b]], items[id_c]) / temp,
    w_c = weights.v[id_c] / B.  ``users`` / ``items`` as in ``ssm_loss_sum`` (a restricted view must mark every batch row);
    under ``deterministic()`` every batch row's gradient is added in position order.  Reads and draws no candidates.  Raises
    ValueError when ``in_batch_binades(B, temp, weights.vmin)`` exceeds IN_BATCH_MAX_BINADES: a smaller term would be flushed
    to 0 or lose digits (B, temp and vmin are host values, so CUDA-graph capture is unaffected)."""
    dev = weights.v.device
    ancs, poss, negs = _i64(ancs, dev), _i64(poss, dev), _i64(negs, dev)
    B = ancs.numel()
    if B < 1 or ancs.dim() != 1 or poss.shape != ancs.shape or negs.shape != ancs.shape:
        raise RuntimeError('sslrec_b200: an in-batch softmax term needs B >= 1 pairs of one anchor, one positive and one negative')
    if not 0.0 < C.c_float(temp).value < math.inf:
        raise ValueError(f'sslrec_b200: the in-batch softmax temperature must be finite and > 0, got {temp!r}')
    binades = in_batch_binades(B, temp, weights.vmin)
    if not binades <= IN_BATCH_MAX_BINADES:
        raise ValueError(f'sslrec_b200: the in-batch softmax at tau {temp!r}, B {B} and smallest weight {weights.vmin:.6g} needs '
                         f'2 log2(e) / tau + max(0, log2(B / min v)) <= {IN_BATCH_MAX_BINADES:g}, so that every term is a normal '
                         f'fp32 number, got {binades:.4f}: raise tau or the smallest weight')
    ops, plain = _mix_operands([users, items])
    pack = (ops, ancs, poss, negs, float(temp), weights, len(plain))
    return _SsmInBatchFn.apply(pack, *plain, *_tokens(*[op for op in ops if isinstance(op, Rows)]))


# ---- HCCF's hyper-graph branch (hccf.py:43-49, HGNNLayer :100-108) on the library's skinny-GEMM kernels ---------------------

def _rowgemm(in1, k1, m1, m1_trans, out, n_out, scale=1.0, slope=1.0, accumulate=False, in2=None, k2=0, m2=None, m2_trans=False, pre_ref=None,
             pre_slope=1.0):
    """out[r, :n_out] (+)= leaky(scale * (in1[r, :k1] M1 + in2[r, :k2] M2)); 2-D row-strided views are fine."""
    with torch.cuda.device(out.device):
        check(lib.ssl_rowgemm(in1.data_ptr(), in1.stride(0), k1, m1.data_ptr(), int(m1_trans), _ptr(in2), 0 if in2 is None else in2.stride(0), k2,
                              _ptr(m2), int(m2_trans), _ptr(pre_ref), 0 if pre_ref is None else pre_ref.stride(0), pre_slope, out.data_ptr(), out.stride(0),
                              n_out, scale, slope, int(accumulate), out.shape[0], _stream(out)), 'ssl_rowgemm')


def _colgemm(in1, k1, in2, k2, scale=1.0, slope=1.0, pre_ref=None, mode=0, ref=None, want_act=False):
    """out [k1, k2] = post(scale * sum_r in1[r]^T (x) in2[r]) (+ leaky(out) when want_act); deterministic two-stage reduction."""
    n = in1.shape[0]
    f = dict(device=in1.device, dtype=torch.float32)
    part = torch.empty(int(lib.ssl_colgemm_parts(n)), k1, k2, **f)
    out = torch.empty(k1, k2, **f)
    act = torch.empty(k1, k2, **f) if want_act else None
    with torch.cuda.device(in1.device):
        check(lib.ssl_colgemm(in1.data_ptr(), in1.stride(0), k1, in2.data_ptr(), in2.stride(0), k2, _ptr(pre_ref), 0 if pre_ref is None else pre_ref.stride(0),
                              slope, n, part.data_ptr(), scale, mode, _ptr(ref), out.data_ptr(), _ptr(act), _stream(in1)), 'ssl_colgemm')
    return (out, act) if want_act else out


class _IncidenceFn(torch.autograd.Function):
    """A = E_side W mult (hccf.py:43-44): [n, d] x [d, H]."""

    @staticmethod
    def forward(ctx, e, w, mult):
        _require_cuda(e, 'embeddings')
        e_, w_ = e.detach(), w.detach().contiguous()
        if e_.stride(1) != 1:
            e_ = e_.contiguous()
        a = torch.empty(e_.shape[0], w_.shape[1], device=e_.device, dtype=torch.float32)
        _rowgemm(e_, e_.shape[1], w_, False, a, w_.shape[1], scale=mult)
        ctx.pack = (e_, w_, mult)
        return a

    @staticmethod
    def backward(ctx, ga):
        e, w, mult = ctx.pack
        ga = ga.contiguous()
        de = dw = None
        if ctx.needs_input_grad[0]:
            de = torch.empty_like(e, memory_format=torch.contiguous_format)
            _rowgemm(ga, ga.shape[1], w, True, de, e.shape[1], scale=mult)              # dA W^T mult  (W [d, H] read as [n_out = d, k = H])
        if ctx.needs_input_grad[1]:
            dw = _colgemm(e, e.shape[1], ga, ga.shape[1], scale=mult)                     # E^T dA mult
        return de, dw, None


def hyper_incidence(e: torch.Tensor, w: torch.Tensor, mult: float) -> torch.Tensor:
    return _IncidenceFn.apply(e, w, float(mult))


@dataclass
class HyperDrop:
    """Dropout of one side's incidence for one layer (hccf.py:48-49): keep probability, and either a seed for the in-kernel
    generator (stream = layer * 2 + side) or an injected [n, H] float 0 / 1 keep mask."""
    keep: float = 1.0
    seed: int = 0
    stream: int = 0
    mask: Optional[torch.Tensor] = None


def _drop(x: torch.Tensor, d: HyperDrop, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    if d.keep == 1.0:
        if out is None:
            return x
        out.add_(x) if accumulate else out.copy_(x)
        return out
    out = torch.empty_like(x) if out is None else out
    mask = None if d.mask is None else d.mask.to(torch.float32).contiguous()
    with torch.cuda.device(x.device):
        ptr = getattr(d.seed, 'ptr', 0)
        if ptr and mask is None:
            check(lib.ssl_hyper_dropout_dev(x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], d.keep, 1, None, ptr, d.stream, int(accumulate),
                                            _stream(x)), 'ssl_hyper_dropout_dev')
        else:
            check(lib.ssl_hyper_dropout(x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], d.keep, 2 if mask is not None else 1, _ptr(mask),
                                        int(d.seed), d.stream, int(accumulate), _stream(x)), 'ssl_hyper_dropout')
    return out


class _HyperLayerFn(torch.autograd.Function):
    """Both sides' hyper-graph message of one layer: Y_side = act(H act(H^T X_side)), H = dropout(A_side) (hccf.py:48-49,
    :100-108).  x is the full [N, d] layer input, a_u / a_i the sides' incidences; the backward returns dX, dA_u, dA_i."""

    @staticmethod
    def forward(ctx, x, a_u, a_i, slope, drop_u: HyperDrop, drop_i: HyperDrop):
        _require_cuda(x, 'layer input')
        x_ = x.detach().contiguous()
        nu, d = a_u.shape[0], x_.shape[1]
        y = torch.empty_like(x_)
        saved = []
        for a, drop, lo, hi in ((a_u.detach().contiguous(), drop_u, 0, nu), (a_i.detach().contiguous(), drop_i, nu, x_.shape[0])):
            h = a.shape[1]
            hk = _drop(a, drop)
            xs, ys = x_[lo:hi], y[lo:hi]
            lat, latact = _colgemm(hk, h, xs, d, slope=slope, want_act=True)               # act(H^T X)   (:105)
            _rowgemm(hk, h, latact, False, ys, d, slope=slope)                               # act(H lat)   (:106)
            saved.append((hk, lat, latact, drop, lo, hi))
        ctx.pack = (x_, y, slope, saved)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, y, slope, saved = ctx.pack
        gy = gy.contiguous()
        d = x.shape[1]
        gx = torch.empty_like(x)
        gas = []
        for hk, lat, latact, drop, lo, hi in saved:
            h = hk.shape[1]
            xs, ys, gs = x[lo:hi], y[lo:hi], gy[lo:hi]
            # dZ = dY * act'(Y) is formed while dY is loaded;  dlat = (H^T dZ) * act'(lat)
            dlat = _colgemm(hk, h, gs, d, slope=slope, pre_ref=ys, mode=1, ref=lat)
            dhk = torch.empty_like(hk)
            _rowgemm(gs, d, latact, True, dhk, h, in2=xs, k2=d, m2=dlat, m2_trans=True, pre_ref=ys, pre_slope=slope)     # dZ lat^T + X dlat^T
            _rowgemm(hk, h, dlat, False, gx[lo:hi], d)                                      # dX = H dlat
            gas.append(_drop(dhk, drop, out=torch.empty_like(dhk)) if drop.keep != 1.0 else dhk)
        return gx, gas[0], gas[1], None, None, None


def hyper_layer(x, a_u, a_i, slope: float, drop_u: HyperDrop, drop_i: HyperDrop) -> torch.Tensor:
    # the backward takes act'(.) from the saved output (Y > 0 -> 1, else slope), which is right only while LeakyReLU keeps
    # the sign; a negative slope would need the pre-activation saved as well
    if not float(slope) >= 0.0:
        raise ValueError(f'hyper_layer: LeakyReLU slope must be >= 0, got {slope}')
    return _HyperLayerFn.apply(x, a_u, a_i, float(slope), drop_u, drop_i)


class _SumSqFn(torch.autograd.Function):
    """reg_params over the flat table: value by a deterministic reduction; the gradient 2 g W is
    added into the state's G_e0 sink (consumed by the last backward layer's epilogue)."""

    @staticmethod
    def forward(ctx, st, e0, *tokens):
        out = torch.empty((), device=e0.device, dtype=torch.float32)
        with torch.cuda.device(e0.device):
            check(lib.ssl_sumsq(e0.data_ptr(), e0.numel(), out.data_ptr(), _stream(e0)), 'ssl_sumsq')
        ctx.st, ctx.e0, ctx.n_in = st, e0, len(tokens)
        return out

    @staticmethod
    def backward(ctx, g):
        st = ctx.st
        g = g.contiguous()
        # the propagation's backward (which autograd runs after this node: it depends on the token) applies 2 g E0
        st.reg_pending = g if st.reg_pending is None else st.reg_pending + g
        return (None, None) + (torch.zeros((), device=g.device),) * ctx.n_in


def table_sumsq(st: PropState) -> torch.Tensor:
    """sum ||W||^2 of the embedding table a PropState was built from (loss_utils.py:20-24)."""
    return _SumSqFn.apply(st, st.e0, *([st.token] if st.token is not None else []))
