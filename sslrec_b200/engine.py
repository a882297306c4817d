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

import ctypes as C
import functools
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

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
        b = self.base.view(-1, self.n_views, self.dim)
        return b[self.off:self.off + self.n, self.v, :]

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


def _bpr_bwd(users: Rows, items: Rows, ancs, poss, negs, coef, g):
    g = g.contiguous()
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


def contraction_kind(d: int, offset: float, raw: bool = False) -> str:
    """The InfoNCE contraction kernel for rows of width ``d`` at ``offset``: 'ffma' (FP32 FMA, any d), 'tf32x3' (3xTF32 on the
    tensor cores: raw rows, which the 3xFP16 operand bound does not cover, and offsets above F16X3_MAX_OFFSET) or 'f16x3'."""
    if not USE_TENSOR_CORES or d not in (32, 64):
        return 'ffma'
    if raw or not f16x3_applies(offset):
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
              live_role: int = LIVE_ROWS):
    """One launch of the contraction of R against C on their kernel, timed as the forward role (R = anchors) or, with
    ``colscale``, the backward role (R = table, C = anchors).  ``live``: the device count that bounds the ``live_role`` side."""
    name = _GEMM_ENTRY[R.kind] + ('' if live is None else '_live')
    if R.kind == 'ffma':
        ops = (R.hat.data_ptr(), R.n, C.hat.data_ptr(), C.t.data_ptr(), C.n)
    elif R.kind == 'tf32x3':
        ops = (R.hi.data_ptr(), R.lo.data_ptr(), R.n, C.hi.data_ptr(), C.lo.data_ptr(), C.thi.data_ptr(), C.tlo.data_ptr(), C.npad, C.n)
    else:
        ops = (R.hi.data_ptr(), R.lo.data_ptr(), R.n, C.hi.data_ptr(), C.lo.data_ptr(), C.n)
    tail = () if live is None else (live.data_ptr(), live_role)
    d, bwd = R.hat.shape[1], colscale is not None
    meta = dict(B=C.n, n=R.n) if bwd else dict(B=R.n, n=C.n)
    with _timed('nce_gemm_bwd' if bwd else 'nce_gemm_fwd', dict(meta, dim=d, tc=R.kind != 'ffma')):
        check(getattr(lib, name)(*ops, d, _ptr(colscale), offset, n_split, _ptr(rowsum_part), o_part.data_ptr(), *tail, s),
              f'{name}({"bwd" if bwd else "fwd"})')


def _nce_fwd(e1: Rows, e2: Rows, table: Rows, idx, idx2, tau, norm_mode, mean, deno_eps, live=None):
    """``live``: optional int64 DEVICE scalar; only the first ``*live`` of the ``idx`` rows are anchors (a padded list of
    capacity idx.numel(), see ``dense_infonce_spec_nodes_mean_dev``).  Shapes and n_split then depend on the capacity only."""
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
    return out, (e1, e2, table, idx, tau, mean, a, p, t, rowsum, obar, full_table, comm, live)


def _nce_bwd(saved, g):
    e1, e2, table, idx, tau, mean, a, p, t, rowsum, obar, full_table, comm, live = saved
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
        if live is not None and (g1 is not None or g2 is not None):        # rows b < live only, mean over live
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


def _align_bwd(pack, g):
    x, y, ix, iy, xh, yh, rx, ry = pack
    B, d = ix.numel(), x.dim
    g = g.contiguous()
    c = 2.0 / B                                                # d/dx^ mean |x^ - y^|^2 = 2 (x^ - y^) / B
    with torch.cuda.device(g.device):
        s = _stream(g)
        for (rows, idx, a, b, ri) in ((x, ix, xh, yh, rx), (y, iy, yh, xh, ry)):
            gp = rows.grad_ptr()
            if gp is not None:
                check(lib.ssl_unit_rows_bwd(a.data_ptr(), ri.data_ptr(), idx.data_ptr(), B, d, a.data_ptr(), c, b.data_ptr(), -c,
                                            g.data_ptr(), 1.0, gp, rows.grad_stride, s), 'ssl_unit_rows_bwd(align)')


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


def _uniform_bwd(pack, g):
    x, ix, c, rinv, w, total = pack
    gp = x.grad_ptr()
    if gp is None:
        return
    coef = (g * 8.0 / total).contiguous()                       # d total / d x^_i = 8 sum_{j != i} e_ij x^_j
    with torch.cuda.device(g.device):
        check(lib.ssl_unit_rows_bwd(c.data_ptr(), rinv.data_ptr(), ix.data_ptr(), ix.numel(), x.dim, w.data_ptr(), 1.0, None, 0.0,
                                    coef.data_ptr(), 1.0, gp, x.grad_stride, _stream(g)), 'ssl_unit_rows_bwd(uniformity)')


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
        _align_bwd(ctx.pack, g)
        return ctx.sinks[0](), ctx.sinks[1]()


class _DenseUniformFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        rx, ctx.sink = _dense_rows(x, True)
        out, ctx.pack = _uniform_fwd(rx, torch.arange(x.shape[0], device=x.device))
        return out

    @staticmethod
    def backward(ctx, g):
        _uniform_bwd(ctx.pack, g)
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
        _bpr_bwd(users, items_r, ar, ar, ar + B, coef, g)
        gi = si()
        return su(), gi[:B], gi[B:]


class _DenseInfoNceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e1, e2, table, idx, idx2, tau, norm_mode, mean, deno_eps, shared_table, live=None):
        ctx.n_inputs = 10 if live is None else 11
        r1, s1 = _dense_rows(e1, ctx.needs_input_grad[0])
        if shared_table:                      # e2 rows are rows of the table itself (spec_nodes)
            rt, st_ = _dense_rows(table, ctx.needs_input_grad[2])
            r2, s2 = rt, st_
        else:
            r2, s2 = _dense_rows(e2, ctx.needs_input_grad[1])
            rt, st_ = _dense_rows(table, ctx.needs_input_grad[2])
        out, ctx.saved_pack = _nce_fwd(r1, r2, rt, idx, idx2, tau, norm_mode, mean, deno_eps, live)
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
    return _DenseInfoNceFn.apply(e1, e2, all2, ar, ar, float(temp), 0, False, 0.0, False)


def dense_infonce_spec_nodes_mean(embeds1, embeds2, nodes, temp):
    """cal_infonce_loss_spec_nodes(embeds1 [N,d], embeds2 [N,d], nodes, temp) -- loss_utils.py:42-51."""
    nodes = _i64(nodes, embeds2.device)
    return _DenseInfoNceFn.apply(embeds1, embeds2, embeds2, nodes, nodes, float(temp), 1, True, 1e-8, True)


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
    return _DenseInfoNceFn.apply(embeds1, embeds2, embeds2, nodes, nodes, float(temp), 1, True, 1e-8, True, count)


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
