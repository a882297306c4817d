"""Row-sharded multi-GPU execution (SURVEY.md section 8e; BASELINE.json north_star): one process per
GPU, ``torch.distributed`` for the plumbing, the data path in the library's own kernels.

Partition.  Every GPU owns the same share of BOTH sides of the bipartite graph: user rows
[u0, u1) and item rows [|U| + i0, |U| + i1) (equal blocks of ceil(n_side / world) rows), so the stored
entries -- half of which sit in the item rows -- are balanced; a contiguous split of the N rows would give the
last rank every item row (half of all entries at BASELINE config 4).  Each GPU keeps FULL [N, V, d]
tables (180 GB of HBM per GPU: the 6 GB tables of config 4 are replicated, the CSR is not) and computes
only the rows it owns from a full copy of the previous layer.

Exchange steps -- the only inter-GPU traffic on the path:
  * per propagation layer and direction the all-gather of the d-wide layer output.  With the
    ``symm`` transport it is FUSED INTO THE SpMM: the tables live in symmetric memory (every rank maps
    every peer's allocation over NVLink), the kernel's epilogue stores each finished row to the same
    row of all peers' tables (``ssl_prop_args.x_out_peers``), so the NVLink traffic overlaps the
    gathers of the rows still being computed; what remains is a cross-GPU barrier on the stream after the
    launch.  (Optionally the row is stored once to the allocation's NVSwitch multicast address instead: measured equal,
    the exchange is ingress-bound.)  The ``nccl`` transport (fallback, and the gloo CPU tests) all-gathers the owned row
    blocks with ``all_gather_into_tensor`` after the launch;
  * the updated parameters: Adam runs on the owned rows only and stores the new values to every peer's
    replica of the table (``ssl_adam_step_peers``) -- the sixth all-gather of a step, fused the same way;
  * per InfoNCE term one all-reduce of the per-anchor partial (row sum, weighted table average)
    [B, d+1], because the table rows (negatives) are sharded and the anchors are replicated, and in the
    backward one all-gather of the [N_side/world, d] dense table-gradient blocks.
Propagation is sharded only when ``shard_propagation`` (automatic by table size): for the bundled-dataset
shapes a layer takes ~0.15 ms while its all-gather would move the whole 123 MB layer, so there the SpMM is
replicated and only the loss is sharded.  With sharded propagation every parameter row has ONE owner that
computes its update and stores it into all replicas, so the replicas are bit-identical by construction; with
loss-only sharding every rank repeats the same propagation / BPR / Adam arithmetic, and because the BPR backward
adds batch rows with floating-point atomics the replicas agree to fp32 rounding (call ``RowShard.resync(params)``
-- a broadcast from rank 0 -- once per epoch if exact agreement matters).

``BatchShard`` is the other way to use N GPUs: the batches are the sharded unit.  Every rank runs the
whole step on its OWN batch of B samples and the only exchange is one all-reduce (average) of the
parameter gradients before the Adam step.  For LightGCN, SimGCL, SGL and NCL every loss term is a batch
sum divided by the batch size (lightgcn.py:52, simgcl.py:48-50, sgl.py:56-60, ncl.py:58,68,82) or does
not depend on the batch (reg_params), and the in-kernel augmentation draws are keyed by the shared seed, so
the averaged gradient IS the gradient of one reference step at ``batch_size = world * B``.  It is the usual
data-parallel APPROXIMATION (not an identity) for HCCF (its contrastive term averages over the batch's
unique nodes, hccf.py:80-81, and F.dropout draws per rank), for DirectAU (uniformity is the log of a
per-batch pair mean, loss_utils.py:82-86) and for NCL's k-means initialisation unless the torch seeds are in
lock-step.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from .graph import GraphPlan


def block_range(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Rank's share of n rows cut into ``world`` equal blocks of ceil(n / world) (the last ones short or empty)."""
    blk = (n + world - 1) // world
    lo = min(n, rank * blk)
    return lo, min(n, lo + blk)


def balanced_bounds(weights: torch.Tensor, world: int) -> List[int]:
    """Cut rows 0..n into ``world`` contiguous blocks of (nearly) equal total weight: [0, b1, ..., n].  With the rows'
    stored-entry counts as weights every GPU's SpMM does the same number of gathers even when a few hub rows (the Zipf head of
    the item side) hold a large share of the entries."""
    n = int(weights.shape[0])
    if n == 0:
        return [0] * (world + 1)
    cum = torch.cumsum(weights.to(torch.float64) + 1e-9, 0)
    targets = cum[-1] * torch.arange(1, world, dtype=torch.float64, device=cum.device) / world
    cuts = torch.searchsorted(cum, targets).clamp_(0, n).tolist()
    b = [0] + [int(c) for c in cuts] + [n]
    for i in range(1, len(b)):
        b[i] = max(b[i], b[i - 1])
    return b


class SharedTable:
    """A [N, ...] fp32 table that exists on every rank at the same logical address: ``t`` is this rank's copy,
    ``peer_ptrs`` the device addresses of the OTHER ranks' copies as mapped into this process (empty for the
    nccl transport)."""

    def __init__(self, t: torch.Tensor, peer_ptrs: List[int], handle=None, mc_ptr: int = 0):
        self.t, self.peer_ptrs, self.handle = t, peer_ptrs, handle
        self.mc_ptr = mc_ptr          # NVSwitch multicast address of the table (0: unavailable): ONE store reaches every GPU's copy


class RowShard:
    def __init__(self, dist, rank: int, world: int, n: int, shard_propagation='auto', dim: int = 64, views: int = 3,
                 n_user: Optional[int] = None, transport: str = 'auto', multicast='auto', user_bounds=None, item_bounds=None):
        """user_bounds / item_bounds: optional block boundaries [0, ..., n_side] (world + 1 entries each, e.g. from
        ``balanced_bounds`` of the rows' entry counts); default: equal blocks of ceil(n_side / world) rows."""
        self.dist, self.rank, self.world, self.n = dist, rank, world, n
        self.n_user = n if n_user is None else int(n_user)          # None: one side only (a contiguous block of rows)
        n_item = n - self.n_user
        self.user_bounds = [block_range(self.n_user, world, r)[0] for r in range(world)] + [self.n_user] if user_bounds is None else [int(b) for b in user_bounds]
        self.item_bounds = [block_range(n_item, world, r)[0] for r in range(world)] + [n_item] if item_bounds is None else [int(b) for b in item_bounds]
        for b, total in ((self.user_bounds, self.n_user), (self.item_bounds, n_item)):
            if len(b) != world + 1 or b[0] != 0 or b[-1] != total or any(b[i] > b[i + 1] for i in range(world)):
                raise ValueError('block boundaries must be world + 1 ascending values from 0 to the side\'s row count')
        self.u0, self.u1 = self.user_bounds[rank], self.user_bounds[rank + 1]
        self.i0, self.i1 = self.n_user + self.item_bounds[rank], self.n_user + self.item_bounds[rank + 1]
        # Row-sharding the propagation costs one all-gather of the whole [N, V, d] layer per layer and
        # direction; it pays when the SpMM is long (HBM-bound tables far beyond L2, BASELINE.json config 4),
        # not when a layer takes ~0.2 ms (the bundled datasets).  The contraction of the contrastive loss
        # is sharded over the table rows in either mode.
        if shard_propagation == 'auto':
            shard_propagation = n * views * dim * 4 >= (1 << 30)
        self.shard_propagation = bool(shard_propagation)
        if transport == 'auto':
            transport = 'symm' if (dist.get_backend() == 'nccl' and world <= 8) else 'nccl'
        if transport not in ('symm', 'nccl'):
            raise ValueError("transport must be 'symm' (fused NVLink stores) or 'nccl' (all_gather after the launch)")
        self.transport = transport
        # symm transport, optional: store finished rows ONCE, to the NVSwitch multicast address of the table (the switch
        # replicates; the sender's egress drops by world - 1) instead of once per peer.  The exchange is bound by what every GPU
        # RECEIVES, not by what it sends, so the plain peer stores stay the default.
        # multicast=True or SSLREC_B200_MULTICAST=1 selects it.
        import os
        env = os.environ.get('SSLREC_B200_MULTICAST')
        self.multicast = (env == '1') if multicast == 'auto' else bool(multicast)
        self._tables: Dict[tuple, SharedTable] = {}
        self._barrier_handle = None
        self.stats = dict(barriers=0, gathers=0, gathered_bytes=0)

    # ---- ownership -----------------------------------------------------------------------------
    @property
    def ranges(self):
        return (self.u0, self.u1), (self.i0, self.i1)

    @property
    def n_local(self) -> int:
        return (self.u1 - self.u0) + (self.i1 - self.i0)

    def make_plan(self, adj: torch.Tensor, device, side_split: int = 0) -> GraphPlan:
        idx, val = adj._indices(), adj._values()
        return GraphPlan(idx[0].cpu().numpy(), idx[1].cpu().numpy(), val.cpu().numpy(), adj.shape[0], device,
                         row_ranges=self.ranges, side_split=side_split)

    # ---- shared tables -------------------------------------------------------------------------
    def table(self, key, shape, device) -> SharedTable:
        """Persistent [N, ...] fp32 table named ``key`` (allocated collectively on first use: every rank must ask for
        the same keys in the same order)."""
        k = (key, tuple(shape))
        tb = self._tables.get(k)
        if tb is None:
            tb = self._alloc(tuple(shape), device)
            self._tables[k] = tb
        return tb

    def _alloc(self, shape, device) -> SharedTable:
        if self.transport == 'symm':
            import torch.distributed._symmetric_memory as symm
            t = symm.empty(shape, dtype=torch.float32, device=device)
            hdl = symm.rendezvous(t, self.dist.group.WORLD.group_name)
            ptrs = [int(p) for q, p in enumerate(hdl.buffer_ptrs) if q != self.rank]
            if self._barrier_handle is None:
                self._barrier_handle = hdl
            mc = int(getattr(hdl, 'multicast_ptr', 0) or 0) if self.multicast else 0
            return SharedTable(t, ptrs, hdl, mc)
        return SharedTable(torch.empty(shape, dtype=torch.float32, device=device), [])

    def sync_rows(self, tb: SharedTable) -> None:
        """After a launch that wrote the owned rows of ``tb``: make every rank's copy complete.  symm: the rows are
        already on their way to the peers (stores issued by the kernel), so a cross-GPU barrier on the stream is all
        that is left; nccl: all-gather the owned row blocks of both sides."""
        if self.transport == 'symm':
            self.barrier()
            return
        t = tb.t
        for bounds, side_lo in ((self.user_bounds, 0), (self.item_bounds, self.n_user)):
            self.gather_blocks(t[side_lo:side_lo + bounds[-1]], bounds)

    def gather_blocks(self, side: torch.Tensor, bounds) -> None:
        """``side``: one side's rows of a table (a view); rank r has written rows [bounds[r], bounds[r+1]).  All-gather the
        blocks (padded to the largest) and copy every rank's block into place."""
        if bounds[-1] == 0:
            return
        blk = max(bounds[r + 1] - bounds[r] for r in range(self.world))
        lo, hi = bounds[self.rank], bounds[self.rank + 1]
        local = torch.zeros((blk,) + tuple(side.shape[1:]), device=side.device, dtype=side.dtype)
        local[:hi - lo].copy_(side[lo:hi])
        full = torch.empty((self.world * blk,) + tuple(side.shape[1:]), device=side.device, dtype=side.dtype)
        self.dist.all_gather_into_tensor(full, local)
        for r in range(self.world):
            a, b = bounds[r], bounds[r + 1]
            if r != self.rank and b > a:
                side[a:b].copy_(full[r * blk:r * blk + (b - a)])
        self.stats['gathers'] += 1
        self.stats['gathered_bytes'] += full.numel() * 4

    def barrier(self) -> None:
        """Cross-GPU barrier ordered on the current stream (no host synchronisation with the symm transport)."""
        self.stats['barriers'] += 1
        if self.transport == 'symm' and self._barrier_handle is not None:
            self._barrier_handle.barrier(channel=0)
        else:
            self.dist.barrier()

    def resync(self, params) -> None:
        """Broadcast rank 0's parameters (loss-only sharding: removes the rounding-level drift between replicas)."""
        for p in params:
            self.dist.broadcast(p.data, src=0)

    # ---- loss sharding (InfoNCE table rows) -------------------------------------------------------
    def allreduce_sum(self, t: torch.Tensor) -> torch.Tensor:
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
        return t

    def side_block(self, n: int) -> int:
        return (n + self.world - 1) // self.world

    def side_range(self, off: int, n: int):
        """This rank's share of the table rows [off, off+n) of one side (equal blocks, last padded)."""
        blk = self.side_block(n)
        lo = min(off + n, off + self.rank * blk)
        return lo, min(off + n, lo + blk)

    def allgather_side(self, local: torch.Tensor, n: int) -> torch.Tensor:
        """local [side_block(n), d] -> [n, d] (rows of all ranks' side blocks in order)."""
        out = torch.empty((self.world * local.shape[0],) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
        self.dist.all_gather_into_tensor(out, local.contiguous())
        return out[:n]


class BatchShard:
    """Data-parallel training over batches (module docstring).  ``average_gradients`` is called between
    ``loss.backward()`` and ``optimizer.step()`` (trainer.py:67-68)."""

    def __init__(self, dist, rank: int, world: int):
        self.dist, self.rank, self.world = dist, rank, world
        self._avg = dist.get_backend() == 'nccl'          # gloo has no ReduceOp.AVG

    @staticmethod
    def coalesce(grads):
        """Merge gradients that are adjacent contiguous views of one storage (user_embeds.grad / item_embeds.grad
        are the two halves of the flat [N, d] sink) into single 1-D views: one collective instead of several."""
        flat, out = [], []                       # out: (position of the group's first member in ``grads``, buffer)
        for pos, g in enumerate(grads):
            if g.is_contiguous() and g.dtype == torch.float32:
                flat.append((pos, g))
            else:
                out.append((pos, g))
        flat.sort(key=lambda e: (e[1].untyped_storage().data_ptr(), e[1].data_ptr()))
        k = 0
        while k < len(flat):
            first, n, pos = flat[k][1], flat[k][1].numel(), flat[k][0]
            j = k + 1
            while (j < len(flat) and flat[j][1].untyped_storage().data_ptr() == first.untyped_storage().data_ptr()
                   and flat[j][1].data_ptr() == first.data_ptr() + 4 * n):
                n += flat[j][1].numel()
                pos = min(pos, flat[j][0])
                j += 1
            out.append((pos, first if j == k + 1 else torch.as_strided(first, (n,), (1,))))
            k = j
        # addresses differ between processes: the collectives must be issued in parameter order on every rank
        return [b for _, b in sorted(out, key=lambda e: e[0])]

    def average_gradients(self, params) -> None:
        grads = [p.grad for p in params if p.grad is not None]
        for g in self.coalesce(grads):
            if self._avg:
                self.dist.all_reduce(g, op=self.dist.ReduceOp.AVG)
            else:
                self.dist.all_reduce(g, op=self.dist.ReduceOp.SUM)
                g.mul_(1.0 / self.world)

    def shard_loader(self, dataset, batch_size: int, seed: int = 0):
        """The train DataLoader of data_handler_general_cf.py:95 with this rank's 1/world share of every epoch's
        shuffle (call ``loader.sampler.set_epoch(e)`` per epoch, as Trainer.train_epoch does)."""
        from torch.utils import data
        sampler = data.distributed.DistributedSampler(dataset, num_replicas=self.world, rank=self.rank, shuffle=True, seed=seed)
        return data.DataLoader(dataset, batch_size=batch_size, sampler=sampler, num_workers=0)
