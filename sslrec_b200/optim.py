"""FusedAdam -- torch.optim.Adam semantics (trainer/trainer.py:45-49: Adam(lr, weight_decay), no
amsgrad) as ONE pass over (p, g, m, v) per parameter with the native kernel; when the parameters are
adjacent views of a flat table and so are their gradients, one launch covers them all."""
from __future__ import annotations

import ctypes as C

import torch

from ._lib import check, lib


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, row_shards=None, comm=None):
        """row_shards / comm (row-sharded multi-GPU, BaseModel.shard_to): {id(param): (lo, hi, peer base addresses)} -- such a
        parameter is updated on its owned rows [lo, hi) only and the new values are stored to the same rows of every
        peer's replica by the kernel (the all-gather of the updated table, fused into the optimizer)."""
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.row_shards = dict(row_shards or {})          # keyed by id(param)
        self.comm = comm
        self._step_dev = None         # CUDA-graph mode: the step count lives on the device (enable_device_step)

    def enable_device_step(self, device) -> None:
        """Keep the 1-based step count in a device word that the optimizer step itself increments, and form the bias corrections on
        the device (``ssl_adam_step_dev``): a captured step then replays correctly.  The count continues from the host's."""
        steps = {int(st['step']) for st in self.state.values() if st}
        if len(steps) > 1:
            raise RuntimeError('parameters with different step counts cannot share the device counter')
        self._step_dev = torch.full((1,), steps.pop() if steps else 0, dtype=torch.int64, device=device)
        self._dyn = {}

    def sync_host_step(self) -> None:
        """Copy the device step count into every parameter's host ``step`` (device mode keeps running): ``state_dict()`` then
        holds the count the next step continues from."""
        if self._step_dev is not None:
            n = int(self._step_dev.item())
            for st in self.state.values():
                if st:
                    st['step'] = n

    def disable_device_step(self) -> None:
        self.sync_host_step()
        self._step_dev = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group['betas']
            todo = []
            for p in group['params']:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32:
                    raise RuntimeError('FusedAdam: CUDA float32 parameters only (no CPU path)')
                st = self.state[p]
                if not st:
                    st['step'] = 0
                    st['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                if self._step_dev is None:
                    st['step'] += 1
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                todo.append((p, g, st))
            if self._step_dev is not None and todo:
                self._step_dev.add_(1)
            sharded = [p for p, _, _ in todo if id(p) in self.row_shards]
            if sharded and self.comm is not None:
                self.comm.barrier()          # every rank has finished reading the old parameters (backward) before any peer store
            from . import engine
            timed = engine._timed('adam', dict(params=len(todo), sharded=len(sharded)))
            timed.__enter__()
            for p, g, st in todo:
                if not p.is_contiguous():
                    raise RuntimeError('FusedAdam: parameters must be contiguous')
                with torch.cuda.device(p.device):
                    stream = torch.cuda.current_stream(p.device).cuda_stream
                    if self._step_dev is not None:
                        if id(p) in self.row_shards:
                            raise RuntimeError('the device step counter is for single-GPU CUDA-graph replay; row-sharded parameters use the host counter')
                        dyn = self._dyn.setdefault(id(p), torch.empty(2, dtype=torch.float32, device=p.device))
                        check(lib.ssl_adam_step_dev(p.data_ptr(), None, 0, g.data_ptr(), st['exp_avg'].data_ptr(), st['exp_avg_sq'].data_ptr(), p.numel(),
                                                    self._step_dev.data_ptr(), dyn.data_ptr(), group['lr'], b1, b2, group['eps'], group['weight_decay'],
                                                    stream), 'ssl_adam_step_dev')
                    elif id(p) in self.row_shards:
                        lo, hi, peers = self.row_shards[id(p)][:3]
                        w = p.shape[1] if p.dim() > 1 else 1
                        off = 4 * lo * w
                        arr = (C.c_void_p * max(1, len(peers)))(*[q + off for q in peers])
                        check(lib.ssl_adam_step_peers(p.data_ptr() + off, arr, len(peers), g.data_ptr() + off, st['exp_avg'].data_ptr() + off,
                                                      st['exp_avg_sq'].data_ptr() + off, (hi - lo) * w, st['step'], group['lr'], b1, b2,
                                                      group['eps'], group['weight_decay'], stream), 'ssl_adam_step_peers')
                    else:
                        check(lib.ssl_adam_step(p.data_ptr(), g.data_ptr(), st['exp_avg'].data_ptr(), st['exp_avg_sq'].data_ptr(),
                                                p.numel(), st['step'], group['lr'], b1, b2, group['eps'], group['weight_decay'], stream),
                              'ssl_adam_step')
            timed.__exit__(None, None, None)
            if sharded and self.comm is not None:
                self._after_sharded_step(sharded)
        return loss

    def _after_sharded_step(self, params):
        """symm transport: the new rows are already in the peers' replicas -> barrier.  nccl transport: all-gather the owned
        row blocks of each parameter."""
        if self.comm.transport == 'symm':
            self.comm.barrier()
            return
        for p in params:
            bounds = self.row_shards[id(p)][3] if len(self.row_shards[id(p)]) > 3 else None
            if bounds is None:
                raise RuntimeError('sharded parameter without block boundaries (BaseModel.shard_to provides them)')
            self.comm.gather_blocks(p.data, bounds)
