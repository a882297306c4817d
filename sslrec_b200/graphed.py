"""One training step -- ``zero_grad, cal_loss, backward, optimizer.step`` (trainer/trainer.py:63-68) -- captured ONCE in a CUDA
graph and replayed per batch.

Why.  A step of the small BASELINE configs is a few dozen sub-100-us kernels: LightGCN on the gowalla shape needs 0.2 ms of GPU
time but ~1 ms of host time to enqueue (Python autograd nodes, ctypes calls, allocator), so the eager loop is host-bound.  A graph
replay is one launch.

What makes a captured step correct here:
  * batch indices are copied into static device buffers before the replay;
  * every in-kernel random draw (edge / node masks, perturbation noise, hyper-graph dropout) takes its seed from a DEVICE word
    (``ssl_prop_args.seed_ptr``, ``ssl_node_drop_dev``, ``ssl_hyper_dropout_dev``); before each replay the host writes the next
    seeds of the model's ``SeedStream`` there -- the SAME sequence the eager loop would draw, so eager and graphed training
    produce the same masks, losses and parameters;
  * Adam's step count lives on the device and the graph increments it (``ssl_adam_step_dev``);
  * nothing inside reads back to the host: the loss scalars stay in static tensors that the caller reads (or copies
    asynchronously) after the replay.
  * the model knows it is driven by a graph (``model._graph_mode``, set here from the dry run on and cleared by ``close``), so
    every step of it -- dry run, warm-up, captured step and ``eager`` -- takes the graph-safe path: HCCF de-duplicates its
    batch on the device and bounds its spec-node InfoNCE by the device count (``engine.dense_infonce_spec_nodes_mean_dev``);
  * host-side work that must not be captured runs before the step through the model's ``graph_pre_step(recluster)`` hook:
    NCL's k-means, when the caller says the batch carries the re-cluster flag (and on the first step, as the eager
    ``cal_loss`` does), copying the new centroids / assignments into the buffers the graph reads.
All seven drop-in models (LightGCN, SimGCL, SGL, NCL, HCCF, LightGCL, DirectAU) capture.  Not capturable: multi-GPU exchanges.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import torch


class GraphedStep:
    def __init__(self, model, optimizer, example_batch: Sequence[torch.Tensor], warmup: int = 3, recluster: bool = False):
        """Runs ``warmup`` eager steps on ``example_batch`` (they DO train: call it with the first batch of the run), then captures.
        ``recluster``: the example batch carries NCL's re-cluster flag (each warm-up step re-clusters, as the eager loop would
        on every step of that batch)."""
        self.model, self.opt = model, optimizer
        dev = example_batch[0].device
        if dev.type != 'cuda':
            raise RuntimeError('GraphedStep needs CUDA tensors')
        self.device = dev
        self.static_batch = [b.clone() for b in example_batch]
        self._pre_step = getattr(model, 'graph_pre_step', None)
        model._graph_mode = True
        # the first warm-up step's host-side work comes before the dry run, which needs its results but must not redo it
        self._run_pre_step(recluster)
        seeds = model._seeds
        # how many seeds does one step draw?  (counted on a dry forward without touching the parameters or the seed sequence)
        state, count = seeds.state, seeds.count
        with torch.no_grad():
            model.cal_loss(self.static_batch)
        self.n_seeds = seeds.count - count
        seeds.state, seeds.count = state, count
        # No autograd graph of earlier eager steps may survive into the capture: a live graph keeps the parameters' AccumulateGrad
        # nodes -- bound to the stream they were created on, usually the default one -- and a capture that has to synchronise with the
        # default stream is invalid.  The dry forward above replaced the model's last state; collect what is left.
        import gc
        gc.collect()
        seeds.enable_device(dev, capacity=max(8, self.n_seeds))
        optimizer.enable_device_step(dev)
        self.graph = None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for i in range(max(1, warmup)):
                if i > 0:
                    self._run_pre_step(recluster)
                self.warm_result = self._body()          # (loss, parts) of the last eager step on the example batch
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # capture: the seeds / batch the captured kernels will read are whatever sits in the static buffers at replay time
        seeds.begin_step(self.n_seeds)
        self.graph = torch.cuda.CUDAGraph()
        self.opt.zero_grad(set_to_none=True)
        with torch.cuda.graph(self.graph):
            self._loss, self._parts = self._forward_backward_step()
        # the capture itself did not execute: the seeds drawn for it are consumed by the first replay
        self._primed = True

    # ---- the step -------------------------------------------------------------------------------------
    def _forward_backward_step(self) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        self.opt.zero_grad(set_to_none=True)
        loss, parts = self.model.cal_loss(self.static_batch)
        loss.backward()
        self.opt.step()
        return loss.detach(), {k: torch.as_tensor(v, device=self.device).detach() for k, v in parts.items()}

    def _run_pre_step(self, recluster: bool) -> None:
        if self._pre_step is not None:
            self._pre_step(bool(recluster))

    def _body(self):
        self.model._seeds.begin_step(self.n_seeds)
        return self._forward_backward_step()

    def __call__(self, batch: Sequence[torch.Tensor], recluster: bool = False) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """One training step on ``batch`` (same shapes as the example).  Returns the static loss tensors of the graph: read or copy
        them before the next call.  ``recluster``: the batch carries NCL's re-cluster flag (host-side: no device read here)."""
        self._run_pre_step(recluster)
        for dst, src in zip(self.static_batch, batch):
            dst.copy_(src, non_blocking=True)
        if self._primed:
            self._primed = False          # the seeds of the capture are still unused
        else:
            self.model._seeds.begin_step(self.n_seeds)
        self.graph.replay()
        return self._loss, self._parts

    def eager(self, batch: Sequence[torch.Tensor], recluster: bool = False):
        """The same step without the graph (a batch of another size, e.g. the last one of an epoch), same seed sequence and the
        same graph-safe path."""
        self._run_pre_step(recluster)
        if self._primed:
            self._primed = False
        else:
            self.model._seeds.begin_step(self.n_seeds)
        self.opt.zero_grad(set_to_none=True)
        loss, parts = self.model.cal_loss(list(batch))
        loss.backward()
        self.opt.step()
        return loss.detach(), parts

    def close(self) -> None:
        """Back to host-side seeds and step count (the sequence and the count continue) and to the model's eager path."""
        torch.cuda.synchronize(self.device)
        self.model._graph_mode = False
        self.model._seeds.disable_device()
        self.opt.disable_device_step()
        self.graph = None
