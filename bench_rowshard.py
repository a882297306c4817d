"""Row-sharded LightGCN training step on the BASELINE.json config-4 graph family (5 M x 1 M nodes, 150 M edges, d = 128,
L = 3: the whole graph trains on one 80 GB H100), used by bench.py: north_star's multi-GPU partition -- adjacency rows and the embedding table row-sharded over
the GPUs, the all-gather of each layer output fused into the SpMM epilogue as NVLink peer stores (sslrec_b200/parallel.py).

``leg(...)`` measures, on ``world`` GPUs, the graph scaled to world/8 of config 4 (per-GPU work fixed: weak scaling) and
reports the record bench.py attaches to every ``--gpus N`` line:
    {graph, nnz_per_rank, ms_per_step, spmm_ms, exchange_ms, nvlink_GBps, efficiency_weak, ...}
together with rank 0's single-GPU baselines measured in the same run (the 1/8 graph; at world = 8 also the full config 4
on ONE GPU, which gives the strong-scaling efficiency of the real config).
"""
from __future__ import annotations

import time

import torch

import synth_graphs as S

BATCH = 4096
DIM, LAYERS = 128, 3
EIGHTH = (625_000, 125_000, 18_750_000)            # |U|, |I|, E of one eighth of config 4


class DeviceGraphHandler:
    """The attributes a general_cf model reads from its data handler, for a graph that only exists as device arrays:
    no torch sparse COO tensor is ever built (config 4 has 300 M stored entries); ``plan_source`` hands the model the CSR
    of the row ranges it owns."""

    def __init__(self, keys: torch.Tensor, n_user: int, n_item: int):
        self.keys, self.n_user, self.n_item = keys, n_user, n_item
        self.torch_adj = None
        self.trn_mat = None
        self.last_plan = None

    def plan_source(self, device, ranges, side_split):
        from sslrec_b200.graph import GraphPlan
        rowptr, colidx, vals = S.normalized_csr_device(self.keys, self.n_user, self.n_item, ranges)
        self.last_plan = GraphPlan.from_csr(rowptr, colidx, vals, self.n_user + self.n_item, row_ranges=ranges, side_split=side_split)
        return self.last_plan


def _make_batches(keys, n_item, count, device, seed):
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    out = []
    for _ in range(count):
        pick = keys[torch.randint(0, keys.shape[0], (BATCH,), device=device, generator=g)]
        out.append([pick // n_item, pick % n_item, torch.randint(0, n_item, (BATCH,), device=device, generator=g)])
    return out


def _build(keys, n_user, n_item, dev, comm):
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.general_cf.lightgcn import LightGCN
    from sslrec_b200.optim import FusedAdam
    cfg = default_config('lightgcn', layer_num=LAYERS, embedding_size=DIM, reg_weight=1.0e-8, keep_rate=1.0, init_on_device=True)
    cfg['train']['batch_size'] = BATCH
    cfg['data'].update(user_num=n_user, item_num=n_item)
    load_config(base=cfg, device=str(dev))
    torch.manual_seed(2023)
    handler = DeviceGraphHandler(keys, n_user, n_item)
    model = LightGCN(handler).to(dev)
    if comm is not None:
        model.shard_to(comm)
    opt = FusedAdam(model.parameters(), lr=1e-3, row_shards=getattr(model, 'row_shards', None), comm=comm)
    return model, opt, handler


def _time_steps(model, opt, batches, steps, warmup, dist, dev):
    """(ms per step [max over ranks], kernel summary of `steps` further profiled steps)."""
    from sslrec_b200 import engine

    def step(i):
        opt.zero_grad()
        loss, _ = model.cal_loss(batches[i % len(batches)])
        loss.backward()
        opt.step()
        return loss

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    first = None
    for i in range(warmup):
        l = step(i)
        if i == 0:
            first = l
    barrier()
    first_loss = float(first.item()) if first is not None else None          # the loss of the very first step: same init, same batch on 1 and on N GPUs
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(warmup + i)
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1) / steps
    if dist is not None:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    # end to end: the batch comes from pinned host memory (H2D inside the timed region), the loss is read back every step
    host = [[t.cpu().pin_memory() for t in b] for b in batches[:4]]
    barrier()
    e0.record()
    for i in range(steps):
        opt.zero_grad()
        loss, _ = model.cal_loss([t.to(dev, non_blocking=True) for t in host[i % len(host)]])
        loss.backward()
        opt.step()
        loss.item()
    e1.record()
    barrier()
    ms_e2e = e0.elapsed_time(e1) / steps
    if dist is not None:
        t = torch.tensor([ms_e2e], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_e2e = float(t.item())
    engine.TIMER = engine.KernelTimer()
    n_prof = min(steps, 3)
    for i in range(n_prof):
        step(warmup + steps + i)
    barrier()
    summ = {k: dict(ms=v['ms'] / n_prof, launches=v['launches'] / n_prof) for k, v in engine.TIMER.summary().items()}
    engine.TIMER = None
    loss = float(step(0).item())
    summ['e2e_ms_per_step'] = ms_e2e
    summ['first_loss'] = first_loss
    return ms, summ, loss


def _single_gpu(keys, n_user, n_item, dev, steps, warmup):
    torch.cuda.reset_peak_memory_stats(dev)
    model, opt, handler = _build(keys, n_user, n_item, dev, None)
    batches = _make_batches(keys, n_item, steps + warmup, dev, 7)
    ms, summ, loss = _time_steps(model, opt, batches, steps, warmup, None, dev)
    stats = handler.last_plan.stats()
    nnz = handler.last_plan.nnz
    peak_gb = torch.cuda.max_memory_allocated(dev) / 1e9
    del model, opt, handler, batches
    torch.cuda.empty_cache()
    return dict(ms_per_step=ms, e2e_ms_per_step=summ['e2e_ms_per_step'], spmm_ms=summ.get('prop_fwd', {}).get('ms', 0.0) + summ.get('prop_bwd', {}).get('ms', 0.0),
                spmm_launches=summ.get('prop_fwd', {}).get('launches', 0) + summ.get('prop_bwd', {}).get('launches', 0), nnz=nnz, max_row_nnz=stats['max_row_nnz'], loss=loss, first_loss=summ['first_loss'],
                peak_mem_gb=peak_gb)


def leg(dist, rank, world, dev, steps=5, warmup=2, full=False, baselines=True, log=lambda *a: None):
    """The measurement (module docstring).  full=True: the whole config 4 regardless of ``world`` (strong scaling)."""
    from sslrec_b200.parallel import RowShard
    scale = 8 if full else world
    n_user, n_item, n_edge = (EIGHTH[0] * scale, EIGHTH[1] * scale, EIGHTH[2] * scale)
    t0 = time.perf_counter()
    # rank 0 generates, everyone receives the same sorted unique edge keys (1.2 GB at config 4: milliseconds over NVLink)
    if rank == 0:
        keys = S.bipartite_keys_device(n_user, n_item, n_edge, 2023, 1.0, dev)
    else:
        keys = torch.empty(n_edge, device=dev, dtype=torch.int64)
    if world > 1:
        dist.broadcast(keys, src=0)
    torch.cuda.synchronize()
    t_gen = time.perf_counter() - t0
    log(f'graph {n_user}x{n_item}, {n_edge} edges generated in {t_gen:.1f}s')
    N = n_user + n_item
    rec = {'graph': f'synthetic config-4 family x {scale}/8: |U|={n_user}, |I|={n_item}, nnz={2 * n_edge}, d={DIM}, L={LAYERS}, B={BATCH}, LightGCN (BPR + reg)',
           'gpus': world, 'graph_gen_s': t_gen, 'partition': 'rows of A and E sharded: each GPU owns a contiguous block of the user rows and one of the item rows, cut so that every GPU has the same number of stored entries (+4 per row); full tables replicated'}
    if world > 1:
        # block boundaries balanced by the rows' cost: stored entries (gathers) + a constant per row (epilogue, output row)
        from sslrec_b200.parallel import balanced_bounds
        ub = balanced_bounds(torch.bincount(keys // n_item, minlength=n_user).float() + 4.0, world)
        ib = balanced_bounds(torch.bincount(keys % n_item, minlength=n_item).float() + 4.0, world)
        comm = RowShard(dist, rank, world, N, n_user=n_user, shard_propagation=True, dim=DIM, views=1, user_bounds=ub, item_bounds=ib)
        rec['transport'] = comm.transport
        model, opt, handler = _build(keys, n_user, n_item, dev, comm)
        batches = _make_batches(keys, n_item, steps + warmup, dev, 7)
        for b in batches:                                   # one replicated batch per step
            for t in b:
                dist.broadcast(t, src=0)
        ms, summ, loss = _time_steps(model, opt, batches, steps, warmup, dist, dev)
        nnz_local = handler.last_plan.nnz
        nnz_all = torch.tensor([float(nnz_local)], device=dev)
        nnz_max = nnz_all.clone()
        dist.all_reduce(nnz_all)
        dist.all_reduce(nnz_max, op=dist.ReduceOp.MAX)
        spmm = summ.get('prop_fwd', {}).get('ms', 0.0) + summ.get('prop_bwd', {}).get('ms', 0.0)
        exch = summ.get('prop_exchange', {}).get('ms', 0.0)
        adam = summ.get('adam', {}).get('ms', 0.0)
        n_gather = int(round(summ.get('prop_exchange', {}).get('launches', 0)))
        peer_bytes = (n_gather + 1) * (world - 1) * comm.n_local * DIM * 4          # stored to peers per rank per step (+1: Adam)
        carrier_ms = spmm + adam
        rec.update({'ms_per_step': ms, 'e2e_ms_per_step': summ['e2e_ms_per_step'], 'steps_per_sec': 1e3 / ms, 'spmm_ms': spmm,
                    'spmm_launches': summ.get('prop_fwd', {}).get('launches', 0) + summ.get('prop_bwd', {}).get('launches', 0), 'rows_per_rank': comm.n_local, 'exchange_ms': exch, 'adam_ms': adam,
                    'allgathers_per_step': n_gather + 1, 'nnz_per_rank': nnz_local, 'nnz_imbalance': float(nnz_max.item() * world / nnz_all.item()),
                    'peer_bytes_per_rank_per_step': peer_bytes,
                    'nvlink_GBps': peer_bytes / (carrier_ms * 1e-3) / 1e9 if carrier_ms else None,
                    'how': 'spmm_ms = CUDA-event time of the 2L propagation launches (the peer stores of the fused all-gather travel inside them); '
                           'exchange_ms = what is left of the exchange after the launch (cross-GPU barrier; with the nccl transport the all_gather itself); '
                           'nvlink_GBps = bytes this rank stored into its peers per step / (spmm_ms + adam_ms)',
                    'loss': loss, 'first_loss': summ['first_loss'], 'steps': steps, 'warmup': warmup})
        rec['multicast'] = bool(comm._tables and next(iter(comm._tables.values())).mc_ptr)
        del model, opt, handler, batches
        comm._tables.clear()                                  # the shared tables (3.1 GB each at config 4) go before rank 0's one-GPU baselines
        comm._barrier_handle = None
        del comm
        import gc
        gc.collect()
        torch.cuda.empty_cache()
    if baselines:
        # rank 0 alone: one GPU on the 1/8 graph (what each GPU of the sharded run owns), and at the full size the whole graph on one GPU
        base = None
        if rank == 0:
            base = {}
            if not full:
                k8 = keys if scale == 1 else S.bipartite_keys_device(*EIGHTH, 2023, 1.0, dev)
                base['one_gpu_eighth'] = _single_gpu(k8, EIGHTH[0], EIGHTH[1], dev, steps, warmup)
                del k8
            if scale == 8 or world == 1:
                kf = keys if scale == 8 else S.bipartite_keys_device(EIGHTH[0] * 8, EIGHTH[1] * 8, EIGHTH[2] * 8, 2023, 1.0, dev)
                try:
                    base['one_gpu_config4'] = _single_gpu(kf, EIGHTH[0] * 8, EIGHTH[1] * 8, dev, max(2, steps // 2), 1)
                except Exception as e:      # noqa: BLE001 -- e.g. out of memory on a shared box: the sharded numbers stand without it
                    base['one_gpu_config4'] = {'error': repr(e)[:300]}
                del kf
            # 1-vs-N equality on the SAME graph: the first step's loss (same seed -> same initial table, same first batch)
            if world > 1 and 'first_loss' in rec:
                same = base.get('one_gpu_config4') if scale == 8 else None
                if same is None or 'first_loss' not in same:
                    try:
                        same = _single_gpu(keys, n_user, n_item, dev, 1, 1)
                        base['one_gpu_same_graph'] = {'first_loss': same['first_loss'], 'ms_per_step': same['ms_per_step']}
                    except Exception as e:      # noqa: BLE001
                        same = None
                        base['one_gpu_same_graph'] = {'error': repr(e)[:300]}
                if same is not None and same.get('first_loss') is not None:
                    rec['first_loss_one_gpu'] = same['first_loss']
                    rec['first_loss_abs_diff'] = abs(rec['first_loss'] - same['first_loss'])
        if world > 1:
            dist.barrier()
        if rank == 0:
            rec['baselines'] = base
            if world > 1 and 'ms_per_step' in rec:
                e = base.get('one_gpu_eighth')
                if e:
                    rec['efficiency_weak'] = e['ms_per_step'] / rec['ms_per_step']
                f = base.get('one_gpu_config4')
                if f and 'ms_per_step' in f and scale == 8:
                    rec['efficiency_strong'] = f['ms_per_step'] / (world * rec['ms_per_step'])
                    rec['speedup_vs_one_gpu_config4'] = f['ms_per_step'] / rec['ms_per_step']
    del keys
    torch.cuda.empty_cache()
    return rec
