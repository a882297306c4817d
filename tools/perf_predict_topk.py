"""The fused evaluation ranking (``ssl_predict_topk``) against the two-kernel path (``ssl_predict_mask`` into a [n_b, n_item] score matrix,
then ``ssl_topk``), alternating the two in one process.  For every shape: CUDA-event milliseconds per batch over --reps launches of each
path after a warm-up (median and min), the speed-up, the peak allocated memory of each path (its own allocations: score matrix + outputs,
or workspace + outputs) and whether ids and value bits are equal.  Then the wall clock of Trainer.evaluate over all users of the amazon
shape (LightGCN, 3 layers, d = 64, 1024-user batches, mask from the device CSR), alternating the path Trainer.evaluate picks for that
shape (trainer.FUSED_TOPK_MIN_ITEMS), the fused path and the two-kernel path.  The card's name and
power limit are read in the same run.  One JSON line on stdout (and in --out).

    python tools/perf_predict_topk.py [--reps 30] [--out FILE] [--no-evaluate]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sslrec_b200._lib import check, lib  # noqa: E402

#          name            n_b   n_item   dim  k    training items per user in the CSR
SHAPES = [('amazon', 1024, 83761, 64, 40, 12),
          ('hccf_batch', 256, 83761, 64, 40, 12),
          ('gowalla_d32', 1024, 19747, 32, 40, 12),
          ('amazon_k256', 1024, 83761, 64, 256, 12),
          ('items_1m_d128', 1024, 1000000, 128, 40, 12),
          ('amazon_nomask', 1024, 83761, 64, 40, 0),
          ('hccf_batch_1m_d128', 256, 1000000, 128, 40, 12)]


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout else None}


def make_inputs(n_b, n_item, dim, deg, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    n_user = 76469
    ut = (torch.rand(n_user, dim, device='cuda', generator=g) - 0.5) * 0.2
    it = (torch.rand(n_item, dim, device='cuda', generator=g) - 0.5) * 0.2
    users = torch.randperm(n_user, device='cuda', generator=g)[:n_b].contiguous()
    cols = torch.randint(0, n_item, (n_user, deg), device='cuda', generator=g).sort(1).values      # duplicates allowed, rows sorted
    if deg == 0:
        return ut, it, users, None, None
    rowptr = torch.arange(0, (n_user + 1) * deg, deg, device='cuda', dtype=torch.int32)
    return ut, it, users, rowptr, cols.flatten().to(torch.int32).contiguous()


def _ptr(t):
    return None if t is None else t.data_ptr()


def pair(ut, it, users, n_item, dim, rowptr, cols, k, preds, idx, val):
    s = torch.cuda.current_stream().cuda_stream
    check(lib.ssl_predict_mask(ut.data_ptr(), ut.stride(0), it.data_ptr(), it.stride(0), users.data_ptr(), users.numel(), n_item, dim, None,
                               _ptr(rowptr), _ptr(cols), preds.data_ptr(), s), 'ssl_predict_mask')
    check(lib.ssl_topk(preds.data_ptr(), users.numel(), n_item, k, idx.data_ptr(), val.data_ptr(), s), 'ssl_topk')


def ws_bytes(n_b, n_item, k):
    b = C.c_int64(0)
    check(lib.ssl_predict_topk_workspace(n_b, n_item, k, C.byref(b)), 'ssl_predict_topk_workspace')
    return b.value


def fused(ut, it, users, n_item, dim, rowptr, cols, k, ws, idx, val):
    check(lib.ssl_predict_topk(ut.data_ptr(), ut.stride(0), it.data_ptr(), it.stride(0), users.data_ptr(), users.numel(), n_item, dim, None,
                               _ptr(rowptr), _ptr(cols), k, ws.data_ptr(), ws.numel(), idx.data_ptr(), val.data_ptr(),
                               torch.cuda.current_stream().cuda_stream), 'ssl_predict_topk')


def peak_of(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def shape_record(name, n_b, n_item, dim, k, deg, reps):
    ut, it, users, rowptr, cols = make_inputs(n_b, n_item, dim, deg, seed=n_item + dim + k)

    def pair_alloc():
        preds = torch.empty(n_b, n_item, device='cuda')
        idx = torch.empty(n_b, k, dtype=torch.int64, device='cuda')
        val = torch.empty(n_b, k, device='cuda')
        pair(ut, it, users, n_item, dim, rowptr, cols, k, preds, idx, val)
        return idx, val

    def fused_alloc():
        ws = torch.empty(ws_bytes(n_b, n_item, k), dtype=torch.uint8, device='cuda')
        idx = torch.empty(n_b, k, dtype=torch.int64, device='cuda')
        val = torch.empty(n_b, k, device='cuda')
        fused(ut, it, users, n_item, dim, rowptr, cols, k, ws, idx, val)
        return idx, val

    peak_pair, (ia, va) = peak_of(pair_alloc)
    peak_fused, (ib, vb) = peak_of(fused_alloc)
    equal = torch.equal(ia, ib) and torch.equal(va.view(torch.int32), vb.view(torch.int32))
    del ia, va, ib, vb
    preds = torch.empty(n_b, n_item, device='cuda')
    ws = torch.empty(ws_bytes(n_b, n_item, k), dtype=torch.uint8, device='cuda')
    idx = [torch.empty(n_b, k, dtype=torch.int64, device='cuda') for _ in range(2)]
    val = [torch.empty(n_b, k, device='cuda') for _ in range(2)]
    run = [lambda: pair(ut, it, users, n_item, dim, rowptr, cols, k, preds, idx[0], val[0]),
           lambda: fused(ut, it, users, n_item, dim, rowptr, cols, k, ws, idx[1], val[1])]
    for _ in range(3):
        for f in run:
            f()
    torch.cuda.synchronize()
    ms = [[], []]
    for _ in range(reps):
        for p, f in enumerate(run):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ms[p].append(a.elapsed_time(b))
    equal = equal and torch.equal(idx[0], idx[1]) and torch.equal(val[0].view(torch.int32), val[1].view(torch.int32))
    med = [statistics.median(m) for m in ms]
    rec = {'shape': name, 'n_b': n_b, 'n_item': n_item, 'dim': dim, 'k': k, 'train_items_per_user': deg, 'reps': reps,
           'pair_ms': med[0], 'pair_ms_min': min(ms[0]), 'fused_ms': med[1], 'fused_ms_min': min(ms[1]), 'speedup': med[0] / med[1],
           'peak_alloc_pair_mib': peak_pair / 2 ** 20, 'peak_alloc_fused_mib': peak_fused / 2 ** 20, 'equal': bool(equal)}
    del preds, ws
    torch.cuda.empty_cache()
    return rec


class TwoKernel:
    """A model seen through full_predict only: Trainer.evaluate ranks it with full_predict + topk."""

    def __init__(self, model):
        self.model = model

    def eval(self):
        self.model.eval()

    def full_predict(self, batch_data):
        return self.model.full_predict(batch_data)


def evaluate_record(rounds=3):
    import types

    import scipy.sparse as sp
    import torch.utils.data as tdata

    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import AllRankTstData, DataHandlerGeneralCF
    from sslrec_b200.general_cf.lightgcn import LightGCN
    from sslrec_b200 import trainer as T
    from sslrec_b200.trainer import Trainer
    from synth_graphs import named_graph
    rows, cols, n_user, n_item = named_graph('amazon', seed=2023)
    cfg = default_config('lightgcn', layer_num=3, embedding_size=64)
    cfg['test']['batch_size'] = 1024
    load_config(base=cfg, device='cuda')
    trn = sp.coo_matrix((np.ones(len(rows), dtype=np.float32), (rows, cols)), shape=(n_user, n_item))
    rs = np.random.RandomState(7)
    val = sp.coo_matrix((np.ones(n_user, dtype=np.float32), (np.arange(n_user), rs.randint(0, n_item, n_user))), shape=(n_user, n_item))
    dh = DataHandlerGeneralCF(trn)
    dh.load_data()
    model = LightGCN(dh).cuda()
    ld = tdata.DataLoader(AllRankTstData(val, trn, dense_mask=False), batch_size=1024, shuffle=False, num_workers=0)
    tr = Trainer(types.SimpleNamespace())
    secs = {'shipped': [], 'fused': [], 'pair': []}
    res = {}
    shipped_threshold = T.FUSED_TOPK_MIN_ITEMS
    for rep in range(rounds + 1):                 # round 0 warms up every path (eval-mode propagation, truth CSR, allocator)
        for key, m, thr in (('shipped', model, shipped_threshold), ('fused', model, 0), ('pair', TwoKernel(model), shipped_threshold)):
            T.FUSED_TOPK_MIN_ITEMS = thr
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[key] = tr.evaluate(m, loader=ld)
            torch.cuda.synchronize()
            if rep:
                secs[key].append(time.perf_counter() - t0)
    T.FUSED_TOPK_MIN_ITEMS = shipped_threshold
    same = all(np.array_equal(res[key][m], res['pair'][m]) for key in res for m in res['pair'])
    return {'users': n_user, 'n_item': n_item, 'batches': len(ld), 'k': cfg['test']['k'], 'rounds': rounds,
            'shipped_path': 'fused' if n_item >= shipped_threshold else 'pair',
            **{key + '_s': min(v) for key, v in secs.items()}, **{key + '_s_all': v for key, v in secs.items()},
            'metrics_equal': bool(same), 'recall': [float(v) for v in res['pair']['recall']]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-evaluate', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_predict_topk.py measures on a CUDA device; none is visible')
    torch.cuda.set_device(0)
    out = {'gpu': gpu_info(), 'shapes': [shape_record(*s, reps=args.reps) for s in SHAPES]}
    if not args.no_evaluate:
        out['trainer_evaluate_amazon'] = evaluate_record()
    out['gpu_after'] = gpu_info()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
