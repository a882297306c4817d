"""Graphed against eager training steps for the models whose batches bench.py --impl graph does not drive, and the HCCF numbers
behind the count-bounded spec-node term.

  python tools/perf_graph_models.py [--steps K]

Prints one JSON line per record:
  * ncl-amazon: eager steps (cal_loss + backward + FusedAdam) against GraphedStep replays, on batches without the k-means flag
    (the re-clustering batches run k-means eagerly on both paths); median of 5 passes of K steps, CUDA events.
  * hccf-amazon: the mean unique fraction of users and items per batch, and the forward spec-node contraction
    (ssl_softmax_gemm_tf32x3_live, R = the padded anchor list, C = the side's table) bounded by the live count against the same
    launch with the count at capacity.
The workloads, graphs and batches are bench.py's (imported, not copied)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import bench  # noqa: E402


def _model(workload, dev):
    import importlib
    import scipy.sparse as sp
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import DataHandlerGeneralCF
    from sslrec_b200.optim import FusedAdam
    model_name, graph, hp = bench.WORKLOADS[workload]
    rows, cols, n_user, n_item = bench.graph_arrays(graph)
    cfg = default_config(model_name, **hp)
    cfg['train']['batch_size'] = bench.BATCH
    if model_name == 'ncl':
        cfg['train']['loss'] = 'pairwise_with_epoch_flag'
    load_config(base=cfg, device=str(dev))
    dh = DataHandlerGeneralCF(sp.coo_matrix((np.ones(len(rows), dtype=np.float32), (rows, cols)), shape=(n_user, n_item)))
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + model_name)
    cls = [getattr(mod, a) for a in dir(mod) if a.lower() == model_name][0]
    torch.manual_seed(2023)
    model = cls(dh).to(dev)
    return model, FusedAdam(model.parameters(), lr=1e-3, weight_decay=0), (rows, cols, n_user, n_item)


def _passes(fn, K, n=5):
    per = []
    for _ in range(n):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(K):
            fn(i)
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) / K)
    per.sort()
    return {'ms_per_step': per[len(per) // 2], 'passes_ms': per}


def ncl_steps(K, dev):
    from sslrec_b200.graphed import GraphedStep
    model, opt, (rows, cols, n_user, n_item) = _model('ncl-amazon', dev)
    flags = torch.zeros(bench.BATCH, dtype=torch.int64, device=dev)
    batches = [[b[0], b[1], b[2], flags] for b in (torch.from_numpy(x).to(dev) for x in bench.make_batches(rows, cols, n_item, K + 3))]

    def eager(i):
        opt.zero_grad()
        loss, _ = model.cal_loss(batches[i % len(batches)])
        loss.backward()
        opt.step()
    eager(0)                                   # the first step clusters
    res = {'eager': _passes(eager, K)}
    gs = GraphedStep(model, opt, batches[0], warmup=3)
    res['graph'] = _passes(lambda i: gs(batches[i % len(batches)]), K)
    gs.close()
    return {'workload': 'ncl-amazon', 'steps': K, **res, 'speedup': res['eager']['ms_per_step'] / res['graph']['ms_per_step']}


def hccf_contraction(K, dev):
    from sslrec_b200 import engine as E
    from sslrec_b200._lib import check, lib
    rows, cols, n_user, n_item = bench.graph_arrays(bench.WORKLOADS['hccf-amazon'][1])
    batches = bench.make_batches(rows, cols, n_item, K)
    fu = float(np.mean([np.unique(b[0]).size / b[0].size for b in batches]))
    fi = float(np.mean([np.unique(b[1]).size / b[1].size for b in batches]))
    out = {'workload': 'hccf-amazon', 'batch': bench.BATCH, 'unique_fraction_users': fu, 'unique_fraction_items': fi}
    d, B = bench.WORKLOADS['hccf-amazon'][2]['embedding_size'], bench.BATCH
    g = torch.Generator(device=dev).manual_seed(0)
    for side, n, frac in (('users', n_user, fu), ('items', n_item, fi)):
        def split(x):
            npad = max(64, E.ceil_to(x.shape[0], 64))
            f = dict(device=dev, dtype=torch.float32)
            o, hi, lo, thi, tlo = (torch.empty(npad, d, **f), torch.empty(npad, d, **f), torch.empty(npad, d, **f),
                                   torch.empty(d, npad, **f), torch.empty(d, npad, **f))
            check(lib.ssl_rows_normalize(x.data_ptr(), d, None, x.shape[0], d, 1, 1.0, o.data_ptr(), None, None, hi.data_ptr(), lo.data_ptr(),
                                         thi.data_ptr(), tlo.data_ptr(), npad, torch.cuda.current_stream().cuda_stream))
            return hi, lo, thi, tlo, npad
        a = split(torch.randn(B, d, device=dev, generator=g))
        t = split(torch.randn(n, d, device=dev, generator=g))
        n_split = E.choose_split((B + 127) // 128, t[4] // 64, slots=E.NUM_SM, prefer_few=True)
        rs, o = torch.zeros(n_split, B, device=dev), torch.zeros(n_split, B, d, device=dev)
        rec = {}
        for name, live in (('bounded', int(round(frac * B))), ('capacity', B)):
            lv = torch.tensor(live, dtype=torch.int64, device=dev)

            def launch(_):
                check(lib.ssl_softmax_gemm_tf32x3_live(a[0].data_ptr(), a[1].data_ptr(), B, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(),
                                                       t[3].data_ptr(), t[4], n, d, None, E.LOG2E / 0.1, n_split, rs.data_ptr(), o.data_ptr(),
                                                       lv.data_ptr(), E.LIVE_ROWS, torch.cuda.current_stream().cuda_stream))
            launch(0)
            rec[name] = {'live': live, **_passes(launch, 20)}
        out[side] = {'n': n, 'n_split': n_split, **rec, 'ratio': rec['bounded']['ms_per_step'] / rec['capacity']['ms_per_step']}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    gpu = bench.gpu_identity(0)
    print(json.dumps({'gpu': gpu, **hccf_contraction(args.steps, dev)}), flush=True)
    print(json.dumps({'gpu': gpu, **ncl_steps(args.steps, dev)}), flush=True)


if __name__ == '__main__':
    main()
