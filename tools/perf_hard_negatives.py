"""Cost of dynamic negative sampling (train.dns_candidates = M) on two of bench.py's workloads.

  python tools/perf_hard_negatives.py [--steps K] [--passes P] [--launches L] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings.
  * step: for SimGCL on the amazon shape and LightGCN on the gowalla shape, eager (cal_loss + backward + FusedAdam) and
    graph (GraphedStep replays), the time per step at M = 1, 2, 8, 32 and 64.  One model per M, built from the same seed,
    timed in alternating passes of K steps (CUDA events around each pass, after a warm-up pass of each), P passes each;
    the median pass and the ratio to M = 1.
  * launches: for each workload and M >= 2, the two new launches alone at the step's shapes, L launches captured in one
    CUDA graph and timed by CUDA events around its replay: ssl_neg_candidates on a batch, and ssl_neg_select on the rows the BPR term reads after a step
    (SimGCL: view 2 of the layer sum, computed at the marked rows only; LightGCN: the layer sum).  For SimGCL also the share of
    item rows its restricted views mark, with and without the candidates.
The workloads, graphs and batches are bench.py's (imported, not copied)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import bench  # noqa: E402
from sslrec_b200 import engine as E  # noqa: E402

WORKLOADS = ['simgcl-amazon', 'lightgcn-gowalla']
MS = [1, 2, 8, 32, 64]


def _model(workload, M, dev):
    import importlib
    import scipy.sparse as sp
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import DataHandlerGeneralCF
    from sslrec_b200.optim import FusedAdam
    model_name, graph, hp = bench.WORKLOADS[workload]
    rows, cols, n_user, n_item = bench.graph_arrays(graph)
    cfg = default_config(model_name, **hp)
    cfg['train'].update(batch_size=bench.BATCH, dns_candidates=M)
    load_config(base=cfg, device=str(dev))
    dh = DataHandlerGeneralCF(sp.coo_matrix((np.ones(len(rows), dtype=np.float32), (rows, cols)), shape=(n_user, n_item)))
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + model_name)
    cls = [getattr(mod, a) for a in dir(mod) if a.lower() == model_name][0]
    torch.manual_seed(2023)
    model = cls(dh).to(dev)
    return model, FusedAdam(model.parameters(), lr=1e-3, weight_decay=0)


class _Arm:
    """One model with train.dns_candidates = M: eager steps, or replays of a GraphedStep captured with it."""

    def __init__(self, workload, driver, M, batches, dev):
        self.batches = batches
        self.model, self.opt = _model(workload, M, dev)
        self.graph = None
        if driver == 'graph':
            from sslrec_b200.graphed import GraphedStep
            self.graph = GraphedStep(self.model, self.opt, batches[0], warmup=2)

    def step(self, i):
        b = self.batches[i % len(self.batches)]
        if self.graph is not None:
            return self.graph(b)
        self.opt.zero_grad()
        loss, parts = self.model.cal_loss(b)
        loss.backward()
        self.opt.step()
        return loss, parts

    def timed_pass(self, K):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(K):
            self.step(i)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / K

    def close(self):
        if self.graph is not None:
            self.graph.close()


def _batches(workload, count, dev):
    rows, cols, _, n_item = bench.graph_arrays(bench.WORKLOADS[workload][1])
    return [[torch.from_numpy(x).to(dev) for x in b] for b in bench.make_batches(rows, cols, n_item, count)]


def step_record(workload, driver, K, passes, dev):
    batches = _batches(workload, max(K, 8), dev)
    arms = {}
    for M in MS:
        arms[M] = _Arm(workload, driver, M, batches, dev)
        arms[M].timed_pass(K)                          # warm-up: every shape of the timed window
    per = {M: [] for M in MS}
    for _ in range(passes):
        for M in MS:
            per[M].append(arms[M].timed_pass(K))
    for arm in arms.values():
        arm.close()
    med = {M: sorted(v)[len(v) // 2] for M, v in per.items()}
    return {'record': 'step', 'workload': workload, 'driver': driver, 'steps_per_pass': K,
            'ms': {str(M): med[M] for M in MS}, 'ratio_to_m1': {str(M): med[M] / med[1] for M in MS},
            'passes_ms': {str(M): per[M] for M in MS}}


def _time(fn, L):
    """Microseconds per launch of ``fn``: L launches captured in one CUDA graph and replayed between two events, so the time is
    the device's and not the host's enqueue rate."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(L):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / L


def _marked_item_share(st, v, n_user, n_item):
    bits = st.prop.views[v].row_bits.to(torch.int64)
    rows = torch.arange(n_user, n_user + n_item, device=bits.device)
    return float(((bits[rows >> 5] >> (rows & 31)) & 1).float().mean().item())


def launch_record(workload, L, dev):
    batch = _batches(workload, 1, dev)[0]
    view = 2 if workload.startswith('simgcl') else 0
    out = {'record': 'launches', 'workload': workload, 'launches': L, 'batch': bench.BATCH, 'us': {}}
    for M in MS[1:]:
        model, opt = _model(workload, M, dev)
        opt.zero_grad()
        model.cal_loss(batch)[0].backward()           # the step's state: the rows the selection reads
        st = model._state
        ancs, negs = batch[0], batch[2]
        rowptr, cols = model._train_csr(dev)
        cands = E.neg_candidates(ancs, negs, M, rowptr, cols, model.item_num, 12345)
        users, items = st.users(view), st.items(view)
        d = model.embedding_size
        rec = {'neg_candidates_us': _time(lambda: E.neg_candidates(ancs, negs, M, rowptr, cols, model.item_num, 12345), L),
               'neg_select_us': _time(lambda: E.hard_negatives(users, items, ancs, cands), L),
               'select_gathered_bytes': bench.BATCH * M * (8 + 4 * d)}
        if workload.startswith('simgcl'):
            rec['marked_item_share'] = _marked_item_share(st, view, model.user_num, model.item_num)
        out['us'][str(M)] = rec
        del model, opt, st, users, items
        torch.cuda.empty_cache()
    if workload.startswith('simgcl'):
        model, opt = _model(workload, 1, dev)
        model.cal_loss(batch)
        out['marked_item_share_m1'] = _marked_item_share(model._state, view, model.user_num, model.item_num)
        del model, opt
    return out


def card_record():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return {'record': 'card', 'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--out')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_hard_negatives.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload in WORKLOADS:
        for driver in ('eager', 'graph'):
            recs.append(step_record(workload, driver, args.steps, args.passes, dev))
            print(json.dumps(recs[-1]), flush=True)
            torch.cuda.empty_cache()
        recs.append(launch_record(workload, args.launches, dev))
        print(json.dumps(recs[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in recs))


if __name__ == '__main__':
    main()
