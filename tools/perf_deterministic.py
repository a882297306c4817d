"""Cost of train.deterministic (the ordered scatter of batch-row gradients) and what it buys, on bench.py's workloads.

  python tools/perf_deterministic.py [--steps K] [--passes P] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings.
  * step: for each workload and driver (eager = cal_loss + backward + FusedAdam; graph = GraphedStep replays) the time per step
    with the key off and on.  Off and on are two models built from the same seed, timed in alternating passes of K steps
    (CUDA events around each pass, after a warm-up pass of each), P passes each; the median pass and the ratio on / off.
  * repeat: at the bench shape (simgcl-amazon), two fresh key-off runs and two fresh key-on runs of the same batches; whether
    each pair's loss, loss terms and updated parameters are bit-equal, and the largest parameter difference.  A report, not an
    assertion.
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

CASES = [('simgcl-amazon', 'eager'), ('simgcl-amazon', 'graph'), ('lightgcn-gowalla', 'graph'), ('hccf-amazon', 'eager'),
         ('lightgcl-gowalla', 'eager'), ('directau-gowalla', 'eager')]


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
    load_config(base=cfg, device=str(dev))
    dh = DataHandlerGeneralCF(sp.coo_matrix((np.ones(len(rows), dtype=np.float32), (rows, cols)), shape=(n_user, n_item)))
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + model_name)
    cls = [getattr(mod, a) for a in dir(mod) if a.lower() == model_name][0]
    torch.manual_seed(2023)
    model = cls(dh).to(dev)
    return model, FusedAdam(model.parameters(), lr=1e-3, weight_decay=0), (rows, cols, n_user, n_item)


class _Arm:
    """One model driven with the key fixed to ``det``: eager steps, or replays of a GraphedStep captured under that key."""

    def __init__(self, workload, driver, det, batches, dev):
        self.det, self.batches = det, batches
        E.DETERMINISTIC = det
        self.model, self.opt, _ = _model(workload, dev)
        self.graph = None
        if driver == 'graph':
            from sslrec_b200.graphed import GraphedStep
            self.graph = GraphedStep(self.model, self.opt, batches[0], warmup=2)

    def step(self, i):
        b = self.batches[i % len(self.batches)]
        if self.graph is not None:
            return self.graph(b)
        E.DETERMINISTIC = self.det
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


def step_record(workload, driver, K, passes, dev):
    rows, cols, _, n_item = bench.graph_arrays(bench.WORKLOADS[workload][1])
    batches = [[torch.from_numpy(x).to(dev) for x in b] for b in bench.make_batches(rows, cols, n_item, max(K, 8))]
    arms = {det: _Arm(workload, driver, det, batches, dev) for det in (False, True)}
    for arm in arms.values():
        arm.timed_pass(K)                                  # warm-up: every shape of the timed window
    per = {False: [], True: []}
    for _ in range(passes):
        for det in (False, True):
            per[det].append(arms[det].timed_pass(K))
    for arm in arms.values():
        arm.close()
    med = {det: sorted(v)[len(v) // 2] for det, v in per.items()}
    return {'record': 'step', 'workload': workload, 'driver': driver, 'steps_per_pass': K,
            'off_ms': med[False], 'on_ms': med[True], 'ratio_on_off': med[True] / med[False],
            'off_passes_ms': per[False], 'on_passes_ms': per[True]}


def repeat_record(steps, dev):
    workload = 'simgcl-amazon'
    rows, cols, _, n_item = bench.graph_arrays(bench.WORKLOADS[workload][1])
    batches = [[torch.from_numpy(x).to(dev) for x in b] for b in bench.make_batches(rows, cols, n_item, steps)]
    out = {'record': 'repeat', 'workload': workload, 'steps': steps}
    for det in (False, True):
        runs = []
        for _ in range(2):
            arm = _Arm(workload, 'eager', det, batches, dev)
            for i in range(steps):
                loss, parts = arm.step(i)
            torch.cuda.synchronize()
            runs.append((loss.detach().clone(), {k: torch.as_tensor(v, device=dev).detach().clone() for k, v in parts.items()},
                         [p.detach().clone() for p in arm.model.parameters()]))
            del arm
        (l0, t0, p0), (l1, t1, p1) = runs
        out['on' if det else 'off'] = {
            'bit_equal': bool(torch.equal(l0, l1) and all(torch.equal(t0[k], t1[k]) for k in t0) and all(torch.equal(a, b) for a, b in zip(p0, p1))),
            'loss': [l0.item(), l1.item()],
            'max_abs_param_diff': max((a - b).abs().max().item() for a, b in zip(p0, p1))}
    return out


def card_record():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return {'record': 'card', 'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--repeat-steps', type=int, default=5)
    ap.add_argument('--out')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_deterministic.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload, driver in CASES:
        recs.append(step_record(workload, driver, args.steps, args.passes, dev))
        print(json.dumps(recs[-1]), flush=True)
        torch.cuda.empty_cache()
    recs.append(repeat_record(args.repeat_steps, dev))
    print(json.dumps(recs[-1]), flush=True)
    E.DETERMINISTIC = None
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in recs))


if __name__ == '__main__':
    main()
