"""Cost of MixGCF negatives (train.mixgcf) on two of bench.py's workloads.

  python tools/perf_mixgcf.py [--steps K] [--passes P] [--launches L] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings.
  * step: for SimGCL on the amazon shape and LightGCN on the gowalla shape, the time per step as a CUDA graph (GraphedStep
    replays) of five configurations: plain, DNS with M = 8, and MixGCF with M = 1, 8 and 64.  One model per configuration,
    built from the same seed, timed in alternating passes of K steps (CUDA events around each pass, after a warm-up pass of
    each), P passes each; the median pass and the ratio to the plain step.
  * kernels: per configuration, the device time of one eager step's launches bracketed by engine.KernelTimer (median over P
    steps): the forward propagation launches (prop_fwd; for SimGCL they compute the last layer at every row under MixGCF, since
    the kept layer drops the row restriction) and the two MixGCF launches (mixgcf_fwd with its sum, mixgcf_bwd with the
    ordered scatters when deterministic).
  * launches: ssl_mixgcf_bpr_fwd (with its sum) alone at the step's shapes for M = 1, 8, 64: L launches captured in one CUDA
    graph and timed by CUDA events around its replay.
The workloads, graphs and batches are bench.py's (imported, not copied)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import bench  # noqa: E402
import perf_hard_negatives as PH  # noqa: E402
from sslrec_b200 import engine as E  # noqa: E402

WORKLOADS = ['simgcl-amazon', 'lightgcn-gowalla']
CONFIGS = {'plain': dict(), 'dns8': dict(dns_candidates=8), 'mix1': dict(mixgcf=True), 'mix8': dict(mixgcf=True, dns_candidates=8),
           'mix64': dict(mixgcf=True, dns_candidates=64)}


def _model(workload, train, dev):
    """perf_hard_negatives._model with the configuration's train keys."""
    from sslrec_b200.config import configs
    import sslrec_b200.config as cfgmod
    default = cfgmod.default_config

    def with_train(name, **kw):
        cfg = default(name, **kw)
        cfg['train'].update(train)
        return cfg

    cfgmod.default_config = with_train
    try:
        model, opt = PH._model(workload, train.get('dns_candidates', 1), dev)
    finally:
        cfgmod.default_config = default
    assert configs['train'].get('mixgcf', False) == train.get('mixgcf', False)
    return model, opt


class _Arm(PH._Arm):
    def __init__(self, workload, train, batches, dev):
        from sslrec_b200.graphed import GraphedStep
        self.batches = batches
        self.model, self.opt = _model(workload, train, dev)
        self.graph = GraphedStep(self.model, self.opt, batches[0], warmup=2)


def step_record(workload, K, passes, dev):
    batches = PH._batches(workload, max(K, 8), dev)
    arms = {}
    for name, train in CONFIGS.items():
        arms[name] = _Arm(workload, train, batches, dev)
        arms[name].timed_pass(K)
    per = {name: [] for name in CONFIGS}
    for _ in range(passes):
        for name in CONFIGS:
            per[name].append(arms[name].timed_pass(K))
    for arm in arms.values():
        arm.close()
    med = {n: sorted(v)[len(v) // 2] for n, v in per.items()}
    return {'record': 'step', 'workload': workload, 'driver': 'graph', 'steps_per_pass': K, 'ms': med,
            'ratio_to_plain': {n: med[n] / med['plain'] for n in CONFIGS}, 'passes_ms': per}


def kernel_record(workload, passes, dev):
    batches = PH._batches(workload, passes + 2, dev)
    out = {'record': 'kernels', 'workload': workload, 'steps': passes, 'ms': {}}
    for name, train in CONFIGS.items():
        model, opt = _model(workload, train, dev)
        samples = []
        for i, b in enumerate(batches):
            E.TIMER = E.KernelTimer() if i >= 2 else None
            opt.zero_grad()
            model.cal_loss(b)[0].backward()
            opt.step()
            torch.cuda.synchronize()
            if E.TIMER is not None:
                samples.append({k: v['ms'] for k, v in E.TIMER.summary().items()})
        E.TIMER = None
        keys = sorted({k for s in samples for k in s})
        out['ms'][name] = {k: sorted(s.get(k, 0.0) for s in samples)[len(samples) // 2] for k in keys}
        del model, opt
        torch.cuda.empty_cache()
    return out


def launch_record(workload, L, dev):
    batch = PH._batches(workload, 1, dev)[0]
    view = 2 if workload.startswith('simgcl') else 0
    out = {'record': 'launches', 'workload': workload, 'launches': L, 'batch': bench.BATCH, 'us': {}}
    for M in (1, 8, 64):
        model, opt = _model(workload, CONFIGS['mix%d' % M], dev)
        opt.zero_grad()
        model.cal_loss(batch)[0].backward()
        st = model._state
        ancs, poss = batch[0], batch[1]
        cands = model._dns_candidates(ancs, batch[2]).cands
        users, items = st.users(view), st.items(view)
        layers = [st.items(view, k) for k in range(model.layer_num + 1)]

        def fwd():
            with torch.no_grad():
                return E.mixgcf_bpr_sum(users, items, layers, ancs, poss, cands, 12345)

        out['us'][str(M)] = {'fwd_us': PH._time(fwd, L)}
        del model, opt, st, users, items, layers
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--out')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_mixgcf.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [PH.card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload in WORKLOADS:
        for rec in (step_record(workload, args.steps, args.passes, dev), kernel_record(workload, args.passes, dev),
                    launch_record(workload, args.launches, dev)):
            recs.append(rec)
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in recs))


if __name__ == '__main__':
    main()
