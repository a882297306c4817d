"""Cost of the sampled softmax loss (train.ssm_temperature) on two of bench.py's workloads.

  python tools/perf_ssm.py [--steps K] [--passes P] [--launches L] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings.
  * step: for SimGCL on the amazon shape and LightGCN on the gowalla shape, the time per step as a CUDA graph (GraphedStep
    replays) of five configurations: plain, and the sampled softmax loss (tau = 0.1) with M = 1, 8, 64 and 256.  One model per
    configuration, built from the same seed, timed in alternating passes of K steps (CUDA events around each pass, after a
    warm-up pass of each), P passes each; the median pass and the ratio to the plain step.
  * launches: ssl_ssm_fwd and ssl_ssm_bwd alone at the step's shapes (B = bench.BATCH, the rows the loss reads) for M = 1, 8,
    64, 256: L launches of each captured in one CUDA graph and timed by CUDA events around its replay; the algorithmic bytes
    of each, B (M + 2) 4d (every row read once; the backward's gradient adds are not counted), and the achieved GB/s.
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
import perf_mixgcf as PM  # noqa: E402
from sslrec_b200 import engine as E  # noqa: E402
from sslrec_b200._lib import lib  # noqa: E402

WORKLOADS = ['simgcl-amazon', 'lightgcn-gowalla']
TAU = 0.1
CONFIGS = {'plain': dict(), 'ssm1': dict(ssm_temperature=TAU), 'ssm8': dict(ssm_temperature=TAU, dns_candidates=8),
           'ssm64': dict(ssm_temperature=TAU, dns_candidates=64), 'ssm256': dict(ssm_temperature=TAU, dns_candidates=256)}


class _Arm(PH._Arm):
    def __init__(self, workload, train, batches, dev):
        from sslrec_b200.graphed import GraphedStep
        self.batches = batches
        self.model, self.opt = PM._model(workload, train, dev)
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


def launch_record(workload, L, dev):
    batch = PH._batches(workload, 1, dev)[0]
    view = 2 if workload.startswith('simgcl') else 0
    out = {'record': 'launches', 'workload': workload, 'launches': L, 'batch': bench.BATCH, 'tau': TAU, 'kernels': {}}
    for M in (1, 8, 64, 256):
        model, opt = PM._model(workload, CONFIGS['ssm%d' % M], dev)
        opt.zero_grad()
        model.cal_loss(batch)[0].backward()
        st = model._state
        ancs, poss = batch[0], batch[1]
        cands = model._dns_candidates(ancs, batch[2]).cands
        u_ptr, u_stride, d = E._score_table(st.users(view))
        i_ptr, i_stride, _ = E._score_table(st.items(view))
        B = ancs.numel()
        f = dict(device=dev, dtype=torch.float32)
        loss_b, s, w, nrm = torch.empty(B, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 2, **f)
        g_u, g_i = torch.zeros(model.user_num, d, **f), torch.zeros(model.item_num, d, **f)
        one = torch.ones((), **f)

        def fwd():
            assert lib.ssl_ssm_fwd(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, M, d, TAU,
                                   loss_b.data_ptr(), s.data_ptr(), w.data_ptr(), nrm.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0

        def bwd():
            assert lib.ssl_ssm_bwd(u_ptr, u_stride, i_ptr, i_stride, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, M, d, TAU,
                                   s.data_ptr(), w.data_ptr(), nrm.data_ptr(), one.data_ptr(), 1e-6, g_u.data_ptr(), d, g_i.data_ptr(), d,
                                   torch.cuda.current_stream().cuda_stream) == 0

        fwd()
        nbytes = B * (M + 2) * 4 * d
        rec = {'bytes': nbytes}
        for name, fn in (('fwd', fwd), ('bwd', bwd)):
            us = PH._time(fn, L)
            rec[name + '_us'] = us
            rec[name + '_GBps'] = nbytes / (us * 1e-6) / 1e9
        out['kernels'][str(M)] = rec
        del model, opt, st
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
        raise SystemExit('perf_ssm.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [PH.card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload in WORKLOADS:
        for rec in (step_record(workload, args.steps, args.passes, dev), launch_record(workload, args.launches, dev)):
            recs.append(rec)
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()
    recs.append(PH.card_record())
    print(json.dumps(recs[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in recs))


if __name__ == '__main__':
    main()
