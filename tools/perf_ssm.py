"""Cost of the sampled softmax loss (train.ssm_temperature) on two of bench.py's workloads.

  python tools/perf_ssm.py [--steps K] [--passes P] [--launches L] [--records step,launches,in_batch] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings.
  * step: for SimGCL on the amazon shape and LightGCN on the gowalla shape, the time per step as a CUDA graph (GraphedStep
    replays) of five configurations: plain, and the sampled softmax loss (tau = 0.1) with M = 1, 8, 64 and 256.  One model per
    configuration, built from the same seed, timed in alternating passes of K steps (CUDA events around each pass, after a
    warm-up pass of each), P passes each; the median pass and the ratio to the plain step.
  * launches: ssl_ssm_fwd and ssl_ssm_bwd alone at the step's shapes (B = bench.BATCH, the rows the loss reads) for M = 1, 8,
    64, 256: L launches of each captured in one CUDA graph and timed by CUDA events around its replay; the algorithmic bytes
    of each, B (M + 2) 4d (every row read once; the backward's gradient adds are not counted), and the achieved GB/s.
  * in_batch: the in-batch softmax (train.ssm_in_batch, a sixth step configuration above) at the step's shapes: every launch
    of engine.ssm_in_batch_sum alone, timed as above (the two operand builds, the weight gather, the weighted forward
    contraction, its epilogue and sum, the colscale, the swapped contraction and the three gradient kernels); the kernel kind
    the forward took and the weights' range that chose it; each contraction's useful FLOP, 2 GEMMs of 2 B 2B d, its rate and,
    with the 3 MMAs per product of a 3x split (1 for FFMA), the rate of MMA work against the data-sheet dense rate of that
    kind (H100 SXM: FP16 989, TF32 495, FP32 67 TFLOP/s); and the bytes the term allocates (the CUDA caching allocator's
    peak over one forward and backward, above what was allocated before it).
The workloads, graphs and batches are bench.py's (imported, not copied)."""
import argparse
import json
import math
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
           'ssm64': dict(ssm_temperature=TAU, dns_candidates=64), 'ssm256': dict(ssm_temperature=TAU, dns_candidates=256),
           'inbatch': dict(ssm_temperature=TAU, ssm_in_batch=True)}
DATASHEET_TFLOPS = dict(f16x3=989.0, tf32x3=495.0, ffma=67.0)        # dense, H100 SXM at 700 W
MMAS_PER_PRODUCT = dict(f16x3=3, tf32x3=3, ffma=1)


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


def in_batch_record(workload, L, dev):
    batch = PH._batches(workload, 1, dev)[0]
    view = 2 if workload.startswith('simgcl') else 0
    model, opt = PM._model(workload, CONFIGS['inbatch'], dev)
    opt.zero_grad()
    model.cal_loss(batch)[0].backward()
    st = model._state
    users, items = st.users(view), st.items(view)
    ancs, poss, negs = (E._i64(t, dev) for t in batch[:3])
    weights = model._in_batch_weights(dev)
    B, d = ancs.numel(), users.dim
    tau, off = TAU, E.LOG2E / TAU
    kind = E.contraction_kind(d, off, colscale_range=weights.range)
    f = dict(device=dev, dtype=torch.float32)
    s = torch.cuda.current_stream().cuda_stream
    cols = torch.cat([poss, negs])
    a = E._operand(users, ancs, 0, off, s, kind, streamed=True)
    t = E._operand(items, cols, 0, 1.0, s, kind, streamed=True)
    w = torch.zeros(t.npad, **f)
    torch.div(weights.v.index_select(0, cols), B, out=w[:2 * B])
    ns_f, ns_b = E._n_split(a, t), E._n_split(t, a)
    rs_part, o_part = torch.zeros(ns_f, B, **f), torch.zeros(ns_f, B, d, **f)
    rowsum, obar, loss_b, out = torch.empty(B, **f), torch.empty(B, d, **f), torch.empty(B, **f), torch.empty((), **f)
    colscale, dt_part = torch.zeros(a.npad, **f), torch.empty(ns_b, 2 * B, d, **f)
    g = torch.ones((), **f)
    g_u, g_i = torch.zeros(model.user_num, d, **f), torch.zeros(model.item_num, d, **f)
    rows = lambda: (a.hat.data_ptr(), t.hat.data_ptr(), obar.data_ptr(), a.rinv.data_ptr(), t.rinv.data_ptr())
    cs = lambda: torch.cuda.current_stream().cuda_stream         # the capturing stream inside a timed graph
    launches = {
        'normalize_users': lambda: E._operand(users, ancs, 0, off, cs(), kind, streamed=True),
        'normalize_columns': lambda: E._operand(items, cols, 0, 1.0, cs(), kind, streamed=True),
        'weight_gather': lambda: torch.div(weights.v.index_select(0, cols), B, out=w[:2 * B]),
        'contract_fwd': lambda: E._contract(a, t, w, off, ns_f, rs_part, o_part, cs(), bwd=False),
        'finalize': lambda: lib.ssl_nce_finalize(rs_part.data_ptr(), o_part.data_ptr(), ns_f, B, d, a.hat.data_ptr(), t.hat.data_ptr(),
                                                 tau, 0.0, rowsum.data_ptr(), obar.data_ptr(), loss_b.data_ptr(), cs()),
        'sum': lambda: lib.ssl_sum(loss_b.data_ptr(), B, 1.0, out.data_ptr(), cs()),
        'colscale': lambda: lib.ssl_nce_colscale(rowsum.data_ptr(), B, g.data_ptr(), 1.0, colscale.data_ptr(), cs()),
        'contract_bwd': lambda: E._contract(t, a, colscale, off, ns_b, None, dt_part, cs(), bwd=True),
        'bwd_rows_users': lambda: lib.ssl_nce_bwd_rows(*rows(), ancs.data_ptr(), B, d, tau, g.data_ptr(), 1e-6, g_u.data_ptr(), d, None, 0,
                                                       cs()),
        'bwd_rows_positives': lambda: lib.ssl_nce_bwd_rows(*rows(), poss.data_ptr(), B, d, tau, g.data_ptr(), 1e-6, None, 0, g_i.data_ptr(),
                                                           d, cs()),
        'bwd_cols': lambda: lib.ssl_nce_bwd_cols(dt_part.data_ptr(), ns_b, t.hat.data_ptr(), t.rinv.data_ptr(), w.data_ptr(), cols.data_ptr(),
                                                 2 * B, d, g_i.data_ptr(), d, cs()),
    }
    for name in ('contract_fwd', 'finalize', 'colscale', 'contract_bwd'):     # fill what the later launches read
        launches[name]()
    us = {name: PH._time(fn, L) for name, fn in launches.items()}
    flop = 2 * (2 * B * 2 * B * d)
    rates = {}
    for name in ('contract_fwd', 'contract_bwd'):
        tf = flop / (us[name] * 1e-6) / 1e12
        rates[name] = {'useful_TFLOPs': tf, 'mma_TFLOPs': tf * MMAS_PER_PRODUCT[kind],
                       'share_of_datasheet': tf * MMAS_PER_PRODUCT[kind] / DATASHEET_TFLOPS[kind]}
    # bytes the term allocates: the allocator's peak over one forward and backward, above what was allocated before
    U = users.base.view(-1, users.n_views, d)[users.off:users.off + users.n, users.v].contiguous().requires_grad_(True)
    I = items.base.view(-1, items.n_views, d)[items.off:items.off + items.n, items.v].contiguous().requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    E.ssm_in_batch_sum(U, I, ancs, poss, negs, tau, weights).backward()
    torch.cuda.synchronize()
    term_bytes = torch.cuda.max_memory_allocated() - base - (U.numel() + I.numel()) * 4     # the two tables' gradients are not the term's
    del model, opt, st
    torch.cuda.empty_cache()
    return {'record': 'in_batch', 'workload': workload, 'launches': L, 'batch': B, 'dim': d, 'tau': tau, 'kind': kind,
            'weight_range': weights.range, 'rule_offset': off + 0.5 * (1 + math.log2(weights.range)), 'n_split': [ns_f, ns_b],
            'launch_us': us, 'total_us': sum(us.values()), 'contraction_flop': flop, 'contraction_rates': rates,
            'term_alloc_bytes': term_bytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--records', default='step,launches,in_batch', help='which records to take, comma-separated')
    ap.add_argument('--out')
    args = ap.parse_args()
    want = set(args.records.split(','))
    if not torch.cuda.is_available():
        raise SystemExit('perf_ssm.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [PH.card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload in WORKLOADS:
        for name, fn in (('step', lambda: step_record(workload, args.steps, args.passes, dev)),
                         ('launches', lambda: launch_record(workload, args.launches, dev)),
                         ('in_batch', lambda: in_batch_record(workload, args.launches, dev))):
            if name not in want:
                continue
            rec = fn()
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
