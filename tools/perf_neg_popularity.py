"""Cost of popularity-proportional candidates (train.neg_popularity) on two of bench.py's workloads.

  python tools/perf_neg_popularity.py [--steps K] [--passes P] [--launches L] [--out FILE]

Prints one JSON line per record (and writes them to FILE when given):
  * card: the GPU's name, power limit and maximum SM clock, read in the same run as the timings (at the start and the end).
  * step: for SimGCL on the amazon shape and LightGCN on the gowalla shape, the time per step as a CUDA graph (GraphedStep
    replays) of the sampled softmax loss (tau = 0.1) at M = 8, 64 and 256, with uniform candidates and with
    train.neg_popularity = 0.75.  One model per configuration, built from the same seed, timed in alternating passes of K steps
    (CUDA events around each pass, after a warm-up pass of each), P passes each; the median pass and the popularity/uniform ratio.
  * launches: at the step's shapes (B = bench.BATCH, the first bench batch) for M = 8, 64, 256: ssl_neg_candidates against
    ssl_neg_candidates_pop (with the bias), and ssl_ssm_fwd against ssl_ssm_fwd_logq, L launches of each captured in one CUDA
    graph and timed by CUDA events around its replay.  With them, the expected number of draws per drawn candidate at the
    batch's users, from the tables: (1 - (1 - a_u)^cap) / a_u with a_u the acceptance probability of one draw ((n_item - deg_u) /
    n_item uniform with cap 256, Z_u = exp(lz_pop[u]) popularity with cap 128), averaged over the batch.
  * table_build: engine.pop_tables on the host (seconds, wall clock, best of three) at the amazon shape and at 1 M items.
The workloads, graphs and batches are bench.py's (imported, not copied)."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import bench  # noqa: E402
import perf_hard_negatives as PH  # noqa: E402
import perf_mixgcf as PM  # noqa: E402
from sslrec_b200 import engine as E  # noqa: E402
from sslrec_b200._lib import lib  # noqa: E402

WORKLOADS = ['simgcl-amazon', 'lightgcn-gowalla']
TAU, BETA = 0.1, 0.75
MS = (8, 64, 256)
CONFIGS = {}
for _m in MS:
    CONFIGS['uni%d' % _m] = dict(ssm_temperature=TAU, dns_candidates=_m)
    CONFIGS['pop%d' % _m] = dict(ssm_temperature=TAU, dns_candidates=_m, neg_popularity=BETA)


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
    return {'record': 'step', 'workload': workload, 'driver': 'graph', 'beta': BETA, 'tau': TAU, 'steps_per_pass': K, 'ms': med,
            'pop_over_uniform': {str(M): med['pop%d' % M] / med['uni%d' % M] for M in MS}, 'passes_ms': per}


def _csr(workload):
    rows, cols, n_user, n_item = bench.graph_arrays(bench.WORKLOADS[workload][1])
    m = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_user, n_item))
    m.sum_duplicates()
    m.sort_indices()
    return m, n_user, n_item


def _expected_draws(a, cap):
    a = np.asarray(a, np.float64)
    return np.where(a > 0, (1 - (1 - a) ** cap) / np.maximum(a, 1e-300), cap)


def launch_record(workload, L, dev):
    m, n_user, n_item = _csr(workload)
    host = E.pop_tables(m.indptr, m.indices, n_item, BETA)
    pop = E.PopTables(m.indptr, m.indices, n_item, BETA, dev)
    rowptr = torch.from_numpy(m.indptr.astype(np.int32)).to(dev)
    cols = torch.from_numpy(m.indices.astype(np.int32)).to(dev)
    ancs, poss, negs = PH._batches(workload, 1, dev)[0][:3]
    B = ancs.numel()
    u = ancs.cpu().numpy()
    deg = np.diff(m.indptr)[u]
    draws = {'uniform': float(_expected_draws((n_item - deg) / n_item, 256).mean()),
             'popularity': float(_expected_draws(np.exp(host['lz_pop'][u].astype(np.float64)), 128).mean())}
    out = {'record': 'launches', 'workload': workload, 'launches': L, 'batch': B, 'beta': BETA, 'tau': TAU,
           'expected_draws_per_candidate': draws, 'kernels': {}}
    g = torch.Generator(device='cpu').manual_seed(0)
    d = 64
    users_t = torch.randn(n_user, d, generator=g).to(dev)
    items_t = torch.randn(n_item, d, generator=g).to(dev)
    st = lambda: torch.cuda.current_stream().cuda_stream
    for M in MS:
        cands = torch.empty(B, M, dtype=torch.int64, device=dev)
        bias = torch.empty(B, M, dtype=torch.float32, device=dev)
        ln_m = float(np.float32(math.log(M)))
        f = dict(device=dev, dtype=torch.float32)
        loss_b, s, w, nrm = torch.empty(B, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 1, **f), torch.empty(B, M + 2, **f)

        def uni():
            assert lib.ssl_neg_candidates(ancs.data_ptr(), negs.data_ptr(), B, M, rowptr.data_ptr(), cols.data_ptr(), n_item, 12345, None,
                                          cands.data_ptr(), st()) == 0

        def popc():
            assert lib.ssl_neg_candidates_pop(ancs.data_ptr(), negs.data_ptr(), B, M, rowptr.data_ptr(), cols.data_ptr(), n_item,
                                              pop.table.data_ptr(), pop.lp.data_ptr(), pop.lz_pop.data_ptr(), pop.lz_uni.data_ptr(), ln_m,
                                              12345, None, cands.data_ptr(), bias.data_ptr(), st()) == 0

        def fwd():
            assert lib.ssl_ssm_fwd(users_t.data_ptr(), d, items_t.data_ptr(), d, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(), B, M,
                                   d, TAU, loss_b.data_ptr(), s.data_ptr(), w.data_ptr(), nrm.data_ptr(), st()) == 0

        def fwd_logq():
            assert lib.ssl_ssm_fwd_logq(users_t.data_ptr(), d, items_t.data_ptr(), d, ancs.data_ptr(), poss.data_ptr(), cands.data_ptr(),
                                        B, M, d, TAU, loss_b.data_ptr(), s.data_ptr(), w.data_ptr(), nrm.data_ptr(), bias.data_ptr(),
                                        st()) == 0

        popc()
        rec = {}
        for _ in range(3):              # alternate the arms; keep each one's best of three
            for name, fn in (('candidates_uniform', uni), ('candidates_pop', popc), ('ssm_fwd', fwd), ('ssm_fwd_logq', fwd_logq)):
                popc()
                us = PH._time(fn, L)
                rec[name + '_us'] = min(us, rec.get(name + '_us', us))
        out['kernels'][str(M)] = rec
    return out


def table_build_record():
    out = {'record': 'table_build', 'beta': BETA, 'seconds': {}}
    m, _, n_item = _csr('simgcl-amazon')
    cases = {'amazon': (m.indptr, m.indices, n_item)}
    rs = np.random.RandomState(4)
    n = 1_000_000
    rows = rs.randint(0, 200_000, 10_000_000)
    cols = (rs.zipf(1.1, 10_000_000) - 1) % n
    big = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(200_000, n))
    big.sum_duplicates()
    big.sort_indices()
    cases['1M_items_200k_users'] = (big.indptr, big.indices, n)
    for name, (ip, ix, ni) in cases.items():
        best = math.inf
        for _ in range(3):
            t = time.perf_counter()
            E.pop_tables(ip, ix, ni, BETA)
            best = min(best, time.perf_counter() - t)
        out['seconds'][name] = best
        out.setdefault('nnz', {})[name] = int(len(ix))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--out')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_neg_popularity.py measures on a GPU; none is visible')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    recs = [PH.card_record()]
    print(json.dumps(recs[-1]), flush=True)
    for workload in WORKLOADS:
        for make in (lambda: launch_record(workload, args.launches, dev), lambda: step_record(workload, args.steps, args.passes, dev)):
            recs.append(make())
            print(json.dumps(recs[-1]), flush=True)
            torch.cuda.empty_cache()
    recs.append(table_build_record())
    print(json.dumps(recs[-1]), flush=True)
    recs.append(PH.card_record())
    print(json.dumps(recs[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(r) + '\n' for r in recs))


if __name__ == '__main__':
    main()
