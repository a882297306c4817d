"""HBM-bound measurement of the propagation kernel: a graph whose table is far larger than the 50 MB L2
(BASELINE.json config 4's per-GPU regime), forward layer launches timed with CUDA events on the launching stream.
Usage (GPU box): python tools/spmm_roofline.py [n_nodes] [avg_degree] [dim] [views]"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from sslrec_b200 import engine as E
from sslrec_b200.graph import GraphPlan

def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3_000_000
    deg = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    d = int(sys.argv[3]) if len(sys.argv) > 3 else 128
    V = int(sys.argv[4]) if len(sys.argv) > 4 else 1
    rng = np.random.Generator(np.random.PCG64(1))
    nu = n * 5 // 6                                   # users : items = 5 : 1 as in config 4 (10M : 2M)
    ni = n - nu
    e = n * deg // 2
    t0 = time.time()
    u = rng.integers(0, nu, size=e, dtype=np.int64)
    pop = rng.zipf(1.3, size=e) % ni                  # skewed item popularity (heavy rows exercise the split path)
    key = np.unique(u * ni + pop)
    u, it = key // ni, key % ni + nu
    rows, cols = np.concatenate([u, it]), np.concatenate([it, u])
    degs = np.bincount(rows, minlength=n).astype(np.float64) + 1e-10
    dinv = degs ** -0.5
    vals = (dinv[rows] * dinv[cols]).astype(np.float32)
    plan = GraphPlan(rows, cols, vals, n, torch.device('cuda'))
    print(f'graph: N={n} nnz={len(rows)} max_row={plan.stats()["max_row_nnz"]} split_rows={plan.stats()["split_rows"]} build {time.time()-t0:.1f}s', flush=True)
    x = torch.randn(n, V, d, device='cuda') * 0.1
    prop = E.Propagation(plan, [E.ViewSpec() for _ in range(V)], 1)
    out = torch.empty(n, V, d, device='cuda')
    a = prop._args(d, 1, False)
    a.in_views, a.x_in, a.x_out = V, x.data_ptr(), out.data_ptr()
    for _ in range(3):
        prop._launch(a, x)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        prop._launch(a, x)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    nnz = len(rows)
    alg = nnz * (8 + 4 * d * V) + n * (16 + 4 * d * V)
    compulsory = 2 * n * 4 * d * V + 8 * nnz + 16 * n
    peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))) if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else {'hbm_gbs': 6650.0}
    print(json.dumps({'kernel': 'prop_kernel forward layer', 'n_nodes': n, 'nnz': nnz, 'dim': d, 'views': V, 'table_MB': n * V * d * 4 / 1e6,
                      'ms': ms, 'alg_GBps': alg / ms / 1e6, 'compulsory_GBps': compulsory / ms / 1e6, 'peak_GBps': peaks['hbm_gbs'],
                      'frac_alg': alg / ms / 1e6 / peaks['hbm_gbs'], 'embeddings_propagated_per_sec': nnz * V / ms * 1e3}))

main()
