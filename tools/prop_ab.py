"""A/B of the propagation kernel's two thread mappings on the bench's amazon-shaped graph (d = 64, 3 views): the interleaved
mapping (a thread accumulates all views of its row: one pass over the CSR, 768 B per gathered row, 123 MB gather set) against
the view-major one (grid.y = view: 41 MB gather set per view phase, three passes over the CSR).  Launch shapes are those of
a SimGCL step: layer >= 2 forward (per-view inputs, layer output + nothing else) and the transposed backward with residual;
plus the SGL shape (per-view RNG edge masks).  Usage (GPU box):  python tools/prop_ab.py [reps] [--ncu]
Under ncu pass --ncu (3 launches per variant, no timing loop)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, scipy.sparse as sp, torch
import synth_graphs as S
from sslrec_b200 import engine as E
from sslrec_b200._lib import check, lib
from sslrec_b200.data_handler import normalized_adjacency
from sslrec_b200.graph import GraphPlan


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 20
    ncu = '--ncu' in sys.argv
    name = 'amazon'
    cache = f'/tmp/sslrec_b200_graph_{name}.npz'
    if os.path.exists(cache):
        z = np.load(cache); rows, cols, nu, ni = z['rows'], z['cols'], int(z['n_user']), int(z['n_item'])
    else:
        rows, cols, nu, ni = S.named_graph(name)
    r, c, v, n = normalized_adjacency(sp.coo_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(nu, ni)))
    plan = GraphPlan(r, c, v, n, torch.device('cuda'), side_split=nu)
    d, V = 64, 3
    x = torch.randn(n, V, d, device='cuda') * 0.1
    res = torch.randn(n, V, d, device='cuda') * 0.1
    out = torch.empty(n, V, d, device='cuda')
    out2 = torch.empty(n, d, device='cuda')
    shapes = {}
    plain = E.Propagation(plan, [E.ViewSpec() for _ in range(V)], 2)
    a = plain._args(d, 2, False); a.in_views, a.x_in, a.x_out = V, x.data_ptr(), out.data_ptr()
    shapes['fwd layer>=2 (per-view in, x_out)'] = (plain, a)
    b = plain._args(d, 2, True); b.in_views, b.x_in, b.x_out, b.residual = V, x.data_ptr(), out.data_ptr(), res.data_ptr()
    shapes['bwd layer (transposed, residual, x_out)'] = (plain, b)
    masked = E.Propagation(plan, [E.ViewSpec(edge_mode=1, keep=0.5, seed=11), E.ViewSpec(edge_mode=1, keep=0.5, seed=12), E.ViewSpec()], 2)
    c_ = masked._args(d, 2, False); c_.in_views, c_.x_in, c_.x_out = V, x.data_ptr(), out.data_ptr()
    shapes['fwd SGL (2 RNG edge masks + clean view)'] = (masked, c_)
    e_ = plain._args(d, 1, True); e_.in_views, e_.x_in, e_.sum_out, e_.reduce_views, e_.residual = V, x.data_ptr(), out2.data_ptr(), 1, res.data_ptr()
    shapes['bwd last layer (reduce over views; interleaved only)'] = (plain, e_)
    # the HBM-bound regime: one GPU's eighth of BASELINE config 4 (1.5 M nodes, 75 M entries, d = 128, one view)
    if '--xl' in sys.argv or '--xlfull' in sys.argv:
        sc = 8 if '--xlfull' in sys.argv else 1            # --xlfull: the whole BASELINE config 4 (6 M nodes, 300 M entries, 3.1 GB table)
        nu_x, ni_x = 1_250_000 * sc, 250_000 * sc
        keys = S.bipartite_keys_device(nu_x, ni_x, 37_500_000 * sc, 2023, 1.0, 'cuda')
        rp, ci, va = S.normalized_csr_device(keys, nu_x, ni_x)
        del keys
        xplan = GraphPlan.from_csr(rp, ci, va, nu_x + ni_x, side_split=nu_x)
        xx = torch.randn(nu_x + ni_x, 1, 128, device='cuda') * 0.1
        xo = torch.empty_like(xx)
        xp = E.Propagation(xplan, [E.ViewSpec()], 2)
        xa = xp._args(128, 2, False); xa.in_views, xa.x_in, xa.x_out = 1, xx.data_ptr(), xo.data_ptr()
        shapes = {('config-4' if sc == 8 else 'xl-8th') + f' fwd (d=128, 1 view, {75 * sc} M entries)': (xp, xa)}
        x, d, V, plan = xx, 128, 1, xplan
    nnz = plan.nnz
    combos = [('interleaved', 0), ('view-major', 1)]
    if ncu and ('--xl' in sys.argv or '--xlfull' in sys.argv):
        combos = combos[:1]
    for what, (prop, args) in shapes.items():
        for mode, vm in combos:
            check(lib.ssl_set_option(b'prop_view_major', vm))
            if ncu:
                for _ in range(3):
                    prop._launch(args, x)
                torch.cuda.synchronize()
                continue
            for _ in range(5):
                prop._launch(args, x)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                prop._launch(args, x)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            gather = nnz * (8 + 4 * d * V)
            print(json.dumps({'shape': what, 'mode': mode, 'ms': round(ms, 4), 'gather_TBps': round(gather / ms / 1e9, 2)}), flush=True)
    check(lib.ssl_set_option(b'prop_view_major', 0))


main()
