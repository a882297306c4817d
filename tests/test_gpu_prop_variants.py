"""Parity net of the propagation kernel (ssl_propagate_layer, sslrec_b200/csrc/propagate.cu) over every variant its
launcher selects, on one graph whose rows fall into every work-list class (isolated, whole, split into 128-, 256- and
384-entry segments).  Each launch is compared per view with a float64 restatement; the properties the kernel's fixed
summation order makes exact are checked with torch.equal.

Which prop_kernel<G, V, MODE, VM> instantiation each case reaches:

    G      from dim / 4: G4 -- 4, 12 (idle lanes), 16; G8 -- 20 (idle), 32; G16 -- 36, 48 (idle), 64;
           G32 -- 68, 124 (idle), 128
    V      1..4: the first V of the four view configurations below
    MODE 0 shared_noise (every V)
    MODE 1 views_noise, epilogue_residual (V >= 2; with one view they are MODE 0)
    MODE 2 mixed_in1 / mixed_in1_T / mixed_inV / mixed_inV_T, epilogue, reduce_T (every V)
    VM     every MODE 1 / MODE 2 case at V >= 2 except reduce_T (the launcher never picks it for a reduced launch):
           <G, 1, 1, true> and <G, 1, 2, true>, required bit-identical to the interleaved launch

That a V-view launch equals V one-view launches of its views is checked at every dim, V = 2..4 and MODE 0 / 1 / 2 by
tests/test_gpu_kernels.py::test_three_views_share_layer_one_and_match_single_views.
"""
import contextlib
import ctypes as C
from dataclasses import dataclass

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cf_oracle as O
from oracle import inputs
from oracle import philox as P

pytestmark = pytest.mark.gpu

N_USER, N_ITEM, N_EDGE = 17000, 1500, 50000
USER_HUBS = (128, 129)                      # degrees of the added user rows (a user has at most N_ITEM partners)
ITEM_HUBS = (128, 129, 4096, 4097, 16385)   # whole row, shortest split row, 128-, 256- and 384-entry segments
N_ISOLATED = 4                              # rows per side kept at degree 0
DIMS = (4, 12, 16, 20, 32, 36, 48, 64, 68, 124, 128)

# the four view configurations: (edge_mode, keep, scale), noise_mode, seed.  View 0 reads its seed from a device word
# (ssl_prop_args.seed_ptr, the CUDA-graph path) while the seed argument holds DECOY.
EDGE = ((1, 0.5, 2.0), (0, 1.0, 1.0), (2, 0.5, 2.0), (1, 0.8, 1.25))
NOISE = (1, 2, 0, 1)
SEEDS = (0x1234_5678_9ABC_DEF1, 0x0BAD_CAFE_0000_0002, 0x0000_0000_0000_0003, 0x7EDC_BA98_7654_3210)
DECOY = 0x5555_5555_5555_5555
EPS = 0.1                    # noise_eps
REG_G = 0.37                 # the device regulariser coefficient (reg_coef_dev); reg_coef = 2
TAU, TAU_ABS = 1e-5, 1e-7    # |got - ref| <= TAU * (|A| |x| + |other terms|) + TAU_ABS


@dataclass(frozen=True)
class Case:
    inv: bool = False          # per-view inputs (in_views = V) instead of one shared input
    edges: bool = False        # the mixed per-view edge modes of EDGE
    noise: bool = False        # the per-view noise of NOISE (forward launches only)
    transpose: bool = False
    residual: bool = False
    sums: bool = False         # x_out and sum_out, two sum_src entries (one with 1 view, one with V)
    reduce: bool = False       # last backward layer: views reduced into sum_out + 2 g E0 + src2


CASES = {
    'shared_noise': Case(noise=True, sums=True),
    'views_noise': Case(inv=True, noise=True),
    'mixed_in1': Case(edges=True),
    'mixed_in1_T': Case(edges=True, transpose=True),
    'mixed_inV': Case(inv=True, edges=True),
    'mixed_inV_T': Case(inv=True, edges=True, transpose=True),
    'epilogue': Case(inv=True, edges=True, noise=True, sums=True),
    'epilogue_residual': Case(inv=True, noise=True, residual=True, sums=True),
    'reduce_T': Case(inv=True, edges=True, transpose=True, residual=True, reduce=True),
}
RATIOS = {}                  # launch shape -> largest err / scale seen


def _set_option(name, value):
    from sslrec_b200._lib import check, lib
    check(lib.ssl_set_option(name, int(value)), 'ssl_set_option')


@contextlib.contextmanager
def _view_major():
    _set_option(b'prop_view_major', 1)
    try:
        yield
    finally:
        _set_option(b'prop_view_major', 0)


def _vm_eligible(c, V):
    """ssl_propagate_layer runs the view-major kernel when the option is on, V >= 2, views are not reduced and the inputs
    are per view or the launch masks edges."""
    return V >= 2 and not c.reduce and (c.inv or c.edges)


class Graph:
    def __init__(self):
        from sslrec_b200.graph import GraphPlan
        rows, cols = inputs.bipartite_edges(N_USER, N_ITEM, N_EDGE, 41)
        rs = np.random.RandomState(42)
        free_u, free_i = np.setdiff1d(np.arange(N_USER), rows), np.setdiff1d(np.arange(N_ITEM), cols)
        hub_u, iso_u = free_u[:len(USER_HUBS)], free_u[-N_ISOLATED:]
        hub_i, iso_i = free_i[:len(ITEM_HUBS)], free_i[-N_ISOLATED:]
        pool_u = np.setdiff1d(np.arange(N_USER), np.concatenate([hub_u, iso_u]))
        pool_i = np.setdiff1d(np.arange(N_ITEM), np.concatenate([hub_i, iso_i]))
        rows, cols = [rows], [cols]
        for u, d in zip(hub_u, USER_HUBS):         # partners without replacement: no pair collapses in the adjacency
            rows.append(np.full(d, u))
            cols.append(rs.choice(pool_i, d, replace=False))
        for i, d in zip(hub_i, ITEM_HUBS):
            rows.append(rs.choice(pool_u, d, replace=False))
            cols.append(np.full(d, i))
        self.adj = adj = O.normalized_adjacency(np.concatenate(rows), np.concatenate(cols), N_USER, N_ITEM)
        assert (adj.vals > 0).all()                # |A| = A below
        self.plan = plan = GraphPlan(adj.rows, adj.cols, adj.vals, adj.n, torch.device('cuda'), need_rev=True, side_split=N_USER)
        deg = np.diff(plan.h_rowptr.astype(np.int64))
        assert tuple(deg[hub_u]) == USER_HUBS and tuple(deg[N_USER + hub_i]) == ITEM_HUBS
        assert (deg[iso_u] == 0).all() and (deg[N_USER + iso_i] == 0).all()
        st = plan.stats()
        assert st['max_row_nnz'] == max(ITEM_HUBS) and st['split_rows'] == int((deg > 128).sum()) >= 4
        self.isolated = torch.from_numpy(np.flatnonzero(deg == 0)).cuda()
        # edge masks in the adjacency's entry order (= CSR order): Philox for the RNG views, a random draw for the injected view
        self.masks = [P.edge_keep(SEEDS[0], 0, adj.rows, adj.cols, EDGE[0][1]), None, rs.rand(adj.nnz) < EDGE[2][1],
                      P.edge_keep(SEEDS[3], 0, adj.rows, adj.cols, EDGE[3][1])]
        self.mask_dev = [None if m is None else plan.mask_to_csr(m) for m in self.masks]
        self.seed_dev = torch.tensor([SEEDS[0]], dtype=torch.int64, device='cuda')
        self.coef_dev = torch.tensor([REG_G], dtype=torch.float32, device='cuda')
        self._mat = {}
        self._prod, self._prod_tag = {}, None

    def matrix(self, v, transpose):
        """float64 A_v (view v's EdgeDrop, or the plain adjacency for v = None), transposed if asked."""
        if (v, transpose) not in self._mat:
            a = O.edge_dropped(self.adj, None if v is None else self.masks[v], 1.0 if v is None else EDGE[v][1], True, torch.float64)
            a = a.coalesce()
            self._mat[(v, transpose)] = a.t().coalesce() if transpose else a
        return self._mat[(v, transpose)]

    def product(self, tag, v, transpose, x):
        """(A_v x, A_v |x|) in float64, cached for one (dim, case) at a time: reused across V and the view-major launch."""
        if tag != self._prod_tag:
            self._prod, self._prod_tag = {}, tag
        key = (v, transpose, x.data_ptr())
        if key not in self._prod:
            x = x.cpu().double()
            both = torch.sparse.mm(self.matrix(v, transpose), torch.cat([x, x.abs()], 1))
            self._prod[key] = both[:, :x.shape[1]], both[:, x.shape[1]:]
        return self._prod[key]

    def spec(self, v, c, I):
        from sslrec_b200 import engine as E
        em, keep, scale = EDGE[v] if c.edges else (0, 1.0, 1.0)
        nm = NOISE[v] if c.noise else 0
        return E.ViewSpec(edge_mode=em, keep=keep, scale=scale, edge_masks=self.mask_dev[v] if em == 2 else None,
                          noise_mode=nm, noise_u=[I.u1] if nm == 2 else None, seed=SEEDS[v])


class Inputs:
    """Seeded fp32 operands of one dim at model magnitudes (randn * 0.1), on the GPU; [N, 4, d] tables hold all four views."""

    def __init__(self, n, dim):
        g = torch.Generator().manual_seed(1000 + dim)
        r = lambda *s: (torch.randn(*s, generator=g) * 0.1).cuda()
        self.dim = dim
        self.x1, self.x4, self.res4, self.s1, self.s4 = r(n, dim), r(n, 4, dim), r(n, 4, dim), r(n, 1, dim), r(n, 4, dim)
        self.e0, self.src2 = r(n, dim), r(n, dim)
        self.u1 = torch.rand(n, dim, generator=g).cuda()           # view 1's injected noise uniforms
        self._u = {}

    def noise_u(self, v):
        """View v's noise uniforms of layer 1: injected, or the Philox draws the kernel makes."""
        if NOISE[v] == 2:
            return self.u1.cpu().double()
        if v not in self._u:
            self._u[v] = torch.from_numpy(P.noise_uniform(SEEDS[v], 1, self.x1.shape[0], self.dim)).double()
        return self._u[v]


_INPUTS = {}


def _inputs(n, dim):
    if dim not in _INPUTS:
        _INPUTS.clear()
        _INPUTS[dim] = Inputs(n, dim)
    return _INPUTS[dim]


@pytest.fixture(scope='module')
def graph():
    yield Graph()
    _INPUTS.clear()
    if RATIOS:
        print('\nlargest err / scale per launch shape (bound %.0e):' % TAU)
        for k, r in sorted(RATIOS.items()):
            print(f'  {k:20s} {r:.3e}')


def _launch(g, I, views, c, specs=None):
    """One ssl_propagate_layer launch of the views `views` (indices into the four configurations) -> its output tables."""
    from sslrec_b200 import engine as E
    V, d, n = len(views), I.dim, g.adj.n
    specs = specs if specs is not None else [g.spec(v, c, I) for v in views]
    prop = E.Propagation(g.plan, specs, 1, noise_eps=EPS)
    a = prop._args(d, 1, c.transpose)
    if 0 in views:
        a.seed_ptr[views.index(0)] = g.seed_dev.data_ptr()
        a.seed[views.index(0)] = DECOY
    live = []

    def per_view(t):
        t = t[:, views].contiguous()
        live.append(t)
        return t.data_ptr()
    a.in_views = V if c.inv else 1
    a.x_in = per_view(I.x4) if c.inv else I.x1.data_ptr()
    if c.residual:
        a.residual = per_view(I.res4)
    out = {}
    if c.reduce:
        out['sum'] = torch.full((n, d), float('nan'), device='cuda')
        a.sum_out, a.reduce_views = out['sum'].data_ptr(), 1
        a.reg_src, a.reg_coef, a.reg_coef_dev, a.reg_src2 = I.e0.data_ptr(), 2.0, g.coef_dev.data_ptr(), I.src2.data_ptr()
    else:
        out['x'] = torch.full((n, V, d), float('nan'), device='cuda')
        a.x_out = out['x'].data_ptr()
        if c.sums:
            out['sum'] = torch.full((n, V, d), float('nan'), device='cuda')
            a.sum_out, a.n_sum_src = out['sum'].data_ptr(), 2
            a.sum_src[0], a.sum_src_views[0] = I.s1.data_ptr(), 1
            a.sum_src[1], a.sum_src_views[1] = per_view(I.s4), V
    prop._launch(a, I.x1)
    torch.cuda.synchronize()
    return out


def _reference(g, I, views, c, tag):
    """float64 (value, scale, slack) of every output table.  scale = the same sums over magnitudes; slack is 2 eps |u| / ||u||
    where the pre-noise value is within the bound of 0, so fp32 may see the other sign and move the noise with it."""
    xs, ss, ks = [], [], []
    for v in views:
        x_in = I.x4[:, v] if c.inv else I.x1
        val, scale = g.product(tag, v if c.edges and EDGE[v][0] else None, c.transpose, x_in)
        slack = torch.zeros_like(val)
        if c.residual:
            r = I.res4[:, v].cpu().double()
            val, scale = val + r, scale + r.abs()
        if c.noise and NOISE[v] and not c.transpose:
            u = I.noise_u(v)
            un = F.normalize(u, p=2, dim=1).abs() * EPS
            slack = torch.where(val.abs() <= TAU * scale + TAU_ABS, 2 * un, slack)
            val, scale = O.perturbed(val, u, EPS), scale + un
        xs.append(val), ss.append(scale), ks.append(slack)
    x, xsc, xk = torch.stack(xs, 1), torch.stack(ss, 1), torch.stack(ks, 1)
    ref = {}
    if c.reduce:
        coef = 2.0 * float(g.coef_dev.item())
        e0, s2 = I.e0.cpu().double(), I.src2.cpu().double()
        ref['sum'] = (x.sum(1) + coef * e0 + s2, xsc.sum(1) + coef * e0.abs() + s2.abs(), xk.sum(1))
        return ref
    ref['x'] = (x, xsc, xk)
    if c.sums:
        s1, s4 = I.s1.cpu().double(), I.s4[:, views].cpu().double()
        ref['sum'] = (x + s1 + s4, xsc + s1.abs() + s4.abs(), xk)
    return ref


def _check(got, want, what):
    val, scale, slack = want
    got = got.cpu().double()
    err = (got - val).abs()
    bad = ~(err <= TAU * scale + TAU_ABS + slack)            # NaN (a row never written) is bad too
    assert not bad.any(), (f'{what}: {int(bad.sum())} / {bad.numel()} off, worst at {np.unravel_index(int((err - TAU * scale).argmax()), err.shape)}; '
                           f'max err {err.max():.3e}')
    on = (scale > 0) & (slack == 0)
    return float((err[on] / scale[on]).max()) if on.any() else 0.0


@pytest.mark.parametrize('dim,case,V', [(d, c, V) for d in DIMS for c in CASES for V in (1, 2, 3, 4)])
def test_layer_matches_float64(graph, dim, case, V):
    """Each view of one launch against float64 A_v x (+ residual, noise, layer sums, or the reduced last backward layer);
    rows of degree 0 exactly; and the view-major kernel bit-identical to the interleaved one wherever the launcher picks it."""
    c = CASES[case]
    I = _inputs(graph.adj.n, dim)
    views = list(range(V))
    out = _launch(graph, I, views, c)
    ref = _reference(graph, I, views, c, (dim, case))
    for k in out:
        r = _check(out[k], ref[k], f'{case} {k} dim={dim} V={V}')
        RATIOS[case] = max(RATIOS.get(case, 0.0), r)
    # isolated rows without a residual: a zero accumulator, which noise (sgn(0) = 0) does not move; the layer sum is then the
    # fp32 sum of the sources in order
    iso = graph.isolated
    if not c.residual and not c.reduce:
        assert torch.equal(out['x'][iso], torch.zeros_like(out['x'][iso]))
        if c.sums:
            assert torch.equal(out['sum'][iso], (I.s1 + I.s4[:, views])[iso])
    if _vm_eligible(c, V):
        with _view_major():
            vm = _launch(graph, I, views, c)
        for k in out:
            assert torch.equal(vm[k], out[k]), f'view-major {k} differs from the interleaved launch'


@pytest.mark.parametrize('dim', DIMS)
def test_rng_edge_masks_equal_injected_at_four_views(graph, dim):
    """edge_mode 1 (Philox keep test in the kernel) == edge_mode 2 with oracle/philox.py's masks, four views with mixed keeps
    in one launch, forward and transposed, interleaved and view-major."""
    from sslrec_b200 import engine as E
    I = _inputs(graph.adj.n, dim)
    keeps = (0.5, 0.8, 0.5, 0.8)
    adj = graph.adj
    rng = [E.ViewSpec(edge_mode=1, keep=k, scale=1.0 / k, seed=s) for k, s in zip(keeps, SEEDS)]
    inj = [E.ViewSpec(edge_mode=2, keep=k, scale=1.0 / k, edge_masks=graph.plan.mask_to_csr(P.edge_keep(s, 0, adj.rows, adj.cols, k)))
           for k, s in zip(keeps, SEEDS)]
    for vm in (False, True):
        for transpose in (False, True):
            c = Case(inv=True, edges=True, transpose=transpose)
            with _view_major() if vm else contextlib.nullcontext():
                a, b = _launch(graph, I, [0, 1, 2, 3], c, rng)['x'], _launch(graph, I, [0, 1, 2, 3], c, inj)['x']
            assert torch.equal(a, b), (vm, transpose)


@pytest.mark.parametrize('dim', DIMS)
def test_split_row_tickets_reset_between_launch_shapes(graph, dim):
    """The arrival tickets of split rows are back at 0 after every launch shape: interleaved V = 3, view-major V = 4,
    interleaved V = 2, then the first launch again, bit-identical."""
    I = _inputs(graph.adj.n, dim)
    first = _launch(graph, I, [0, 1, 2], CASES['mixed_inV_T'])['x']
    with _view_major():
        _launch(graph, I, [0, 1, 2, 3], CASES['mixed_inV'])
    _launch(graph, I, [0, 1], CASES['mixed_in1'])
    assert torch.equal(_launch(graph, I, [0, 1, 2], CASES['mixed_inV_T'])['x'], first)


@pytest.mark.parametrize('dim', [4, 20, 128])
@pytest.mark.parametrize('V', [1, 4])
def test_node_drop_matches_float64(graph, dim, V):
    """ssl_node_drop_dev, views mixing RNG (view 0's seed read from the device), no and injected masks: forward exactly
    O.node_dropped per view, backward accumulated into a non-zero table against the float64 sum."""
    from sslrec_b200._lib import check, lib
    modes, keeps = (1, 0, 2, 1)[:V], (0.5, 1.0, 0.6, 0.8)[:V]
    n = graph.adj.n
    g = torch.Generator().manual_seed(2000 + dim)
    masks = []
    for v in range(V):
        if modes[v] == 1:
            masks.append(torch.from_numpy(P.node_keep(SEEDS[v], np.arange(n), keeps[v])))
        else:
            masks.append(torch.rand(n, generator=g) < keeps[v] if modes[v] == 2 else torch.ones(n, dtype=torch.bool))
    inj = [m.to(torch.uint8).cuda() for m in masks]
    args = ((C.c_int32 * V)(*modes), (C.c_float * V)(*keeps),
            (C.c_void_p * V)(*[inj[v].data_ptr() if modes[v] == 2 else None for v in range(V)]),
            (C.c_uint64 * V)(*([DECOY] + list(SEEDS[1:V]))), (C.c_void_p * V)(*([graph.seed_dev.data_ptr()] + [None] * (V - 1))))
    stream = torch.cuda.current_stream().cuda_stream
    x = torch.randn(n, dim, generator=g) * 0.1
    out = torch.full((n, V, dim), float('nan'), device='cuda')
    check(lib.ssl_node_drop_dev(x.cuda().data_ptr(), out.data_ptr(), n, dim, V, 0, *args, 0, stream), 'ssl_node_drop')
    want = torch.stack([O.node_dropped(x.double(), m) for m in masks], 1)
    assert torch.equal(out.cpu().double(), want)
    gv = torch.randn(n, V, dim, generator=g) * 0.1
    acc0 = torch.randn(n, dim, generator=g) * 0.1
    acc = acc0.cuda()
    check(lib.ssl_node_drop_dev(gv.cuda().data_ptr(), acc.data_ptr(), n, dim, V, 1, *args, 0, stream), 'ssl_node_drop')
    kept = gv.double() * torch.stack(masks, 1).double().unsqueeze(-1)
    ratio = _check(acc, (acc0.double() + kept.sum(1), acc0.double().abs() + kept.abs().sum(1), torch.zeros(n, dim, dtype=torch.float64)),
                   f'node drop backward dim={dim} V={V}')
    RATIOS['node_drop_bwd'] = max(RATIOS.get('node_drop_bwd', 0.0), ratio)
