"""train.cuda_graph for HCCF, NCL, LightGCL and DirectAU, and the device pieces that make HCCF capturable:
ssl_unique_ids (sorted de-duplication on the device), the InfoNCE contraction and epilogues bounded by a device row count,
and the graph-safe spec-node term built from them."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import cf_oracle as O
from oracle import inputs, replay
import ssl_test_helpers as H

pytestmark = pytest.mark.gpu


def _L():
    from sslrec_b200._lib import check, lib
    return check, lib


def _s():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape):
    return torch.full(shape, float('nan'), device='cuda')


def _ceil(n, m):
    return (n + m - 1) // m * m


# ---- 1. ssl_unique_ids ------------------------------------------------------------------------------------------

def _unique(idx, n_range, scratch=None):
    check, lib = _L()
    words = C.c_int64()
    check(lib.ssl_unique_ids_scratch(n_range, C.byref(words)))
    if scratch is None:
        scratch = torch.full((words.value,), -1, dtype=torch.int32, device='cuda')       # dirty: the launch clears it
    out = torch.full_like(idx, -7)
    count = torch.full((), -7, dtype=torch.int64, device='cuda')
    check(lib.ssl_unique_ids(idx.data_ptr(), idx.numel(), n_range, scratch.data_ptr(), words.value, out.data_ptr(), count.data_ptr(), _s()))
    return out, count, scratch


def _check_unique(idx, out, count):
    ref = torch.unique(idx, sorted=True)
    c = int(count.item())
    assert c == ref.numel()
    assert torch.equal(out[:c], ref)
    assert torch.equal(out[c:], torch.full_like(out[c:], int(ref[-1])))


UNIQUE_CASES = [  # (n, n_range, kind)
    (1, 1, 'random'), (2, 1, 'random'), (2, 4097, 'ends'), (4096, 4097, 'equal'), (4096, 4097, 'distinct'), (4096, 4097, 'ends'),
    (4096, 5_000_000, 'random'), (4096, 5_000_000, 'ends'), (100_003, 5_000_000, 'random'), (100_003, 100_003, 'distinct'),
    (100_003, 4097, 'random'), (4096, 300, 'random'), (4096, 5_000_000, 'from300'), (100_003, 5_000_000, 'equal'),
]


@pytest.mark.parametrize('n,n_range,kind', UNIQUE_CASES)
def test_unique_ids_equals_torch_unique(n, n_range, kind):
    g = torch.Generator(device='cuda').manual_seed(n * 31 + n_range)
    if kind == 'random':
        idx = torch.randint(0, n_range, (n,), device='cuda', generator=g)
    elif kind == 'equal':
        idx = torch.full((n,), n_range // 2, dtype=torch.int64, device='cuda')
    elif kind == 'distinct':
        idx = torch.randperm(n_range, device='cuda', generator=g)[:n]
    elif kind == 'from300':      # a batch drawn from 300 ids spread over the whole range
        pool = torch.randperm(n_range, device='cuda', generator=g)[:300]
        idx = pool[torch.randint(0, 300, (n,), device='cuda', generator=g)]
    else:                        # 0 and n_range - 1 present
        idx = torch.randint(0, n_range, (n,), device='cuda', generator=g)
        idx[0], idx[-1] = n_range - 1, 0
    out, count, scratch = _unique(idx, n_range)
    _check_unique(idx, out, count)
    # a second launch over the same, now dirty, scratch with other ids
    idx2 = torch.randint(0, max(1, n_range // 3), (n,), device='cuda', generator=g)
    out2, count2, _ = _unique(idx2, n_range, scratch)
    _check_unique(idx2, out2, count2)


def test_unique_ids_rejects_bad_arguments():
    from sslrec_b200._lib import SslError
    check, lib = _L()
    idx = torch.zeros(8, dtype=torch.int64, device='cuda')
    out, count = torch.empty_like(idx), torch.empty((), dtype=torch.int64, device='cuda')
    words = C.c_int64()
    check(lib.ssl_unique_ids_scratch(100, C.byref(words)))
    scratch = torch.empty(words.value, dtype=torch.int32, device='cuda')
    args = [idx.data_ptr(), 8, 100, scratch.data_ptr(), words.value, out.data_ptr(), count.data_ptr(), _s()]
    for k, bad in ((0, None), (3, None), (5, None), (6, None), (1, -1), (2, 0), (2, -5), (4, words.value - 1)):
        a = list(args)
        a[k] = bad
        assert lib.ssl_unique_ids(*a) != 0, (k, bad)
    assert lib.ssl_unique_ids_scratch(0, C.byref(words)) != 0
    with pytest.raises(SslError):
        check(lib.ssl_unique_ids(idx.data_ptr(), -1, 100, scratch.data_ptr(), words.value, out.data_ptr(), count.data_ptr(), _s()))


# ---- 2. the contraction bounded by a device row count ---------------------------------------------------------

def _operand(x, tc):
    """Normalised rows of x with the copies either contraction reads (as engine._nce_fwd builds them)."""
    check, lib = _L()
    n, d = x.shape
    npad = max(64, _ceil(n, 64))
    f = dict(device='cuda', dtype=torch.float32)
    out = torch.zeros(npad, d, **f)
    if tc:
        hi, lo, thi, tlo = torch.zeros(npad, d, **f), torch.zeros(npad, d, **f), torch.zeros(d, npad, **f), torch.zeros(d, npad, **f)
        check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), None, None, hi.data_ptr(), lo.data_ptr(),
                                     thi.data_ptr(), tlo.data_ptr(), npad, _s()))
        return dict(n=n, hi=hi, lo=lo, thi=thi, tlo=tlo, pitch=npad)
    out_t = torch.zeros(npad // 64, d, 64, **f)
    check(lib.ssl_rows_normalize(x.data_ptr(), d, None, n, d, 0, 1.0, out.data_ptr(), out_t.data_ptr(), None, None, None, None, None, 0, _s()))
    return dict(n=n, x=out, t=out_t)


def _contract(tc, R, n_r, Cop, n_c, d, cs, n_split, rs, o, live=None, role=0):
    check, lib = _L()
    off = 2.0
    csp = None if cs is None else cs.data_ptr()
    if tc and live is None:
        rc = lib.ssl_softmax_gemm_tf32x3(R['hi'].data_ptr(), R['lo'].data_ptr(), n_r, Cop['hi'].data_ptr(), Cop['lo'].data_ptr(),
                                         Cop['thi'].data_ptr(), Cop['tlo'].data_ptr(), Cop['pitch'], n_c, d, csp, off, n_split,
                                         rs.data_ptr(), o.data_ptr(), _s())
    elif tc:
        rc = lib.ssl_softmax_gemm_tf32x3_live(R['hi'].data_ptr(), R['lo'].data_ptr(), n_r, Cop['hi'].data_ptr(), Cop['lo'].data_ptr(),
                                              Cop['thi'].data_ptr(), Cop['tlo'].data_ptr(), Cop['pitch'], n_c, d, csp, off, n_split,
                                              rs.data_ptr(), o.data_ptr(), live.data_ptr(), role, _s())
    elif live is None:
        rc = lib.ssl_softmax_gemm(R['x'].data_ptr(), n_r, Cop['x'].data_ptr(), Cop['t'].data_ptr(), n_c, d, csp, off, n_split,
                                  rs.data_ptr(), o.data_ptr(), _s())
    else:
        rc = lib.ssl_softmax_gemm_live(R['x'].data_ptr(), n_r, Cop['x'].data_ptr(), Cop['t'].data_ptr(), n_c, d, csp, off, n_split,
                                       rs.data_ptr(), o.data_ptr(), live.data_ptr(), role, _s())
    check(rc)


LIVES = [1, 63, 64, 65, 127, 128, 129, -1, 0]          # -1: cap - 1, 0: cap
KERNELS = [(True, 32), (True, 64), (False, 48), (False, 128)]


@pytest.mark.parametrize('tc,d', KERNELS)
@pytest.mark.parametrize('cap', [4096, 1000])
def test_bounded_contraction_resident_rows(tc, d, cap):
    """R = a padded anchor list of capacity cap, live rows bounded on the device: outputs equal the plain launch at n_r = live
    bit for bit; rows past live keep their NaN sentinel."""
    g = torch.Generator(device='cuda').manual_seed(cap + d)
    anchors = torch.randn(cap, d, device='cuda', generator=g)
    n_c = 700
    Cop = _operand(torch.randn(n_c, d, device='cuda', generator=g), tc)
    Rcap = _operand(anchors, tc)
    for lv in LIVES:
        live = cap + lv if lv <= 0 else lv
        Rl = _operand(anchors[:live].contiguous(), tc)
        dl = torch.tensor(live, dtype=torch.int64, device='cuda')
        for n_split in range(1, _ceil(n_c, 64) // 64 + 1):
            rs_ref, o_ref = _nan(n_split, live), _nan(n_split, live, d)
            _contract(tc, Rl, live, Cop, n_c, d, None, n_split, rs_ref, o_ref)
            rs, o = _nan(n_split, cap), _nan(n_split, cap, d)
            _contract(tc, Rcap, cap, Cop, n_c, d, None, n_split, rs, o, dl, 1)
            assert torch.equal(o[:, :live], o_ref) and torch.equal(rs[:, :live], rs_ref), (live, n_split)
            assert not torch.isnan(o_ref).any() and not torch.isnan(rs_ref).any()
            assert torch.isnan(o[:, live:]).all() and torch.isnan(rs[:, live:]).all(), (live, n_split)


@pytest.mark.parametrize('tc,d', KERNELS)
@pytest.mark.parametrize('cap', [4096, 1000])
def test_bounded_contraction_streamed_columns(tc, d, cap):
    """C = a padded anchor list, live columns bounded on the device, colscale NaN past live: outputs equal the plain launch at
    n_c = live bit for bit for every n_split it accepts; chunks left empty by the live count write zero partials."""
    g = torch.Generator(device='cuda').manual_seed(7 * cap + d)
    anchors = torch.randn(cap, d, device='cuda', generator=g)
    n_r = 300
    R = _operand(torch.randn(n_r, d, device='cuda', generator=g), tc)
    Ccap = _operand(anchors, tc)
    cs_vals = torch.rand(_ceil(cap, 64), device='cuda', generator=g) + 0.5
    for lv in LIVES:
        live = cap + lv if lv <= 0 else lv
        Cl = _operand(anchors[:live].contiguous(), tc)
        cs = cs_vals.clone()
        cs[live:] = float('nan')
        dl = torch.tensor(live, dtype=torch.int64, device='cuda')
        for n_split in range(1, _ceil(live, 64) // 64 + 1):
            rs_ref, o_ref = _nan(n_split, n_r), _nan(n_split, n_r, d)
            _contract(tc, R, n_r, Cl, live, d, cs, n_split, rs_ref, o_ref)
            rs, o = _nan(n_split, n_r), _nan(n_split, n_r, d)
            _contract(tc, R, n_r, Ccap, cap, d, cs, n_split, rs, o, dl, 2)
            assert not torch.isnan(o_ref).any() and not torch.isnan(rs_ref).any(), (live, n_split)
            assert torch.equal(o, o_ref) and torch.equal(rs, rs_ref), (live, n_split)
        # every chunk of the capacity: the ones past the live tiles are empty and write zeros
        n_split = _ceil(cap, 64) // 64
        rs, o = _nan(n_split, n_r), _nan(n_split, n_r, d)
        _contract(tc, R, n_r, Ccap, cap, d, cs, n_split, rs, o, dl, 2)
        assert not torch.isnan(o).any() and not torch.isnan(rs).any()
        n_ct = _ceil(live, 64) // 64
        empty = [sp for sp in range(n_split) if n_ct * sp // n_split == n_ct * (sp + 1) // n_split]
        assert len(empty) == n_split - n_ct
        for sp in empty:
            assert (o[sp] == 0).all() and (rs[sp] == 0).all(), (live, sp)
        rs1, o1 = _nan(1, n_r), _nan(1, n_r, d)
        _contract(tc, R, n_r, Cl, live, d, cs, 1, rs1, o1)
        H.close(o.double().sum(0), o1[0].double(), 1e-5, 1e-5 * o1.abs().max().item(), 'summed chunks')


def test_live_epilogues():
    """ssl_sum_live, ssl_nce_colscale_live, ssl_nce_bwd_rows_live: nothing of a padding row reaches a sum, a colscale or a sink."""
    check, lib = _L()
    cap, d, live = 1000, 32, 377
    g = torch.Generator(device='cuda').manual_seed(5)
    dl = torch.tensor(live, dtype=torch.int64, device='cuda')
    x = torch.randn(cap, device='cuda', generator=g)
    x[live:] = float('nan')
    out = torch.empty((), device='cuda')
    check(lib.ssl_sum_live(x.data_ptr(), cap, dl.data_ptr(), 3.0, out.data_ptr(), _s()))
    ref = 3.0 * x[:live].double().sum() / live
    assert abs(out.item() - ref.item()) <= 1e-6 * x[:live].abs().sum().item() / live
    rowsum = torch.rand(cap, device='cuda', generator=g) + 0.5
    gsc = torch.tensor(2.0, device='cuda')
    cs = _nan(cap)
    check(lib.ssl_nce_colscale_live(rowsum.data_ptr(), cap, dl.data_ptr(), gsc.data_ptr(), 1.5, cs.data_ptr(), _s()))
    want = (1.5 / live) * 2.0 * 0.6931471805599453 / rowsum[:live].double()
    H.close(cs[:live], want, 1e-6, 0, 'colscale')
    assert (cs[live:] == 0).all()
    # bwd rows: the live call equals the plain call on the first live rows with scale / live
    a_hat, p_hat, obar = (torch.randn(cap, d, device='cuda', generator=g) for _ in range(3))
    r1, r2 = torch.rand(cap, device='cuda', generator=g) + 0.5, torch.rand(cap, device='cuda', generator=g) + 0.5
    for t in (a_hat, p_hat, obar):
        t[live:] = float('nan')
    idx = torch.randint(0, 50, (cap,), device='cuda', generator=g)
    g1, g2 = torch.zeros(50, d, device='cuda'), torch.zeros(50, d, device='cuda')
    check(lib.ssl_nce_bwd_rows_live(a_hat.data_ptr(), p_hat.data_ptr(), obar.data_ptr(), r1.data_ptr(), r2.data_ptr(), idx.data_ptr(), cap,
                                    dl.data_ptr(), d, 0.2, gsc.data_ptr(), 1.0, g1.data_ptr(), d, g2.data_ptr(), d, _s()))
    h1, h2 = torch.zeros(50, d, device='cuda'), torch.zeros(50, d, device='cuda')
    check(lib.ssl_nce_bwd_rows(a_hat.data_ptr(), p_hat.data_ptr(), obar.data_ptr(), r1.data_ptr(), r2.data_ptr(), idx.data_ptr(), live,
                               d, 0.2, gsc.data_ptr(), 1.0 / live, h1.data_ptr(), d, h2.data_ptr(), d, _s()))
    assert not torch.isnan(g1).any() and not torch.isnan(g2).any()
    H.close(g1, h1, 1e-5, 1e-6 * h1.abs().max().item(), 'bwd rows g1')
    H.close(g2, h2, 1e-5, 1e-6 * h2.abs().max().item(), 'bwd rows g2')
    for fn, args in ((lib.ssl_sum_live, [x.data_ptr(), cap, None, 1.0, out.data_ptr(), _s()]),
                     (lib.ssl_nce_colscale_live, [rowsum.data_ptr(), cap, None, None, 1.0, cs.data_ptr(), _s()])):
        assert fn(*args) != 0


# ---- 3. the graph-safe spec-node term ---------------------------------------------------------------------------

@pytest.mark.parametrize('d', [32, 64, 48])
@pytest.mark.parametrize('dup', ['heavy', 'none'])
def test_spec_nodes_dev_term_matches_unique_path(d, dup):
    from sslrec_b200 import engine as E
    g = torch.Generator().manual_seed(d)
    N = 900
    e1, e2 = torch.randn(N, d, generator=g), torch.randn(N, d, generator=g)
    ids = torch.randint(0, 40, (512,), generator=g) * 17 if dup == 'heavy' else torch.randperm(N, generator=g)[:512]
    nodes = torch.unique(ids)
    res = {}
    for name in ('dev', 'unique'):
        a, b = e1.clone().cuda().requires_grad_(True), e2.clone().cuda().requires_grad_(True)
        if name == 'dev':
            loss = E.dense_infonce_spec_nodes_mean_dev(a, b, ids.cuda(), 0.2)
        else:
            loss = E.dense_infonce_spec_nodes_mean(a, b, nodes.cuda(), 0.2)
        loss.backward()
        res[name] = (loss.item(), a.grad, b.grad)
    a, b = e1.double().requires_grad_(True), e2.double().requires_grad_(True)
    ref = O.infonce_spec_nodes_mean(a, b, nodes, 0.2)
    ref.backward()
    for name, (lv, ga, gb) in res.items():
        assert abs(lv - ref.item()) <= 2e-6 * abs(ref.item()) + 1e-6, (name, lv, ref.item())
        H.close(ga, a.grad, 2e-4, 2e-6 * a.grad.abs().max().item(), name + ' grad e1')
        H.close(gb, b.grad, 2e-4, 2e-6 * b.grad.abs().max().item(), name + ' grad e2')
    H.close(res['dev'][1], res['unique'][1], 2e-4, 2e-6 * a.grad.abs().max().item(), 'dev vs unique e1')
    H.close(res['dev'][2], res['unique'][2], 2e-4, 2e-6 * b.grad.abs().max().item(), 'dev vs unique e2')


# ---- 4. graph equals eager, per model ---------------------------------------------------------------------------

GRAPH_CASES = [('hccf', 'tiny'), ('hccf_h128', 'small'), ('ncl', 'tiny'), ('ncl_k50', 'small'), ('lightgcl', 'tiny'), ('lightgcl', 'small'),
               ('directau', 'tiny'), ('directau', 'small')]


def _model(key, size):
    g = replay.load_golden(key, size)
    case = inputs.make_case(size)
    torch.manual_seed(0)                    # same parameter init, and the same generator for k-means / svd_lowrank, in both runs
    np.random.seed(0)
    model, dh = H.make_model(key, case, g['hp'])
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']}, strict=False)
    return model, dh, case, g


def _batches(case, ncl, flagged, n=5):
    rs = np.random.RandomState(3)
    B = case['batch']
    out = []
    for k in range(n):
        pick = rs.randint(0, len(case['rows']), size=B)
        b = [torch.from_numpy(np.asarray(a)).long().cuda() for a in (case['rows'][pick], case['cols'][pick], rs.randint(0, case['n_item'], size=B))]
        if ncl:
            f = torch.zeros(B, dtype=torch.int64)
            f[0] = int(k in flagged)
            b.append(f.cuda())
        out.append(b)
    return out


def _count_kmeans(model):
    calls = [0]
    inner = model.kmeans

    def counted(x):
        calls[0] += 1
        return inner(x)
    model.kmeans = counted
    return calls


@pytest.mark.parametrize('key,size', GRAPH_CASES)
def test_cuda_graph_step_equals_eager_step_models(key, size):
    """HCCF's eager reference is the eager loop on the path a GraphedStep takes (device de-duplication, count-bounded term), the
    path of ``GraphedStep.eager`` too; its first loss also equals the plain eager (torch.unique) loss within 1e-6.  The two paths
    sum in different orders (n_split is chosen from the batch capacity), and Adam at lr 1e-2 amplifies that fp32 difference
    over later steps, so they are not compared there."""
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    name = key.split('_')[0]
    ncl = name == 'ncl'
    flagged = {0, 3}                       # NCL: re-cluster on the first batch and on a later one
    out = {}
    for mode in ('plain', 'eager', 'graph'):
        if mode == 'plain' and name != 'hccf':
            continue
        model, _, case, _ = _model(key, size)
        batches = _batches(case, ncl, flagged)
        calls = _count_kmeans(model) if ncl else [0]
        opt = FusedAdam(model.parameters(), lr=1e-2)
        losses = []
        if mode == 'plain':
            loss, _ = model.cal_loss(batches[0])
            out[mode] = loss.item()
            continue
        if mode == 'eager':
            model._graph_mode = name == 'hccf'
            for b in [batches[0]] * 2 + batches[1:]:
                opt.zero_grad()
                loss, _ = model.cal_loss(b)
                loss.backward()
                opt.step()
                losses.append(loss.item())
            model._graph_mode = False
        else:
            step = GraphedStep(model, opt, batches[0], warmup=2, recluster=0 in flagged)
            losses += [float('nan')] * 2
            want = {'hccf': 2, 'ncl': 0, 'lightgcl': int(getattr(model, 'dropout', 0) > 0)}.get(name)
            if want is not None:
                assert step.n_seeds == want, (key, step.n_seeds)
            for k, b in enumerate(batches[1:], start=1):
                loss, _ = step(b, recluster=k in flagged)
                losses.append(loss.item())
            step.close()
            assert all(int(st['step']) == 6 for st in opt.state.values())
        params = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).clone()
        clusters = (model.user2cluster.clone(), model.item2cluster.clone()) if ncl else None
        out[mode] = (losses, params, calls[0], clusters)
    if name == 'hccf':
        assert abs(out['eager'][0][0] - out['plain']) <= 1e-6 * abs(out['plain']), (out['eager'][0][0], out['plain'])
    for a, b in zip(out['graph'][0][2:], out['eager'][0][2:]):
        assert abs(a - b) <= 1e-6 * max(1.0, abs(b)), (key, out['graph'][0], out['eager'][0])
    assert torch.allclose(out['graph'][1], out['eager'][1], rtol=1e-5, atol=3e-4), (key, (out['graph'][1] - out['eager'][1]).abs().max().item())
    if ncl:
        assert out['graph'][2] == out['eager'][2] == 2 * (1 + 1 + 1), (out['graph'][2], out['eager'][2])   # first, batch 0 again, batch 3
        assert torch.equal(out['graph'][3][0], out['eager'][3][0]) and torch.equal(out['graph'][3][1], out['eager'][3][1])


# ---- 5. Trainer.train_epoch with train.cuda_graph ---------------------------------------------------------------

@pytest.mark.parametrize('key,size', [('hccf', 'tiny'), ('ncl', 'tiny')])
@pytest.mark.parametrize('loader', ['host', 'device'])
def test_trainer_cuda_graph_epoch_matches_eager_models(key, size, loader):
    import types
    from sslrec_b200.config import configs
    from sslrec_b200.data_handler import DeviceLoader, DeviceTrnData, HostBatchLoader, PairwiseTrnData, PairwiseWEpochFlagTrnData
    from sslrec_b200.trainer import Trainer
    ncl = key == 'ncl'
    res = {}
    for graph in (False, True):
        model, dh, case, _ = _model(key, size)
        calls = _count_kmeans(model) if ncl else [0]
        configs['train']['cuda_graph'] = graph
        if ncl:
            configs['model']['epoch_period'] = 1
        n = len(case['rows'])
        bs = max(8, n // 3 - 1)                       # the last batch is smaller
        configs['train']['batch_size'] = bs
        torch.manual_seed(1)
        np.random.seed(1)
        if loader == 'device':
            ld = DeviceLoader(DeviceTrnData(dh.trn_mat, 'cuda', 2023, epoch_period=1 if ncl else None), bs, seed=2023)
        else:
            ds = (PairwiseWEpochFlagTrnData if ncl else PairwiseTrnData)(dh.trn_mat.tocoo())
            ld = HostBatchLoader(ds, bs)
        assert len(ld) >= 3 and len(ld.dataset) % bs != 0
        tr = Trainer(types.SimpleNamespace(train_dataloader=ld))
        tr.create_optimizer(model)
        try:
            ep = [tr.train_epoch(model, e)[0] for e in range(3)]
        finally:
            if tr._graphed is not None:
                tr._graphed.close()
            configs['train']['cuda_graph'] = False
        res[graph] = (ep, torch.cat([p.detach().reshape(-1) for p in model.parameters()]).clone(), calls[0])
    for a, b in zip(res[True][0], res[False][0]):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), res
    assert torch.allclose(res[True][1], res[False][1], rtol=1e-5, atol=3e-4)
    if ncl:
        assert res[True][2] == res[False][2] >= 2 * 3, (res[True][2], res[False][2])     # re-clustered every epoch


# ---- 6. no host synchronisation inside a graphed step ----------------------------------------------------------

@pytest.mark.parametrize('key,size', [('hccf', 'tiny'), ('lightgcl', 'tiny'), ('ncl', 'tiny')])
def test_graphed_replays_do_not_sync(key, size):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    ncl = key == 'ncl'
    model, _, case, _ = _model(key, size)
    batches = _batches(case, ncl, {0})
    opt = FusedAdam(model.parameters(), lr=1e-2)
    step = GraphedStep(model, opt, batches[0], warmup=1, recluster=ncl)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for b in batches[1:]:
            step(b)                          # NCL: the steps without a re-cluster flag
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    step.close()
