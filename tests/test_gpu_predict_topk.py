"""ssl_predict_topk (csrc/predict_topk.cuh) on the GPU: the fused score + mask + top-k call against ssl_predict_mask followed by ssl_topk,
bit for bit (torch.equal on the ids and on the value bits), from one user up to a 1 M-item catalogue; the rejected arguments; the memory the
fused call needs; and, per model, ``predict_topk`` against ``topk(full_predict(...))`` and Trainer.evaluate against a two-kernel evaluation."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(n_b, n_item, dim, k, mode, seed):
    """Seeded inputs of one call: the user table is the strided view [:, 2, :] of a [n_user, 3, dim] tensor (as SGL's final_embeds), the
    item table a view with a row stride of dim + 4.  A few item rows are copies of one large row -- at both ends of the catalogue, on both
    sides of tile (and so chunk) boundaries -- so exact ties rank near the top.  User 0's row is all zeros, user 1 has all but k // 2 items
    masked, the users repeat.  mode: 'none' | 'dense' | 'csr' (training rows sorted ascending, 12 items per user)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    n_user = max(4, n_b // 2 + 3)
    ut = torch.randn(n_user, 3, dim, device='cuda', generator=g)[:, 2, :]
    ibase = torch.randn(n_item, dim + 4, device='cuda', generator=g) * 0.3
    it = ibase[:, :dim]
    dup = torch.tensor(sorted({0, 1, n_item // 2, n_item - 2, n_item - 1} | {t * 128 + d for t in range(1, n_item // 128, max(1, n_item // 128 // 40))
                                                                             for d in (-1, 0)}), device='cuda')
    dup = dup[(dup >= 0) & (dup < n_item)]
    it[dup] = it[0] * 4.0
    ut[0] = 0.0
    users = torch.randint(0, n_user, (n_b,), device='cuda', generator=g)
    users[: min(n_b, 3)] = torch.tensor([1, 0, 1], device='cuda')[: min(n_b, 3)]
    rows = [torch.randint(0, n_item, (min(12, n_item),), device='cuda', generator=g).unique() for _ in range(n_user)]
    keep = torch.randperm(n_item, device='cuda', generator=g)[: max(0, k // 2)]
    heavy = torch.ones(n_item, dtype=torch.bool, device='cuda')
    heavy[keep] = False
    rows[1] = heavy.nonzero().flatten()
    mask = rowptr = cols = None
    if mode == 'csr':
        lens = torch.tensor([0] + [r.numel() for r in rows], device='cuda')
        rowptr = lens.cumsum(0).to(torch.int32)
        cols = torch.cat(rows).to(torch.int32)
    elif mode == 'dense':
        mask = torch.zeros(n_b, n_item, dtype=torch.int64, device='cuda')
        for b, u in enumerate(users.tolist()):
            mask[b, rows[u]] = 1
    return ut, ibase, it, users, mask, rowptr, cols


def _ptr(t):
    return None if t is None else t.data_ptr()


def _pair(ut, it, users, n_item, dim, mask, rowptr, cols, k):
    from sslrec_b200._lib import check, lib
    n_b = users.numel()
    preds = torch.empty(n_b, n_item, device='cuda')
    idx = torch.empty(n_b, k, dtype=torch.int64, device='cuda')
    val = torch.empty(n_b, k, device='cuda')
    s = torch.cuda.current_stream().cuda_stream
    check(lib.ssl_predict_mask(ut.data_ptr(), ut.stride(0), it.data_ptr(), it.stride(0), users.data_ptr(), n_b, n_item, dim, _ptr(mask),
                               _ptr(rowptr), _ptr(cols), preds.data_ptr(), s), 'ssl_predict_mask')
    check(lib.ssl_topk(preds.data_ptr(), n_b, n_item, k, idx.data_ptr(), val.data_ptr(), s), 'ssl_topk')
    return idx, val


def _ws_bytes(n_b, n_item, k):
    from sslrec_b200._lib import check, lib
    b = C.c_int64(0)
    check(lib.ssl_predict_topk_workspace(n_b, n_item, k, C.byref(b)), 'ssl_predict_topk_workspace')
    return b.value


def _fused_rc(ut, it, users, n_item, dim, mask, rowptr, cols, k, ws, ws_bytes, idx, val, n_b=None):
    from sslrec_b200._lib import lib
    return lib.ssl_predict_topk(ut.data_ptr(), ut.stride(0), it.data_ptr(), it.stride(0), _ptr(users), users.numel() if n_b is None else n_b,
                                n_item, dim, _ptr(mask), _ptr(rowptr), _ptr(cols), k, _ptr(ws), ws_bytes, _ptr(idx), _ptr(val),
                                torch.cuda.current_stream().cuda_stream)


def _fused(ut, it, users, n_item, dim, mask, rowptr, cols, k):
    """The fused call into NaN / -1 sentinels, with a workspace that starts as garbage."""
    from sslrec_b200._lib import check
    n_b = users.numel()
    nbytes = _ws_bytes(n_b, n_item, k)
    ws = torch.full((max(nbytes, 16),), 0xA5, dtype=torch.uint8, device='cuda')
    idx = torch.full((n_b, k), -1, dtype=torch.int64, device='cuda')
    val = torch.full((n_b, k), float('nan'), device='cuda')
    check(_fused_rc(ut, it, users, n_item, dim, mask, rowptr, cols, k, ws, nbytes, idx, val), 'ssl_predict_topk')
    return idx, val


def _same(a, b):
    ia, va = a
    ib, vb = b
    return torch.equal(ia, ib) and torch.equal(va.view(torch.int32), vb.view(torch.int32))


#         n_b   n_item   dim  k    mask
SHAPES = [(1, 1, 4, 1, 'none'), (1, 1, 4, 1, 'csr'), (1, 7, 4, 7, 'dense'), (127, 300, 32, 7, 'dense'), (128, 1000, 36, 40, 'csr'),
          (257, 5000, 64, 40, 'none'), (257, 20000, 128, 256, 'dense'), (128, 256, 4, 256, 'csr'), (1024, 300, 4, 256, 'csr'),
          (1024, 83761, 64, 40, 'csr'), (256, 83761, 64, 40, 'csr'), (1024, 19747, 32, 40, 'csr'), (1024, 83761, 64, 256, 'csr'),
          (1024, 83761, 64, 40, 'none'), (1024, 1000000, 128, 40, 'csr'), (1, 1000000, 128, 256, 'none'), (257, 130000, 36, 100, 'csr')]


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'b%d_i%d_d%d_k%d_%s' % s)
def test_fused_equals_predict_mask_then_topk(shape):
    n_b, n_item, dim, k, mode = shape
    ut, _, it, users, mask, rowptr, cols = _inputs(n_b, n_item, dim, k, mode, seed=n_b * 7 + n_item + dim)
    want = _pair(ut, it, users, n_item, dim, mask, rowptr, cols, k)
    got = _fused(ut, it, users, n_item, dim, mask, rowptr, cols, k)
    assert _same(got, want)
    assert torch.equal(_fused(ut, it, users, n_item, dim, mask, rowptr, cols, k)[1].view(torch.int32), got[1].view(torch.int32))   # relaunch
    if n_b >= 3 and mode != 'none':
        # user 1 has k // 2 unmasked items: the rest of its top k are masked entries at exactly -1e8, lowest ids first
        assert (got[1][0, k // 2:] == -1e8).all() and (got[1][0, : k // 2] > -1e8).all()
    # the tied copies of one item row rank in ascending id order
    i, v = got
    tie = (v[:, 1:] == v[:, :-1])
    assert (i[:, 1:][tie] > i[:, :-1][tie]).all()


def test_two_launches_are_bit_identical_and_values_are_optional():
    n_b, n_item, dim, k = 1024, 83761, 64, 40
    ut, _, it, users, mask, rowptr, cols = _inputs(n_b, n_item, dim, k, 'csr', seed=5)
    a = _fused(ut, it, users, n_item, dim, mask, rowptr, cols, k)
    b = _fused(ut, it, users, n_item, dim, mask, rowptr, cols, k)
    assert _same(a, b)
    from sslrec_b200._lib import check
    nbytes = _ws_bytes(n_b, n_item, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    idx = torch.full((n_b, k), -1, dtype=torch.int64, device='cuda')
    check(_fused_rc(ut, it, users, n_item, dim, mask, rowptr, cols, k, ws, nbytes, idx, None), 'ssl_predict_topk')
    assert torch.equal(idx, a[0])


def test_rejected_arguments_write_nothing():
    from sslrec_b200._lib import lib
    n_b, n_item, dim, k = 130, 1000, 32, 40
    ut, _, it, users, mask, rowptr, cols = _inputs(n_b, n_item, dim, k, 'csr', seed=9)
    nbytes = _ws_bytes(n_b, n_item, k)
    ws = torch.zeros(nbytes + 64, dtype=torch.uint8, device='cuda')
    idx = torch.full((n_b, k), -1, dtype=torch.int64, device='cuda')
    val = torch.full((n_b, k), float('nan'), device='cuda')
    ws_sent = ws.clone()
    bad = [dict(k=0), dict(k=257), dict(n_item=39, k=40), dict(dim=0), dict(dim=129), dict(n_b=65536), dict(ws_bytes=nbytes - 1),
           dict(ws_off=8), dict(users=None), dict(ut=None), dict(idx=None), dict(ws=None)]
    for over in bad:
        a = dict(ut=ut, it=it, users=users, n_item=n_item, dim=dim, k=k, ws=ws, ws_bytes=nbytes, idx=idx, n_b=n_b, ws_off=0)
        a.update(over)
        rc = lib.ssl_predict_topk(_ptr(a['ut']), ut.stride(0), it.data_ptr(), it.stride(0), _ptr(a['users']), a['n_b'], a['n_item'], a['dim'],
                                  None, rowptr.data_ptr(), cols.data_ptr(), a['k'],
                                  None if a['ws'] is None else a['ws'].data_ptr() + a['ws_off'], a['ws_bytes'], _ptr(a['idx']),
                                  val.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert rc == -1, over
    torch.cuda.synchronize()
    assert (idx == -1).all() and torch.isnan(val).all() and torch.equal(ws, ws_sent)
    b = C.c_int64(-5)
    for args in [(n_b, n_item, 0), (n_b, n_item, 257), (n_b, 10, 11), (65536, n_item, k), (n_b, 2 ** 32, k)]:
        assert lib.ssl_predict_topk_workspace(*args, C.byref(b)) == -1 and b.value == -5
    assert lib.ssl_predict_topk_workspace(n_b, n_item, k, None) == -1


def test_peak_memory_at_a_million_items_stays_far_below_the_score_matrix():
    n_b, n_item, dim, k = 1024, 1000000, 128, 40
    ut, _, it, users, mask, rowptr, cols = _inputs(n_b, n_item, dim, k, 'csr', seed=11)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx, val = _fused(ut, it, users, n_item, dim, mask, rowptr, cols, k)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f'fused peak {peak / 2**20:.1f} MiB against a {4 * n_b * n_item / 2**20:.0f} MiB score matrix')
    assert peak < 0.05 * 4 * n_b * n_item


# ---- model level -------------------------------------------------------------------------------------------------------------------------
MODEL_CASES = [('lightgcn', 'small'), ('simgcl', 'small'), ('sgl', 'small'), ('ncl_k50', 'small'), ('hccf_h128', 'small'),
               ('directau', 'small'), ('lightgcl', 'small')]


def _model(model_key, case_name):
    from test_gpu_models import _run
    g, case, model, _ = _run(model_key, case_name)
    model.eval()
    return case, model


def _batches(case):
    bt = min(64, case['n_user'])
    users = torch.arange(bt).cuda()
    mask = torch.zeros(bt, case['n_item'], dtype=torch.int64)
    sel = case['rows'] < bt
    mask[torch.from_numpy(case['rows'][sel]), torch.from_numpy(case['cols'][sel])] = 1
    return {'dense': [users, mask.cuda()], 'train': [users, 'train'], 'none': [users, None], 'lean': [users]}


@pytest.mark.parametrize('model_key,case_name', MODEL_CASES)
def test_model_predict_topk_equals_topk_of_full_predict(model_key, case_name):
    from sslrec_b200.trainer import topk
    case, model = _model(model_key, case_name)
    k = min(40, case['n_item'])
    for form, batch in _batches(case).items():
        with torch.no_grad():
            want = topk(model.full_predict(batch), k, return_values=True)
            got = model.predict_topk(batch, k, return_values=True)
            assert _same(got, want), form
            assert torch.equal(model.predict_topk(batch, k), want[0]), form
    # the side effects are full_predict's: is_training and the cached evaluation table
    _, a = _model(model_key, case_name)
    _, b = _model(model_key, case_name)
    for m in (a, b):
        if hasattr(m, 'is_training'):
            m.is_training = True
    batch = _batches(case)['train']
    with torch.no_grad():
        a.full_predict(batch)
        b.predict_topk(batch, k)
    assert getattr(a, 'is_training', None) == getattr(b, 'is_training', None)
    fa, fb = getattr(a, 'final_embeds', None), getattr(b, 'final_embeds', None)
    assert (fa is None) == (fb is None) and (fa is None or torch.equal(fa, fb))


def test_lightgcn_exact_order_predict_topk():
    from sslrec_b200.config import configs
    from sslrec_b200.trainer import topk
    case, model = _model('lightgcn', 'small')
    configs['test']['exact_order'] = True
    try:
        for form, batch in _batches(case).items():
            with torch.no_grad():
                assert _same(model.predict_topk(batch, 40, return_values=True), topk(model.full_predict(batch), 40, return_values=True)), form
    finally:
        configs['test']['exact_order'] = False


class _TwoKernel:
    """The model seen through full_predict only: Trainer.evaluate then ranks with full_predict + topk."""

    def __init__(self, model):
        self.model = model

    def eval(self):
        self.model.eval()

    def full_predict(self, batch_data):
        return self.model.full_predict(batch_data)


@pytest.mark.parametrize('name', ['lightgcn', 'simgcl'])
def test_trainer_evaluate_matches_the_two_kernel_evaluation(name, monkeypatch):
    import importlib

    from sslrec_b200 import trainer as T

    import scipy.sparse as sp
    import torch.utils.data as tdata

    from oracle import inputs
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import AllRankTstData, DataHandlerGeneralCF
    from sslrec_b200.trainer import Trainer, init_seed
    case = inputs.make_case('small')
    hp = dict(layer_num=2, embedding_size=32, reg_weight=1e-6, keep_rate=0.8, cl_weight=1e-2, temperature=0.2, eps=0.2)
    cfg = default_config(name, **hp)
    cfg['train'].update(batch_size=1024, epoch=1)
    cfg['test']['batch_size'] = 100
    cfg['test']['dense_mask'] = True
    load_config(base=cfg, device='cuda')
    init_seed()
    U, I = case['n_user'], case['n_item']
    trn = sp.coo_matrix((np.ones(len(case['rows']), dtype=np.float32), (case['rows'], case['cols'])), shape=(U, I))
    rs = np.random.RandomState(1)
    val = sp.coo_matrix((np.ones(400), (rs.randint(0, U, 400), rs.randint(0, I, 400))), shape=(U, I))
    dh = DataHandlerGeneralCF(trn, val, val)
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + name)
    model = [getattr(mod, a) for a in dir(mod) if a.lower() == name][0](dh).cuda()
    tr = Trainer(dh)
    tr.create_optimizer(model)
    tr.train_epoch(model, 0)
    lean = tdata.DataLoader(AllRankTstData(val, trn, dense_mask=False), batch_size=100, shuffle=False)
    assert T.FUSED_TOPK_MIN_ITEMS > I          # this catalogue is ranked by the pair unless the threshold is lowered
    for loader in (None, lean):
        pair = tr.evaluate(_TwoKernel(model), loader=loader)
        assert all(np.array_equal(v, pair[m]) for m, v in tr.evaluate(model, loader=loader).items())
        monkeypatch.setattr(T, 'FUSED_TOPK_MIN_ITEMS', I)
        fused = tr.evaluate(model, loader=loader)
        monkeypatch.setattr(T, 'FUSED_TOPK_MIN_ITEMS', I + 1)
        assert set(fused) == set(pair)
        for m in fused:
            assert np.array_equal(fused[m], pair[m]), (m, fused[m], pair[m])
