"""Shared helpers of the GPU parity tests: build a drop-in model on the GPU from a golden case."""
import numpy as np
import scipy.sparse as sp
import torch

import mixgcf_oracle
from oracle import cf_oracle as O
from oracle import inputs, replay


def make_model(model_key, case, hp, inject=None, device='cuda'):
    import sslrec_b200
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import DataHandlerGeneralCF
    name = model_key.split('_')[0]
    cfg = default_config(name, **hp)
    cfg['model']['embedding_size'] = case['dim']
    cfg['train']['batch_size'] = case['batch']
    if name == 'ncl':
        cfg['train']['loss'] = 'pairwise_with_epoch_flag'
    load_config(base=cfg, device=device)
    trn = sp.coo_matrix((np.ones(len(case['rows']), dtype=np.float32), (case['rows'], case['cols'])),
                        shape=(case['n_user'], case['n_item']))
    dh = DataHandlerGeneralCF(trn)
    dh.load_data()
    import importlib
    mod = importlib.import_module('sslrec_b200.general_cf.' + name)
    cls = [getattr(mod, a) for a in dir(mod) if a.lower() == name][0]
    model = cls(dh)
    model._inject = inject
    model = model.to(device)
    return model, dh


def gpu_injection(model_key, case, hp, adj, dr, device='cuda'):
    """replay.draws (oracle Adj order == CSR order) -> the model's ``_inject`` dict on the GPU."""
    name = model_key.split('_')[0]
    inj = {}
    u8 = lambda m: None if m is None else torch.from_numpy(np.asarray(m).astype(np.uint8)).to(device)
    if name == 'lightgcn':
        inj['edge_masks'] = [u8(dr['edge_keep'])] + [None] * 3
    elif name == 'simgcl':
        inj['noise_u'] = [[u.to(device).contiguous() for u in view] for view in dr['uniforms']]
    elif name == 'sgl':
        inj['edge_masks'] = [u8(m) for m in dr['edge_keeps']] + [None, None]
        inj['node_masks'] = [None if m is None else m.to(torch.uint8).to(device) for m in dr['node_keeps']]
    elif name == 'hccf':
        inj['edge_masks_per_layer'] = [u8(m) for m in dr['edge_keeps']]
        inj['hyper_keeps'] = [(ku.to(device), ki.to(device)) for ku, ki in dr['hyper_keeps']]
    return inj


# ---- model-level cases off the golden shapes (tests/test_gpu_model_paths.py, tests/test_host_model_paths.py) -------------------

# hyper-parameters of each drop-in model: the goldens' (the YAML values, with BASELINE.json's layer counts)
PATH_HP_FROM = {'lightgcn': ('lightgcn', 'small'), 'simgcl': ('simgcl', 'small'), 'sgl': ('sgl', 'small'), 'sgl_nd': ('sgl_nd', 'tiny'),
                'ncl': ('ncl_k50', 'small'), 'hccf': ('hccf_h128', 'small'), 'directau': ('directau', 'small'),
                'lightgcl': ('lightgcl', 'small')}
PATH_USERS, PATH_ITEMS, PATH_EDGES = 600, 450, 5000
HUB_USER, HUB_ITEM = 0, 0
HUB_USER_DEG, HUB_ITEM_MIN_DEG = 160, 320         # a split row on each side of side_split (rows of > 128 entries are split)
LOSS_RTOL, GRAD_RTOL, GRAD_MAXTOL, PRED_RTOL = 1e-5, 2e-4, 5e-6, 1e-5
KINK_MARGIN = 1e-6


def _path_matrix():
    """(model_key, embedding_size, temperature or None, batch, hyper_num or None) of every model-level path case."""
    out = []
    for d in (16, 20, 48, 128):              # the FP32-FMA contraction; propagation G = 4, 8 (idle lanes), 16 (idle lanes), 32
        out.append(('lightgcn', d, None, 300, None))
        out += [(m, d, 0.2, 300, None) for m in ('simgcl', 'sgl', 'sgl_nd', 'ncl', 'hccf', 'lightgcl')]
        out += [('directau', d, None, 300, None), ('directau', d, None, 100, None)]     # contraction / pairwise uniformity
    out += [('lightgcn', 4, None, 300, None), ('simgcl', 4, 0.2, 300, None)]          # propagation G = 1
    # 3xTF32 InfoNCE.  Not SGL: with its cl_weight of 1 the two edge-dropped views of a hub row nearly coincide, the softmax
    # of its anchor row sits almost all on the positive, and below tau ~ 0.09 even a float32 evaluation of the loss misses the
    # gradient bound by 4-50x against float64 (the per-row gradient is a small difference of O(1 / tau) terms)
    out += [(m, d, 0.05, 300, None) for d in (32, 64) for m in ('simgcl', 'ncl', 'hccf')]
    out += [('simgcl', 64, 0.0900, 300, None), ('simgcl', 64, 0.0905, 300, None)]     # either side of the 3xFP16 offset bound
    out += [('hccf', 20, 0.2, 300, 16), ('hccf', 48, 0.2, 300, 40)]                   # hyper branch at other (d, H)
    return out


PATH_CASES = _path_matrix()
# cases whose default seed puts a kink input within KINK_MARGIN of its |term| sum (kink_margin): the first later seed that does not
PATH_SEEDS = {('simgcl', 128, 0.2): 43, ('hccf', 128, 0.2): 42, ('hccf', 64, 0.05): 43}


def path_case_id(case):
    m, d, tau, b, h = case
    return f'{m}-d{d}' + ('' if tau is None else f'-tau{tau}') + f'-b{b}' + ('' if h is None else f'-h{h}')


def path_setup(model_key, dim, tau, batch, hyper_num):
    """-> case, hp, adjacency, draws and injected state of one path case."""
    case = path_case(dim, batch, PATH_SEEDS.get((model_key, dim, tau), 41))
    hp = path_hp(model_key, dim, tau, hyper_num)
    adj = O.normalized_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
    dr = replay.draws(model_key, case, hp, adj)
    return case, hp, adj, dr, path_state(model_key, case, hp, adj, dr)


def path_hp(model_key, dim, tau=None, hyper_num=None):
    hp = dict(replay.load_golden(*PATH_HP_FROM[model_key])['hp'])
    hp['embedding_size'] = dim
    if tau is not None:
        hp['temp' if model_key == 'lightgcl' else 'temperature'] = tau
    if hyper_num is not None:
        hp['hyper_num'] = hyper_num
    return hp


def path_case(dim, batch=300, seed=41):
    """A ``inputs.make_case``-shaped case of 600 users x 450 items: the skewed graph of ``inputs.bipartite_edges`` (its last
    users / items are isolated), a user hub of degree 160 and an item hub of degree >= 320, and a batch of ``batch`` edges with
    repeated anchors, both hubs and an isolated item among the negatives."""
    U, I = PATH_USERS, PATH_ITEMS
    rows, cols = inputs.bipartite_edges(U, I, PATH_EDGES, seed)
    rs = np.random.RandomState(seed + 1000)
    live_u, live_i = U - U // 40, I - I // 40
    pairs = {(u, i) for u, i in zip(rows.tolist(), cols.tolist()) if u != HUB_USER}
    pairs |= {(HUB_USER, int(i)) for i in rs.choice(live_i, HUB_USER_DEG, replace=False)}
    for u in rs.permutation(live_u).tolist():
        if sum(1 for p in pairs if p[1] == HUB_ITEM) >= HUB_ITEM_MIN_DEG:
            break
        pairs.add((u, HUB_ITEM))
    pairs = np.array(sorted(pairs), dtype=np.int64)[rs.permutation(len(pairs))]
    rows, cols = pairs[:, 0].copy(), pairs[:, 1].copy()
    g = torch.Generator().manual_seed(seed + 2000)
    a, b = float(np.sqrt(6.0 / (U + dim))), float(np.sqrt(6.0 / (I + dim)))
    user_e = (torch.rand(U, dim, generator=g) * 2 - 1) * a
    item_e = (torch.rand(I, dim, generator=g) * 2 - 1) * b
    pick = rs.randint(0, len(rows), size=batch)
    pick[:3] = np.flatnonzero(rows == HUB_USER)[:3]         # the user hub, three times
    pick[3:6] = np.flatnonzero(cols == HUB_ITEM)[:3]        # the item hub as a positive
    ancs, poss = rows[pick].copy(), cols[pick].copy()
    negs = rs.randint(0, I, size=batch).astype(np.int64)
    negs[0], negs[1] = HUB_ITEM, I - 1                      # the item hub and an isolated item as negatives
    return dict(name=f'paths_d{dim}_b{batch}', n_user=U, n_item=I, dim=dim, batch=batch, seed=seed,
                rows=rows, cols=cols, user_e=user_e, item_e=item_e, ancs=ancs, poss=poss, negs=negs)


def path_state(model_key, case, hp, adj, dr):
    """The state both sides are given besides the draws: NCL's k-means (float64 Lloyd iterations from the drawn initial
    centroids, rounded to float32) and LightGCL's SVD factors (a seeded ``torch.svd_lowrank`` of its adjacency, float32),
    in the keys ``replay.oracle_loss`` reads from its ``golden`` argument."""
    name = model_key.split('_')[0]
    st = {}
    if name == 'ncl':
        for side, e in (('user', case['user_e']), ('item', case['item_e'])):
            cents, idx, _ = O.kmeans(e.double(), dr[f'init_{side}_centroids'].double(), iters=100)
            st[f'{side}_centroids'] = cents.float().numpy()
            st[f'{side}2cluster'] = idx.numpy()
    elif name == 'lightgcl':
        ladj = O.lightgcl_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
        up = ladj.rows < ladj.n_user
        m = torch.sparse_coo_tensor(torch.from_numpy(np.vstack([ladj.rows[up], ladj.cols[up] - ladj.n_user])),
                                    torch.from_numpy(ladj.vals[up]).double(), (ladj.n_user, ladj.n_item)).coalesce()
        with torch.random.fork_rng():
            torch.manual_seed(case['seed'])
            u, s, v = torch.svd_lowrank(m, q=hp['svd_q'])
        st['svd_ut'], st['svd_vt'] = u.T.contiguous().float().numpy(), v.T.contiguous().float().numpy()
        st['svd_u_mul_s'], st['svd_v_mul_s'] = (u * s).float().numpy(), (v * s).float().numpy()
    return st


def path_params(model_key, case, dr, dtype):
    params = {'user_embeds': case['user_e'], 'item_embeds': case['item_e']}
    if 'user_w' in dr:
        params['user_hyper_embeds'], params['item_hyper_embeds'] = dr['user_w'], dr['item_w']
    for i, w in enumerate(dr.get('ws', [])):
        params[f'Ws.{i}.W'] = w
    return {k: v.to(dtype).clone().requires_grad_(True) for k, v in params.items()}


def pred_users_mask(case, n=64):
    bt = min(n, case['n_user'])
    mask = torch.zeros(bt, case['n_item'], dtype=torch.int64)
    sel = case['rows'] < bt
    mask[torch.from_numpy(case['rows'][sel]), torch.from_numpy(case['cols'][sel])] = 1
    return torch.arange(bt), mask


def path_oracle(model_key, case, hp, adj, dr, st, dtype=torch.float64):
    """cal_loss, backward and full_predict of the oracle in ``dtype`` -> dict(loss, parts, grads, preds) of float64 numpy."""
    params = path_params(model_key, case, dr, dtype)
    loss, parts = replay.oracle_loss(model_key, case, hp, adj, dr, params, st)
    loss.backward()
    out = dict(loss=float(loss), parts={k: float(v) for k, v in parts.items()},
               grads={k: p.grad.double().numpy() for k, p in params.items()})
    with torch.no_grad():
        e = replay.clean_embeds(model_key, adj, hp, params)
        users, mask = pred_users_mask(case)
        out['preds'] = O.full_predict(e[:case['n_user']], e[case['n_user']:], users, mask).double().numpy()
    return out


def path_errors(got, ref):
    """Largest error of each output as a fraction of its bound (<= 1 passes): loss and terms |d| <= 1e-5 max(1, |ref|);
    gradients 2e-4 |ref| + 5e-6 max|ref|; scores 1e-5 max(1, |ref|)."""
    def frac(a, b, tol):
        err = np.abs(np.asarray(a, dtype=np.float64) - b)
        return float(np.max(np.divide(err, tol, out=np.where(err > 0, np.inf, 0.0), where=tol > 0), initial=0.0))
    r = {'loss': frac(got['loss'], ref['loss'], LOSS_RTOL * max(1.0, abs(ref['loss'])))}
    assert set(got['parts']) == set(ref['parts']), (sorted(got['parts']), sorted(ref['parts']))
    for k, v in ref['parts'].items():
        r['part_' + k] = frac(got['parts'][k], v, LOSS_RTOL * max(1.0, abs(v)))
    assert set(got['grads']) == set(ref['grads']), (sorted(got['grads']), sorted(ref['grads']))
    for k, g in ref['grads'].items():
        assert got['grads'][k].shape == g.shape, (k, got['grads'][k].shape, g.shape)
        r['grad_' + k] = frac(got['grads'][k], g, GRAD_RTOL * np.abs(g) + GRAD_MAXTOL * np.abs(g).max())
    if 'preds' in ref:
        r['preds'] = frac(got['preds'], ref['preds'], PRED_RTOL * np.maximum(1.0, np.abs(ref['preds'])))
    return r


def kink_margin(model_key, case, hp, adj, dr, st):
    """Smallest |v| / sum|terms of v| over the nonzero float64 values v that a kink of the model acts on (SimGCL's sign(x),
    HCCF's two LeakyReLUs, LightGCL's clamp at +-5: there the distance to the clamp bound); inf when the model has none.
    Exact zeros (isolated rows) are exact in float32 too and are skipped."""
    name = model_key.split('_')[0]
    best = [np.inf]

    def see(v, terms):
        v, terms = v.detach().double().numpy(), terms.detach().double().numpy()
        nz = v != 0
        if nz.any():
            best[0] = min(best[0], float((np.abs(v[nz]) / terms[nz]).min()))

    f64 = torch.float64
    e0 = torch.cat([case['user_e'], case['item_e']], 0).to(f64)
    if name == 'simgcl':
        a = adj.torch_coo(f64)
        for view in dr['uniforms']:
            x = e0
            for u in view:
                pre = O.propagate(a, x)
                see(pre, O.propagate(a, x.abs()))
                x = O.perturbed(pre, u, hp['eps'])
    elif name == 'hccf':
        nu, keep, slope = case['n_user'], hp['keep_rate'], hp['leaky']
        x = e0
        hs = (case['user_e'].to(f64) @ dr['user_w'].to(f64) * hp['mult'], case['item_e'].to(f64) @ dr['item_w'].to(f64) * hp['mult'])
        for k in range(hp['layer_num']):
            a = O.edge_dropped(adj, dr['edge_keeps'][k], keep, True, f64)
            hyp = []
            for h, kp, xs in zip(hs, dr['hyper_keeps'][k], (x[:nu], x[nu:])):
                h = h * kp.to(f64) / keep if keep != 1.0 else h
                inner = h.T @ xs
                see(inner, h.T.abs() @ xs.abs())
                act = O.leaky(inner, slope)
                outer = h @ act
                see(outer, h.abs() @ act.abs())
                hyp.append(O.leaky(outer, slope))
            x = O.propagate(a, x) + torch.cat(hyp, 0)
    elif name == 'lightgcl':
        ladj = O.lightgcl_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
        svd = [torch.from_numpy(st['svd_' + k]).to(f64) for k in ('ut', 'vt', 'u_mul_s', 'v_mul_s')]
        eu, ei, gu, gi = O.lightgcl_embeds(ladj, case['user_e'].to(f64), case['item_e'].to(f64), hp['layer_num'], *svd)
        for g, e, idx in ((gu, eu, case['ancs']), (gi, ei, case['poss'])):
            prod = g[idx] * e[idx] / hp['temp']
            s = prod.sum(1)
            see(s.abs() - 5.0, prod.abs().sum(1))
    return best[0]


# ---- whole steps with the BPR term replaced: MixGCF and the sampled softmax loss (tests/test_gpu_mixgcf.py, test_gpu_ssm.py,
# tests/test_host_mixgcf.py, test_host_ssm.py) ----------------------------------------------------------------------------------

# (model_key, hyper-parameters over the goldens') of every BPR model.  NCL's context layer 2 high_order lies beyond (3, 2),
# inside (3, 1) and at the last (2, 1) of the L + 1 layers MixGCF mixes; HCCF's hyper branch at two widths with injected drops
BPR_TERM_MODELS = [('lightgcn', {}), ('simgcl', {}), ('sgl', {}),
                   ('ncl', dict(layer_num=3, high_order=2)), ('ncl', dict(layer_num=3, high_order=1)), ('ncl', dict(layer_num=2, high_order=1)),
                   ('hccf', dict(hyper_num=128, keep_rate=0.5)), ('hccf', dict(hyper_num=16, keep_rate=0.5)),
                   ('lightgcl', dict(dropout=0))]
BPR_TERM_DIMS = (20, 64, 128)       # the FFMA contraction with idle propagation lanes, a tensor-core contraction, the widest row
BPR_TERM_TAU, BPR_TERM_SMALL_TAU = 0.1, 0.02
# cases whose default seed puts a kink input within KINK_MARGIN of its |term| sum: the first later seed that does not
BPR_TERM_SEEDS = {('simgcl', 128, None): 43, ('hccf', 64, 128): 43, ('hccf', 128, 128): 42}     # (model_key, dim, hyper_num)
PICK_GAP_RTOL = 1e-4                # a MixGCF pick is decided when its score beats the runner-up by this much of their |terms|


def bpr_term_cases(ssm: bool):
    """(model_key, hyper-parameter overrides, embedding_size, M, sampled-softmax tau or None) of every whole-step case: each
    BPR model at each dim with M = 8, one row at M = 32 and, for the sampled softmax loss, one row at a small tau."""
    tau = BPR_TERM_TAU if ssm else None
    out = [(m, hp, d, 8, tau) for m, hp in BPR_TERM_MODELS for d in BPR_TERM_DIMS]
    out.append(('lightgcl', dict(dropout=0), 64, 32, tau))
    if ssm:
        out.append(('ncl', dict(layer_num=3, high_order=1), 64, 8, BPR_TERM_SMALL_TAU))
    return out


IN_BATCH_SMALLEST_TAU = 'min'      # the smallest tau engine.ssm_in_batch_sum accepts for the case's B and weights


def in_batch_step_cases():
    """(id, model_key, case name, hyper-parameter overrides, dim, tau, deterministic, tensor cores, the kernel the weighted
    forward must take) of every whole step of train.ssm_in_batch: the goldens' ``small`` rows; each BPR model at every
    BPR_TERM_DIMS at tau 0.1, on the train.deterministic route at d = 64 and at d = 64, tau 0.5 (3xFP16 on the graph of
    ``path_case``); d = 32 at tau 0.1 and 0.5 for LightGCN and HCCF; NCL (3, 1) and LightGCL at IN_BATCH_SMALLEST_TAU; HCCF
    on the FP32-FMA contraction."""
    hccf = dict(hyper_num=128, keep_rate=0.5)
    rows = [(f'{m}-small', m, 'small', {}, 64, BPR_TERM_TAU, False, True, 'tf32x3') for m in ('lightgcn', 'simgcl', 'sgl')]

    def row(m, hp, d, tau, det=False, tc=True):
        # tau 0.1: offset 14.4, past the weighted 3xFP16 bound; tau 0.5: 2.9 + (1 + log2 27.3) / 2 = 5.8 <= 13.5 on these graphs
        kind = 'ffma' if not tc or d not in (32, 64) else 'f16x3' if tau == 0.5 else 'tf32x3'
        rid = '-'.join([m] + [f'{k}{v}' for k, v in sorted(hp.items())]) + f'-paths-d{d}' + \
            ('' if tau == BPR_TERM_TAU else f'-tau{tau}') + ('-det' if det else '') + ('' if tc else '-ffma')
        return rid, m, 'paths', hp, d, tau, det, tc, kind

    for m, hp in BPR_TERM_MODELS:
        rows += [row(m, hp, d, BPR_TERM_TAU) for d in BPR_TERM_DIMS]
        rows += [row(m, hp, 64, BPR_TERM_TAU, det=True), row(m, hp, 64, 0.5)]
    for m, hp in (('lightgcn', {}), ('hccf', hccf)):
        rows += [row(m, hp, 32, BPR_TERM_TAU), row(m, hp, 32, 0.5)]
    rows += [row('ncl', dict(layer_num=3, high_order=1), 64, IN_BATCH_SMALLEST_TAU), row('lightgcl', dict(dropout=0), 64, IN_BATCH_SMALLEST_TAU)]
    rows.append(row('hccf', hccf, 64, BPR_TERM_TAU, tc=False))
    return rows


def bpr_term_case_id(case):
    m, hp, d, M, tau = case
    return '-'.join([m] + [f'{k}{v}' for k, v in sorted(hp.items())] + [f'd{d}', f'M{M}'] + ([] if tau is None else [f'tau{tau}']))


def bpr_term_setup(model_key, hp_over, dim):
    """-> case, hp, adjacency, draws and injected state of one whole-step case on the graph of ``path_case``."""
    case = path_case(dim, seed=BPR_TERM_SEEDS.get((model_key, dim, hp_over.get('hyper_num')), 41))
    hp = dict(path_hp(model_key, dim), **hp_over)
    adj = O.normalized_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item'])
    dr = replay.draws(model_key, case, hp, adj)
    return case, hp, adj, dr, path_state(model_key, case, hp, adj, dr)


def bpr_tables(model_key, case, hp, adj, dr, params):
    """The tables the BPR term of ``replay.oracle_loss`` reads, in the dtype of ``params``: (summed user table, summed item
    table, item rows of layers 0 .. L of the same view).  LightGCN: its edge-dropped view; SimGCL, SGL: the un-augmented view;
    NCL: the first L + 1 of its max(L, 2 high_order) layers; HCCF: x_k = gcn_(k-1) + hyper_(k-1) with the injected edge and
    hyper keeps; LightGCL: the per-layer Z on its own adjacency (dropout 0)."""
    name = model_key.split('_')[0]
    ue, ie = params['user_embeds'], params['item_embeds']
    dt, nu, L = ue.dtype, case['n_user'], hp['layer_num']
    e0 = torch.cat([ue, ie], 0)
    if name == 'ncl':
        e, xs = O.ncl_embeds_list(adj.torch_coo(dt), e0, L, hp['high_order'])
        xs = xs[:L + 1]
    elif name == 'hccf':
        e, gcn, hyp = O.hccf_embeds(adj, ue, ie, params['user_hyper_embeds'], params['item_hyper_embeds'], L, hp['keep_rate'],
                                    hp['mult'], hp['leaky'], dr['edge_keeps'], dr['hyper_keeps'])
        xs = [e0] + [g + h for g, h in zip(gcn, hyp)]
    else:
        if name == 'lightgcn':
            a_t = O.edge_dropped(adj, dr['edge_keep'], hp['keep_rate'], False, dt)
        elif name == 'lightgcl':
            assert hp['dropout'] == 0
            a_t = O.lightgcl_adjacency(case['rows'], case['cols'], case['n_user'], case['n_item']).torch_coo(dt)
        else:                                   # SimGCL's clean view, SGL's keep_rate 1.0 view
            a_t = adj.torch_coo(dt)
        xs = [e0]
        for _ in range(L):
            xs.append(torch.sparse.mm(a_t, xs[-1]))
        e = sum(xs)
    return e[:nu], e[nu:], [x[nu:] for x in xs]


def bpr_part(model_key, ue, ie, batch):
    """The BPR term of ``replay.oracle_loss`` on summed tables, in the oracle's own expression for the model."""
    ancs, poss, negs = batch
    a, p, n = ue[ancs], ie[poss], ie[negs]
    if model_key.split('_')[0] in ('hccf', 'lightgcl'):
        return -((a * p).sum(-1) - (a * n).sum(-1)).sigmoid().log().mean()
    return O.bpr_loss_sum(a, p, n) / ancs.shape[0]


def bpr_term_oracle(model_key, case, hp, adj, dr, st, dtype, term, name):
    """The whole step of the oracle in ``dtype`` with its BPR term replaced: ``replay.oracle_loss`` minus its bpr_loss plus
    ``term(users, items, item_layers) / B`` on the tables of ``bpr_tables``, reported as ``name``; backward -> dict(loss,
    parts, grads) of float64 numpy, every parameter's gradient.  Asserts first that the tables are the ones the loss read:
    the BPR term on them equals the oracle's bit for bit."""
    params = path_params(model_key, case, dr, dtype)
    loss, parts = replay.oracle_loss(model_key, case, hp, adj, dr, params, st)
    ue, ie, layers = bpr_tables(model_key, case, hp, adj, dr, params)
    batch = tuple(torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs'))
    assert torch.equal(bpr_part(model_key, ue, ie, batch), parts['bpr_loss']), 'the tables are not the ones the BPR term read'
    t = term(ue, ie, layers) / len(case['ancs'])
    loss = loss - parts.pop('bpr_loss') + t
    parts[name] = t
    loss.backward()
    return dict(loss=float(loss.detach()), parts={k: float(v.detach()) for k, v in parts.items()},
                grads={k: p.grad.double().numpy() for k, p in params.items()})


def train_csr(case):
    """The training matrix as a sorted int64 CSR (rowptr, cols), the form the candidate draw reads."""
    order = np.lexsort((case['cols'], case['rows']))
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(case['rows'], minlength=case['n_user']))]).astype(np.int64)
    return rowptr, case['cols'][order].astype(np.int64)


def pop_draw(case, ancs, negs, M, beta, seed):
    """The train.neg_popularity candidates and fp32 logQ bias a step must draw for the pairs (ancs, ., negs) with ``seed``:
    tests/pop_oracle's draw and bias on the host tables of the case's own training pairs (``train_csr``) -> ([B, M] int64,
    [B, M] float32)."""
    import pop_oracle
    from sslrec_b200 import engine as E
    rowptr, cols = train_csr(case)
    t = E.pop_tables(rowptr, cols, case['n_item'], beta)
    cands = pop_oracle.neg_candidates(ancs, negs, M, rowptr, cols, case['n_item'], t['table'], int(seed))
    return cands, pop_oracle.bias(ancs, cands, t['lp'], t['lz_pop'], t['lz_uni'])


def assert_step_seed(model):
    """-> the candidate seed of the model's last step, asserting it is the last seed the step drew from its stream."""
    seed = int(model._mix_seed)
    assert seed == model._seeds.state, 'the candidates were not drawn with the step\'s last seed'
    return seed


def mixgcf_pick_check(users, layers, ancs, poss, cands, alpha_t, picks):
    """The picks of a MixGCF step against float64: ``users`` / ``layers`` the float64 summed user table and item layer rows,
    ``picks`` [B, L+1] the step's.  Where the best float64 score beats the best other item's by more than PICK_GAP_RTOL of
    the sum of their |terms| (sum_k |u_k m_k|) the pick must be float64's; -> the fraction of (pair, layer) picks so decided."""
    a = alpha_t.double()[:, None, :, None]
    xp = torch.stack([x[poss] for x in layers], 1)[:, None]
    xc = torch.stack([x[cands] for x in layers], 2)                      # [B, M, L+1, d]
    m = a * xp + (1 - a) * xc
    u = users[ancs][:, None, None, :]
    s, A = (u * m).sum(-1), (u * m).abs().sum(-1)                        # [B, M, L+1]
    want = mixgcf_oracle.picks(users, layers, ancs, poss, cands, alpha_t)
    j = s.argmax(1, keepdim=True)
    other = torch.where(cands[:, :, None] == want[:, None, :], torch.full_like(s, -np.inf), s)    # candidates of other items
    k = other.argmax(1, keepdim=True)
    gap = s.gather(1, j) - other.gather(1, k)
    decided = (gap > PICK_GAP_RTOL * (A.gather(1, j) + A.gather(1, k)))[:, 0]
    bad = decided & (picks != want)
    assert not bool(bad.any()), f'{int(bad.sum())} decided picks differ from float64 (first (pair, layer): {bad.nonzero()[0].tolist()})'
    return float(decided.double().mean())


def golden_loss_grads_close(g, loss, parts, named_params, what=''):
    """cal_loss and the gradients of a drop-in model against a golden case: loss and terms |d| <= 1e-5 max(1, |ref|);
    gradients rtol 2e-4 + 5e-6 max|ref| (head, row sums and |.| sum for the large tables the golden stores in part)."""
    assert abs(loss.item() - float(g['loss'])) <= 1e-5 * max(1.0, abs(float(g['loss']))), (what, loss.item(), float(g['loss']))
    for k, v in parts.items():
        assert abs(float(v) - float(g['part_' + k])) <= 1e-5 * max(1.0, abs(float(g['part_' + k]))), (what, k, float(v), float(g['part_' + k]))
    for name, p in named_params:
        gr = p.grad
        if 'grad_' + name in g:
            ref = g['grad_' + name]
            close(gr, ref, 2e-4, 5e-6 * np.abs(ref).max() + 1e-9, what + 'grad_' + name)
        else:
            ref = g['grad_' + name + '_head']
            scale = g['grad_' + name + '_abssum'] / gr.numel()
            close(gr[:32], ref, 2e-4, 2e-4 * scale + 1e-9, what + 'grad_' + name + '_head')
            close(gr.double().sum(1), g['grad_' + name + '_rowsum'], 1e-3, 1e-3 * scale * gr.shape[1], what + 'grad_' + name + '_rowsum')
            assert abs(gr.double().abs().sum().item() - g['grad_' + name + '_abssum']) <= 1e-4 * g['grad_' + name + '_abssum'], (what, name)


# ---- NCL's k-means, one Lloyd pass (tests/test_gpu_kmeans.py, tests/test_host_kmeans.py) -----------------------------------------

U32 = 2.0 ** -24                      # unit roundoff of fp32
KMEANS_SMEM_BYTES = 200 * 1024        # ssl_kmeans_workspace's shared-memory budget
KMEANS_MAX_CTAS = 132                 # one CTA per SM of an H100 SXM
KMEANS_ROWS_PER_ROUND = 4             # the widest kmeans_assign_kernel<R>, which the workspace is sized for
KMEANS_EPS = float(np.float32(1e-6))  # the update kernel's empty-cluster guard, as the fp32 constant it is


def gamma(m):
    """gamma_m = m u / (1 - m u): the relative error bound of m chained fp32 roundings."""
    return m * U32 / (1 - m * U32)


def kmeans_smem_floats(K, d, W, R=KMEANS_ROWS_PER_ROUND):
    """csrc/kmeans_assign.cuh smem_floats: padded centroids, staged rows, W warp slabs and W count rows."""
    return K * (d + 1) + W * R * d + W * K * d + W * K


def kmeans_k_limit(d, W):
    """The largest K whose launch with W warps fits the shared-memory budget."""
    R = KMEANS_ROWS_PER_ROUND
    return (KMEANS_SMEM_BYTES // 4 - W * R * d) // (d + 1 + W * d + W)


def kmeans_launch(n, d, K):
    """ssl_kmeans_workspace's partition restated -> (n_cta, W, rows_per_cta, rows_per_warp), or None when K * d does not fit.
    W halves from 8 until the launch fits; about 8 rows per warp, at most one CTA per SM."""
    W = 8
    while W > 1 and 4 * kmeans_smem_floats(K, d, W) > KMEANS_SMEM_BYTES:
        W //= 2
    if 4 * kmeans_smem_floats(K, d, W) > KMEANS_SMEM_BYTES:
        return None
    n_cta = min(-(-n // (W * 8)), KMEANS_MAX_CTAS)
    rows_per_cta = -(-n // n_cta)
    return n_cta, W, rows_per_cta, -(-rows_per_cta // W)


def kmeans_case(n, d, K, seed, device='cpu'):
    """-> x [n, d], centroids [K, d] (float32) and a given incoming assignment [n] (int64) for one Lloyd pass.

    The centroids are t.rand draws (aug_utils.py:147) with exact ties planted: centroid pairs equal across lanes (k, k + 1),
    (4, 21) and within one lane (5, 37), (9, 41), and two or three all-zero rows, which is what an empty cluster becomes.
    Half the rows sit near a centroid drawn uniformly (so duplicates and zeros win rows and their twins stay empty), a
    quarter are uniform like the centroids (generic near-ties), and the rest are exact copies of a centroid or exact zeros
    (distance exactly 0)."""
    g = torch.Generator(device=device).manual_seed(seed)
    f32 = dict(device=device, dtype=torch.float32)
    c = torch.rand(K, d, generator=g, **f32)
    if K >= 3:
        for z in (K // 3, K - 1, K // 3 + 32):
            if z < K:
                c[z] = 0.0
        for i, j in ((1, 2), (4, 21), (5, 37), (9, 41)):
            if j < K:
                c[j] = c[i]
    src = torch.randint(0, K, (n,), generator=g, device=device)
    kind = torch.randint(0, 8, (n,), generator=g, device=device)
    x = c[src] + 0.05 * torch.randn(n, d, generator=g, **f32)
    x = torch.where((kind >= 4)[:, None], torch.rand(n, d, generator=g, **f32), x)
    x = torch.where((kind == 6)[:, None], c[src], x)
    x = torch.where((kind == 7)[:, None], torch.zeros_like(x), x)
    given = torch.randint(0, K, (n,), generator=g, device=device)
    return x, c, given


def _kmeans_dist64(x, c):
    """float64 sum_j (x_j - c_j)^2 of every (row, centroid) pair [n, K], in row chunks of about 2^27 elements."""
    x, c = x.double(), c.double()
    step = max(1, (1 << 27) // max(1, c.shape[0] * c.shape[1]))
    return torch.cat([(x[i:i + step, None, :] - c[None]).square().sum(-1) for i in range(0, x.shape[0], step)], 0)


def kmeans_pass_check(x, c0, a0, ch0, out, W, n_cta, rows_per_warp):
    """One Lloyd pass from centroids ``c0`` and incoming assignment ``a0`` (counter value ``ch0``) against float64; ``out``
    holds the pass's ``assign`` [n], ``cents`` [K, d], ``counts`` [K] and ``changed`` (int).  Asserts, and returns the worst
    err / bound of the assignment and the centroids:

    - lowest id on exact ties: every row goes to the lowest id of its centroid's class of bit-equal rows;
    - the assignment: with D the float64 distances, the kernel's fp32 chain (one rounding per difference, d fused
      multiply-adds) is within gamma_{d+2} D of D.  Where the best and second-best class differ by more than both bounds,
      the row must go to float64's argmin; elsewhere its distance must be within both bounds of the minimum;
    - counts == bincount(assign), and changed == ch0 + the number of rows whose assignment differs from a0;
    - centroids: the float64 mean of each cluster's members, sum / (count + 1e-6).  A member passes through at most
      rows_per_warp + W + n_cta fp32 additions (its warp's slab, the per-CTA sum over W slabs, the update's sum over n_cta
      partials) and two more roundings (the denominator, the division): the error is at most gamma_{m+2} sum |x| / (count + 1e-6)
      over the members.  An empty cluster is exactly 0."""
    n, d = x.shape
    K = c0.shape[0]
    dev = x.device
    a = out['assign'].to(dev)
    assert a.dtype == torch.int64 and a.shape == (n,)
    assert bool(((a >= 0) & (a < K)).all()), 'assignment out of range'
    cls, inv = torch.unique(c0.to(dev).double(), dim=0, return_inverse=True)
    lowest = torch.full((cls.shape[0],), K, dtype=torch.int64, device=dev).scatter_reduce(0, inv, torch.arange(K, device=dev), 'amin')
    canon = lowest[inv]
    tie_bad = canon[a] != a
    assert not bool(tie_bad.any()), f'{int(tie_bad.sum())} rows went to a higher id of an exact tie (first: row {int(tie_bad.nonzero()[0])})'

    D = _kmeans_dist64(x, cls)                                                  # [n, classes]
    bnd = gamma(d + 2) * D
    got = D.gather(1, inv[a][:, None])[:, 0]
    best, arg = D.min(1)
    bb = bnd.gather(1, arg[:, None])[:, 0]
    if cls.shape[0] > 1:
        two = D.topk(2, dim=1, largest=False)
        second, arg2 = two.values[:, 1], two.indices[:, 1]
        safe = (second - best) > bb + bnd.gather(1, arg2[:, None])[:, 0]
    else:
        safe = torch.ones(n, dtype=torch.bool, device=dev)
    wrong = safe & (a != lowest[arg])
    assert not bool(wrong.any()), f'{int(wrong.sum())} rows with a clear nearest centroid assigned elsewhere (first: row {int(wrong.nonzero()[0])})'
    slack = bnd.gather(1, inv[a][:, None])[:, 0] + bb
    excess = got - best
    bad = ~(excess <= slack)
    assert not bool(bad.any()), f'{int(bad.sum())} rows assigned beyond the distance bound, max excess / bound {(excess / slack.clamp_min(1e-300)).max().item():.3e}'
    r_assign = float((excess / slack.clamp_min(1e-300)).max()) if n else 0.0
    # the smallest gap between the best and second-best class, as a multiple of both bounds (> 1: the argmin is exact)
    tie_gap = float(((second - best) / (bb + bnd.gather(1, arg2[:, None])[:, 0]).clamp_min(1e-300)).min()) if cls.shape[0] > 1 else float('inf')

    want = torch.bincount(a, minlength=K)
    cnt = out['counts'].to(dev).reshape(-1)
    assert torch.equal(cnt.double(), want.double()), f'counts differ from bincount(assign) in {int((cnt.double() != want.double()).sum())} clusters'
    ch_want = int(ch0) + int((a != a0.to(dev)).sum())
    assert int(out['changed']) == ch_want, f'changed {int(out["changed"])}, want {ch_want}'

    x64 = x.double()
    S = torch.zeros(K, d, dtype=torch.float64, device=dev).index_add_(0, a, x64)
    A = torch.zeros(K, d, dtype=torch.float64, device=dev).index_add_(0, a, x64.abs())
    den = want.double()[:, None] + KMEANS_EPS
    ref = S / den
    cb = gamma(rows_per_warp + W + n_cta + 2) * A / den
    c = out['cents'].to(dev).double()
    empty = want == 0
    assert torch.equal(c[empty], torch.zeros_like(c[empty])), 'an empty cluster is not exactly 0'
    err = (c - ref).abs()
    bad = ~(err <= cb)
    assert not bool(bad.any()), f'centroids: {int(bad.sum())} / {bad.numel()} off, max err / bound {(err / cb.clamp_min(1e-300)).max().item():.3e}'
    r_cents = float((err / cb.clamp_min(1e-300)).max())
    return {'assign': r_assign, 'cents': r_cents, 'tie_gap': tie_gap}


def close(a, b, rtol, atol, what):
    a = np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a, dtype=np.float64)
    b = np.asarray(b.detach().cpu() if isinstance(b, torch.Tensor) else b, dtype=np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = np.abs(a - b)
    tol = atol + rtol * np.abs(b)
    bad = err > tol
    assert not bad.any(), f'{what}: {bad.sum()} / {bad.size} off, max err {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)} (ref {b.flat[err.argmax()]:.4e})'
