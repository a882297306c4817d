"""Generate ``tests/golden/*.npz`` by running the UNMODIFIED reference (HKUDS/SSLRec, the
checkout named by $SSLREC_REFERENCE) on CPU with injected inputs.  TEST INFRASTRUCTURE ONLY.

Needs the reference checkout; the outputs are committed so the tests never need the reference.  Usage:

    python oracle/gen_golden.py            # all cases (one subprocess per case)
    python oracle/gen_golden.py --one lightgcn tiny

How the reference is driven (SURVEY.md section 8c): a scratch CWD holds symlinks to the
reference's ``config/ data_utils/ models/ trainer/`` and a ``datasets/general_cf/sparse_gowalla``
directory with *our* synthetic pickles (oracle/inputs.py); ``sys.argv`` is set before
``config.configurator`` is imported; hyper-parameters are overridden in ``configs['model']`` in
place; parameters are injected through ``load_state_dict``; every random draw the reference
makes inside ``cal_loss`` (``t.rand`` in aug_utils.py:28,49,130,147 and ``F.dropout`` in
hccf.py:48-49) is served from a queue filled from ``inputs.uniform_stream`` so the oracle and
the CUDA path can replay the same bits.  ``Tensor.cuda`` is shimmed to identity because
aug_utils.py:130,147-154 hard-code ``.cuda()``.  No reference source is modified or copied.
"""
from __future__ import annotations

import argparse
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get('SSLREC_REFERENCE', '/root/reference')
OUT = os.path.join(ROOT, 'tests', 'golden')

# model -> overrides of configs['model'] (BASELINE.json values where they differ from the YAML)
MODEL_HP = {
    'lightgcn': dict(layer_num=3, keep_rate=0.5),
    'simgcl': dict(layer_num=3, temperature=0.2),
    'sgl': dict(layer_num=3, keep_rate=0.5, augmentation='edge_drop'),
    'sgl_nd': dict(layer_num=2, keep_rate=0.5, augmentation='node_drop'),
    'ncl': dict(layer_num=3, high_order=2, cluster_num=5),
    'hccf': dict(layer_num=2, keep_rate=0.5, hyper_num=16, leaky=0.5),
    # the YAML sizes of the proto / hyper contrastive models (ncl.yml: cluster_num 50; hccf.yml: hyper_num 128)
    'ncl_k50': dict(layer_num=3, high_order=2, cluster_num=50),
    'hccf_h128': dict(layer_num=2, keep_rate=0.5, hyper_num=128, leaky=0.5),
    'directau': dict(layer_num=2, gamma=2.0),
    'lightgcl': dict(layer_num=2, dropout=0, cl_weight=0.1, reg_weight=1.0e-6, temp=0.1, svd_q=5),
}
CASES = [('lightgcn', 'tiny'), ('simgcl', 'tiny'), ('sgl', 'tiny'), ('sgl_nd', 'tiny'), ('ncl', 'tiny'),
         ('hccf', 'tiny'), ('lightgcn', 'small'), ('simgcl', 'small'), ('sgl', 'small'), ('simgcl', 'mid'),
         ('directau', 'tiny'), ('directau', 'small'), ('lightgcl', 'tiny'), ('lightgcl', 'small'),
         ('ncl_k50', 'small'), ('hccf_h128', 'small')]


def _scratch(case):
    import scipy.sparse as sp
    d = tempfile.mkdtemp(prefix='sslrec_ref_')
    for sub in ('config', 'data_utils', 'models', 'trainer'):
        os.symlink(os.path.join(REF, sub), os.path.join(d, sub))
    dd = os.path.join(d, 'datasets', 'general_cf', 'sparse_gowalla')
    os.makedirs(dd)
    shape = (case['n_user'], case['n_item'])
    trn = sp.coo_matrix((np.ones(len(case['rows'])), (case['rows'], case['cols'])), shape=shape)
    rs = np.random.RandomState(case['seed'] + 77)
    k = 40
    oth = sp.coo_matrix((np.ones(k), (rs.randint(0, shape[0], k), rs.randint(0, shape[1], k))), shape=shape)
    for name, m in (('train_mat.pkl', trn), ('valid_mat.pkl', oth), ('test_mat.pkl', oth)):
        with open(os.path.join(dd, name), 'wb') as f:
            pickle.dump(m, f)
    return d


def run_one(model_key: str, case_name: str):
    sys.path.insert(0, ROOT)
    from oracle import inputs
    case = inputs.make_case(case_name)
    model_name = model_key.split('_')[0]
    scratch = _scratch(case)
    os.chdir(scratch)
    sys.path.insert(0, scratch)
    sys.argv = ['main.py', '--model', model_name, '--device', 'cpu']

    import torch
    import torch.nn.functional as F
    torch.Tensor.cuda = lambda self, *a, **k: self          # aug_utils.py:130,147-154
    queue = []
    real_rand = torch.rand

    def fake_rand(*size, **kw):
        if queue and not kw:
            t = queue.pop(0)
            shp = tuple(size[0]) if len(size) == 1 and not isinstance(size[0], int) else tuple(size)
            assert tuple(t.shape) == shp, (t.shape, shp)
            return t.clone()
        return real_rand(*size, **kw)
    torch.rand = fake_rand
    drop_queue = []
    real_dropout = F.dropout

    def fake_dropout(x, p=0.5, training=True, inplace=False):
        if drop_queue:
            keep = drop_queue.pop(0)
            assert keep.shape == x.shape
            return x * keep.to(x.dtype) / (1.0 - p)
        return real_dropout(x, p, training, inplace)
    F.dropout = fake_dropout

    from config.configurator import configs
    hp = MODEL_HP[model_key]
    configs['model'].update(hp)
    configs['model']['embedding_size'] = case['dim']
    configs['train']['batch_size'] = case['batch']
    from trainer.trainer import init_seed
    from data_utils.build_data_handler import build_data_handler
    from models.bulid_model import build_model
    init_seed()
    dh = build_data_handler()
    dh.load_data()
    model = build_model(dh)
    mc = dict(configs['model'])

    gen = inputs.uniform_stream(case['seed'])
    U, I, D = case['n_user'], case['n_item'], case['dim']
    N = U + I
    adj = dh.torch_adj
    idx = adj._indices().numpy()
    vals = adj._values().numpy()
    nnz = vals.shape[0]
    out = dict(adj_rows=idx[0], adj_cols=idx[1], adj_vals=vals)

    sd = {'user_embeds': case['user_e'].clone(), 'item_embeds': case['item_e'].clone()}
    if model_name == 'hccf':
        H = mc['hyper_num']
        a = float(np.sqrt(6.0 / (D + H)))
        sd['user_hyper_embeds'] = (inputs.draw_uniform(gen, D, H) * 2 - 1) * a
        sd['item_hyper_embeds'] = (inputs.draw_uniform(gen, D, H) * 2 - 1) * a
    if model_name == 'lightgcl':
        a = float(np.sqrt(6.0 / (D + D)))
        for li in range(mc['layer_num']):
            sd[f'Ws.{li}.W'] = (inputs.draw_uniform(gen, D, D) * 2 - 1) * a       # W_contrastive: only reg_params sees it
        out['svd_ut'], out['svd_vt'] = model.ut.numpy().copy(), model.vt.numpy().copy()       # t.svd_lowrank at lightgcl.py:25
        out['svd_u_mul_s'], out['svd_v_mul_s'] = model.u_mul_s.numpy().copy(), model.v_mul_s.numpy().copy()
        out['lgcl_rows'], out['lgcl_cols'] = model.adj.indices().numpy().copy()
        out['lgcl_vals'] = model.adj.values().numpy().copy()
    model.load_state_dict(sd)

    L = mc['layer_num']
    keep = mc.get('keep_rate', 1.0)
    # fill the queues in the order the reference consumes them
    if model_name == 'lightgcn':
        if keep != 1.0:
            queue.append(inputs.draw_uniform(gen, nnz))                       # aug_utils.py:28
    elif model_name == 'simgcl':
        for _view in range(2):
            for _l in range(L):
                queue.append(inputs.draw_uniform(gen, N, D))                  # aug_utils.py:130
    elif model_name == 'sgl':
        for _view in range(2):
            if mc['augmentation'] == 'edge_drop':
                queue.append(inputs.draw_uniform(gen, nnz))                   # sgl.py:27-28
            else:
                queue.append(inputs.draw_uniform(gen, N))                     # sgl.py:24-25, aug_utils.py:49
    elif model_name == 'ncl':
        K = mc['cluster_num']
        queue.append(inputs.draw_uniform(gen, K, D))                          # aug_utils.py:147 (users)
        queue.append(inputs.draw_uniform(gen, K, D))                          # (items)
    elif model_name == 'hccf':
        H = mc['hyper_num']
        for _l in range(L):
            queue.append(inputs.draw_uniform(gen, nnz))                       # hccf.py:47
            drop_queue.append((inputs.draw_uniform(gen, U, H) + keep).floor())   # hccf.py:48
            drop_queue.append((inputs.draw_uniform(gen, I, H) + keep).floor())   # hccf.py:49

    batch = [torch.from_numpy(case[k]) for k in ('ancs', 'poss', 'negs')]
    if model_name == 'ncl':
        batch.append(torch.ones(case['batch'], dtype=torch.int64))
    opt = torch.optim.Adam(model.parameters(), lr=configs['optimizer']['lr'],
                           weight_decay=configs['optimizer']['weight_decay'])     # trainer.py:45-49
    opt.zero_grad()
    loss, parts = model.cal_loss(batch)                                            # trainer.py:65
    assert not queue and not drop_queue, 'injected draws were not all consumed'
    out['loss'] = np.float32(loss.item())
    for k, v in parts.items():
        out['part_' + k] = np.float32(float(v))
    loss.backward()
    for name, p in model.named_parameters():
        out['grad_' + name] = p.grad.detach().numpy().copy()
    if model_name == 'ncl':
        out['user_centroids'] = model.user_centroids.numpy()
        out['item_centroids'] = model.item_centroids.numpy()
        out['user2cluster'] = model.user2cluster.numpy()
        out['item2cluster'] = model.item2cluster.numpy()

    # evaluation path (metrics.py:95-108) before the optimiser step: first Bt users, dense train mask
    import scipy.sparse as sp
    bt = min(64, U)
    users = torch.arange(bt, dtype=torch.int64)
    trn_csr = sp.csr_matrix((np.ones(len(case['rows'])), (case['rows'], case['cols'])), shape=(U, I))
    mask = torch.from_numpy((trn_csr[:bt].toarray() != 0).astype(np.float64)).long()
    model.eval()
    with torch.no_grad():
        preds = model.full_predict([users, mask])
    k = min(40, I)
    top = torch.topk(preds, k=k)
    out['topk_idx'] = top.indices.numpy()
    out['topk_val'] = top.values.numpy()
    if case_name == 'tiny':
        out['preds'] = preds.numpy()
    model.train()

    opt.step()                                                                     # trainer.py:68
    for name, p in model.named_parameters():
        if case_name == 'tiny' or name.endswith('hyper_embeds'):
            out['new_' + name] = p.detach().numpy().copy()
        else:
            out['new_' + name + '_head'] = p.detach().numpy()[:32].copy()
    if case_name != 'tiny':
        for name in list(out):
            if name.startswith('grad_') and out[name].shape[0] > 64:
                g = out.pop(name)
                out[name + '_head'] = g[:32].copy()
                out[name + '_rowsum'] = g.astype(np.float64).sum(1)
                out[name + '_abssum'] = np.float64(np.abs(g.astype(np.float64)).sum())
        out.pop('adj_rows'); out.pop('adj_cols')
        out['adj_vals_sum'] = np.float64(out.pop('adj_vals').astype(np.float64).sum())
    out['hp_json'] = np.array(repr({k: mc[k] for k in sorted(mc) if k != 'name'}))
    out['opt_lr'] = np.float64(configs['optimizer']['lr'])                     # trainer.py:45-49
    out['opt_weight_decay'] = np.float64(configs['optimizer']['weight_decay'])
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f'{model_key}_{case_name}.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, {k: (v.shape if hasattr(v, 'shape') else v) for k, v in out.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--one', nargs=2, default=None)
    a = ap.parse_args()
    if a.one:
        run_one(*a.one)
        return
    for m, c in CASES:
        subprocess.run([sys.executable, os.path.abspath(__file__), '--one', m, c], check=True)


if __name__ == '__main__':
    main()
