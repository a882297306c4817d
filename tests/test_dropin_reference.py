"""Executed drop-in (SURVEY.md 8b): the UNMODIFIED reference tree (oracle/_ref, vendored by oracle/vendor_ref.py) with the
seven one-line shim modules of INTEGRATION.md section 2 overlaid, driven through the reference's own
``build_data_handler -> build_model (models/bulid_model.py:4-15) -> build_trainer -> Trainer.train_epoch
(trainer/trainer.py:51-84) -> Metric.eval (trainer/metrics.py:82-127)`` from the five in-scope ``config/modelconf/*.yml``
files UNCHANGED.  One subprocess per model (the reference's config is a module-level singleton)."""
import json
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, 'oracle', '_ref')
SHIMS = {'lightgcn': 'LightGCN', 'simgcl': 'SimGCL', 'sgl': 'SGL', 'ncl': 'NCL', 'hccf': 'HCCF', 'directau': 'DirectAU', 'lightgcl': 'LightGCL'}


def _graph(n_user=600, n_item=500, n_edge=9000, seed=3):
    rs = np.random.RandomState(seed)
    key = np.unique(rs.randint(0, n_user, 4 * n_edge).astype(np.int64) * n_item + rs.randint(0, n_item, 4 * n_edge))
    key = rs.permutation(key)[:n_edge]
    # every user and item gets at least one training edge
    key = np.unique(np.concatenate([key, np.arange(n_user) * n_item + rs.randint(0, n_item, n_user), rs.randint(0, n_user, n_item) * n_item + np.arange(n_item)]))
    key = rs.permutation(key)
    n_tst = len(key) // 10
    mk = lambda k: sp.coo_matrix((np.ones(len(k)), (k // n_item, k % n_item)), shape=(n_user, n_item))
    return mk(key[2 * n_tst:]), mk(key[:n_tst]), mk(key[n_tst:2 * n_tst])


def make_scratch_tree():
    """scratch/: config, data_utils, trainer -> symlinks into oracle/_ref; models/ -> a directory of symlinks to the
    reference's files EXCEPT the seven shimmed modules, which are the one-line re-exports; datasets/ -> a small synthetic
    graph pickled the way the reference loads it (data_handler_general_cf.py:12-35)."""
    d = tempfile.mkdtemp(prefix='sslrec_dropin_')
    for sub in ('config', 'data_utils', 'trainer'):
        os.symlink(os.path.join(REFDIR, sub), os.path.join(d, sub))
    src_models = os.path.join(REFDIR, 'models')
    os.makedirs(os.path.join(d, 'models', 'general_cf'))
    for name in os.listdir(src_models):
        if name != 'general_cf':
            os.symlink(os.path.join(src_models, name), os.path.join(d, 'models', name))
    for name in os.listdir(os.path.join(src_models, 'general_cf')):
        stem = name[:-3] if name.endswith('.py') else None
        dst = os.path.join(d, 'models', 'general_cf', name)
        if stem in SHIMS:
            with open(dst, 'w') as f:
                f.write(f'from sslrec_b200.general_cf.{stem} import {SHIMS[stem]}          # noqa: F401\n')
        else:
            os.symlink(os.path.join(src_models, 'general_cf', name), dst)
    dd = os.path.join(d, 'datasets', 'general_cf', 'sparse_gowalla')
    os.makedirs(dd)
    for fname, m in zip(('train_mat.pkl', 'valid_mat.pkl', 'test_mat.pkl'), _graph()):
        with open(os.path.join(dd, fname), 'wb') as f:
            pickle.dump(m, f)
    return d


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFDIR, 'models')), reason='oracle/_ref not vendored (python oracle/vendor_ref.py)')
def test_scratch_tree_overlays_only_the_shims():
    d = make_scratch_tree()
    gc = os.path.join(d, 'models', 'general_cf')
    for stem, cls in SHIMS.items():
        p = os.path.join(gc, stem + '.py')
        assert not os.path.islink(p) and open(p).read().strip().startswith(f'from sslrec_b200.general_cf.{stem} import {cls}')
    others = [n for n in os.listdir(gc) if n.endswith('.py') and n[:-3] not in SHIMS]
    assert others and all(os.path.islink(os.path.join(gc, n)) for n in others)
    for sub in ('config', 'data_utils', 'trainer'):
        assert os.path.realpath(os.path.join(d, sub)) == os.path.realpath(os.path.join(REFDIR, sub))
    assert os.path.islink(os.path.join(d, 'models', 'bulid_model.py'))


@pytest.mark.gpu
@pytest.mark.parametrize('model', ['lightgcn', 'simgcl', 'sgl', 'ncl', 'hccf'])
def test_reference_tree_trains_and_evaluates_our_models(model):
    if not os.path.isdir(os.path.join(REFDIR, 'models')):
        pytest.skip('oracle/_ref not vendored')
    d = make_scratch_tree()
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dropin_driver.py'), d, ROOT, model], capture_output=True, text=True, timeout=600)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('DROPIN_JSON ')]
    assert r.returncode == 0 and lines, r.stdout[-2000:] + '\n' + r.stderr[-3000:]
    out = json.loads(lines[-1][len('DROPIN_JSON '):])
    assert out['model_class'] == f'sslrec_b200.general_cf.{model}.{SHIMS[model]}'          # build_model found the shimmed class
    assert out['trainer_class'] == 'trainer.trainer.Trainer'                                # the reference's own trainer
    assert out['device'].startswith('cuda') and out['native_launches'] > 0
    assert {'user_embeds', 'item_embeds'} <= set(out['state_dict_keys']) and out['state_dict_roundtrip']
    s0, o0 = out['step0'], out['oracle_step0']
    for k, v in o0.items():
        assert abs(s0[k] - v) <= 1e-5 * max(1.0, abs(v)), (k, s0[k], v)
    assert np.isfinite(s0['loss']) and out['grad_finite'] and out['params_moved'] > 0
    # the reference's Metric.eval (torch.topk on full_predict's masked scores) and the native evaluator agree
    for metric, vals in out['reference_metric_eval'].items():
        assert np.allclose(vals, out['native_eval'][metric], rtol=0, atol=1e-9), (metric, vals, out['native_eval'][metric])
        assert all(0.0 <= v <= 1.0 for v in vals)
    print(model, 'step0', s0, 'recall@k', out['reference_metric_eval'].get('recall'))
