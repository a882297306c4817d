"""Resuming training from a checkpoint (``train.checkpoint_step`` / ``train.resume_path``) on the GPU.

Under train.deterministic, for all seven models (SGL with edge and node drop; NCL with a resume between re-clusters and one that
lands on a re-cluster), eager and with train.cuda_graph, with the host and the device loader: 2 epochs with a checkpoint per epoch,
then fresh global generators, data handler, model and trainer resuming for epochs 2 and 3, end with the same bits as 4 epochs
without a stop -- parameters, Adam moments and step count, epoch losses, evaluation metrics, seed stream and global generators.
With patience, a resume inside the waiting period picks the same best epoch and best model.  Without train.deterministic, the
resumed run sees the same batches and seeds, and its losses agree to fp32 rounding."""
import shutil

import numpy as np
import pytest
import torch

from test_host_resume import make_run

pytestmark = pytest.mark.gpu

MODELS = [('lightgcn', {}), ('simgcl', {}), ('sgl', {}), ('sgl_nd', {}), ('ncl', {'epoch_period': 2}), ('ncl', {'epoch_period': 3}),
          ('hccf', {}), ('lightgcl', {}), ('directau', {})]


def _scramble():
    np.random.seed(12345)
    torch.manual_seed(54321)
    torch.cuda.manual_seed_all(999)


def _train(key, model_hp, train, seed_globals=True, record_steps=False):
    """Trainer.train on a fresh run; records epoch losses, evaluations (the final test last), the epochs NCL clustered in and,
    with ``record_steps``, every eager step's batch and seed-stream position."""
    m, tr, _ = make_run(key, device='cuda', train=train, model=model_hp, seed_globals=seed_globals)
    rec = {'losses': {}, 'evals': [], 'clusters': [], 'steps': [], 'epoch': None}
    train_epoch, evaluate = tr.train_epoch, tr.evaluate

    def epoch_hook(model, e):
        rec['epoch'] = e
        rec['losses'][e] = train_epoch(model, e)
        return rec['losses'][e]

    def eval_hook(model, epoch_idx=None, **kw):
        out = evaluate(model, epoch_idx, **kw)
        rec['evals'].append((epoch_idx, out))
        return out

    tr.train_epoch, tr.evaluate = epoch_hook, eval_hook
    if hasattr(m, '_cluster'):
        cluster = m._cluster
        m._cluster = lambda: (rec['clusters'].append(rec['epoch']), cluster())[1]
    if record_steps:
        cal_loss = m.cal_loss
        m.cal_loss = lambda b: (rec['steps'].append(([t.detach().cpu().clone() for t in b], m._seeds.state)), cal_loss(b))[1]
    out = tr.train(m)
    if tr._graphed is not None:
        tr._graphed.close()                     # the device step count back on the host
    torch.cuda.synchronize()
    rec['params'] = {n: p.detach().clone() for n, p in out.named_parameters()}
    rec['adam'] = [dict(tr.optimizer.state[p]) for p in m.parameters()]
    rec['seeds'] = m._seeds.state
    rec['numpy'] = np.random.get_state()
    rec['torch'] = torch.get_rng_state()
    rec['trainer'], rec['model'] = tr, m
    return rec


def _checkpoint(tmp_path, key):
    name = key.split('_')[0]
    return tmp_path / 'checkpoint' / name / f'{name}-synthetic-resume.pth'


def _assert_same_params_and_adam(ref, res):
    for n in ref['params']:
        assert torch.equal(ref['params'][n], res['params'][n]), (n, (ref['params'][n] - res['params'][n]).abs().max().item())
    for a, b in zip(ref['adam'], res['adam']):
        assert a.keys() == b.keys()
        if a:
            assert a['step'] == b['step'], (a['step'], b['step'])
            assert torch.equal(a['exp_avg'], b['exp_avg']) and torch.equal(a['exp_avg_sq'], b['exp_avg_sq'])


def _assert_same_evals(a, b):
    assert [e for e, _ in a] == [e for e, _ in b]
    for (e, x), (_, y) in zip(a, b):
        for m in x:
            assert np.array_equal(x[m], y[m]), (e, m, x[m], y[m])


def _no_svd(*a, **kw):
    raise AssertionError('svd_lowrank ran again: the restored factors were not used')


@pytest.mark.parametrize('graph,loader', [(False, 'host'), (False, 'device'), (True, 'host'), (True, 'device')])
@pytest.mark.parametrize('key,hp', MODELS, ids=[k + ''.join(f'-{a}{b}' for a, b in h.items()) for k, h in MODELS])
def test_resume_is_bit_identical(tmp_path, monkeypatch, key, hp, graph, loader):
    monkeypatch.chdir(tmp_path)
    base = dict(deterministic=True, cuda_graph=graph, device_loader=loader == 'device')
    ref = _train(key, hp, dict(base, epoch=4))
    first = _train(key, hp, dict(base, epoch=2, checkpoint_step=1))
    assert first['losses'] == {e: ref['losses'][e] for e in (0, 1)}
    path = _checkpoint(tmp_path, key)
    assert path.exists()
    _scramble()
    if key == 'lightgcl':
        monkeypatch.setattr(torch, 'svd_lowrank', _no_svd)
    res = _train(key, hp, dict(base, epoch=4, resume_path=str(path)), seed_globals=False)
    assert sorted(res['losses']) == [2, 3]
    for e in (2, 3):
        assert res['losses'][e] == ref['losses'][e], (e, res['losses'][e], ref['losses'][e])
    _assert_same_evals(ref['evals'][2:], res['evals'])
    _assert_same_params_and_adam(ref, res)
    assert res['seeds'] == ref['seeds']
    assert all(np.array_equal(a, b) for a, b in zip(res['numpy'], ref['numpy']))
    assert torch.equal(res['torch'], ref['torch'])
    if key == 'ncl':
        # the restored model counts as clustered: it re-clusters only where the restored flag counter says so
        assert res['clusters'] == [e for e in ref['clusters'] if e >= 2]
        assert res['clusters'] == ([2] if hp['epoch_period'] == 3 else [3])      # on a re-cluster / between two
    if key == 'lightgcl':
        assert res['model'].ut is not None


def test_early_stop_resumes_inside_the_waiting_period(tmp_path, monkeypatch):
    from sslrec_b200.trainer import Trainer
    monkeypatch.chdir(tmp_path)
    kept = {}                                   # epoch -> (copy of that epoch's checkpoint, early-stop counter)
    save = Trainer.save_checkpoint

    def save_and_keep(self, model, path):
        save(self, model, path)
        kept[self.epoch_done] = (f'{path}.{self.epoch_done}', self.early_stop_state['waited'])
        shutil.copy(path, kept[self.epoch_done][0])
        return path

    monkeypatch.setattr(Trainer, 'save_checkpoint', save_and_keep)
    train = dict(deterministic=True, epoch=12, patience=2, checkpoint_step=1)
    ref = _train('simgcl', {}, train)
    monkeypatch.setattr(Trainer, 'save_checkpoint', save)
    last = max(ref['losses'])
    waiting = [e for e, (_, w) in sorted(kept.items()) if 0 < w < 2 and e < last]
    assert waiting, ('no epoch inside a waiting period', {e: w for e, (_, w) in kept.items()})
    _scramble()
    res = _train('simgcl', {}, dict(train, resume_path=kept[waiting[0]][0]), seed_globals=False)
    assert sorted(res['losses']) == list(range(waiting[0] + 1, last + 1))
    ref_es, res_es = ref['trainer'].early_stop_state, res['trainer'].early_stop_state
    assert res_es['best_epoch'] == ref_es['best_epoch'] and res_es['waited'] == ref_es['waited']
    for n in ref['params']:                    # the rebuilt best model
        assert torch.equal(ref['params'][n], res['params'][n]), n
    _assert_same_evals(ref['evals'][-2:], res['evals'][-2:])      # the best model's validation, then its test metrics


@pytest.mark.parametrize('loader', ['host', 'device'])
@pytest.mark.parametrize('key', ['sgl', 'hccf'])
def test_default_mode_resumes_the_same_batches_and_seeds(tmp_path, monkeypatch, key, loader):
    monkeypatch.chdir(tmp_path)
    base = dict(device_loader=loader == 'device')
    ref = _train(key, {}, dict(base, epoch=4), record_steps=True)
    _train(key, {}, dict(base, epoch=2, checkpoint_step=1))
    _scramble()
    res = _train(key, {}, dict(base, epoch=4, resume_path=str(_checkpoint(tmp_path, key))), seed_globals=False, record_steps=True)
    per_epoch = len(ref['steps']) // 4
    assert per_epoch >= 3 and len(res['steps']) == 2 * per_epoch
    for k, ((b_ref, s_ref), (b_res, s_res)) in enumerate(zip(ref['steps'][2 * per_epoch:], res['steps'])):
        assert s_ref == s_res, k
        for x, y in zip(b_ref, b_res):
            assert torch.equal(x, y), k
    assert res['seeds'] == ref['seeds']
    for e in (2, 3):
        (la, da), (lb, db) = ref['losses'][e], res['losses'][e]
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)), (e, la, lb)
        for t in da:
            assert abs(da[t] - db[t]) <= 1e-5 * max(1.0, abs(da[t])), (e, t, da[t], db[t])


def test_changed_loader_kind_is_refused(tmp_path):
    m, tr, _ = make_run('lightgcn', device='cuda')
    path = str(tmp_path / 'resume.pth')
    tr.save_checkpoint(m, path)
    m2, tr2, _ = make_run('lightgcn', device='cuda', train=dict(device_loader=True))
    with pytest.raises(ValueError, match="loader: saved 'host', now 'device'"):
        tr2.load_checkpoint(m2, path)
