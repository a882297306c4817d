"""Training checkpoints without a GPU: what ``Trainer.load_checkpoint`` refuses (another model, another model or optimizer section,
batch size, train.deterministic, multi-GPU), the atomic write (a ``torch.save`` that fails halfway leaves the previous checkpoint
loadable), the loaders it cannot resume (torch's DataLoader), and a round trip of the host-side state: parameters, seed stream,
numpy's and torch's generators, NCL's flag counter and the trainer's position."""
import importlib
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import inputs

HP = {
    'lightgcn': dict(keep_rate=0.8),
    'simgcl': dict(cl_weight=1e-2, temperature=0.2, eps=0.2),
    'sgl': dict(augmentation='edge_drop', keep_rate=0.8, cl_weight=1e-2, temperature=0.2),
    'sgl_nd': dict(augmentation='node_drop', keep_rate=0.8, cl_weight=1e-2, temperature=0.2),
    'ncl': dict(proto_weight=1e-4, struct_weight=1e-3, temperature=0.1, high_order=1, cluster_num=5, epoch_period=2),
    'hccf': dict(keep_rate=0.8, cl_weight=1e-2, temperature=0.2, hyper_num=16, mult=1.0, leaky=0.5),
    'lightgcl': dict(temp=0.2, dropout=0.1, cl_weight=1e-2, svd_q=5),
    'directau': dict(gamma=2.0),
}


def make_run(key, device='cpu', train=None, model=None, test=None, seed_globals=True):
    """A data handler, model and trainer (optimizer created) for ``key`` (a model name, ``sgl_nd`` = SGL with node drop) on the
    'tiny' graph with a random validation / test split.  ``seed_globals``: seed numpy and torch from train.seed (init_seed), as
    a fresh run does."""
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import DataHandlerGeneralCF
    from sslrec_b200.trainer import Trainer, init_seed
    name = key.split('_')[0]
    cfg = default_config(name, layer_num=2, embedding_size=32, reg_weight=1e-6, **HP[key])
    cfg['model'].update(model or {})
    cfg['train'].update(batch_size=128, epoch=2, test_step=1, loss='pairwise_with_epoch_flag' if name == 'ncl' else 'pairwise')
    cfg['train'].update(train or {})
    cfg['optimizer']['lr'] = 1e-2
    cfg['test'].update(k=[5, 10], batch_size=32)
    cfg['test'].update(test or {})
    load_config(base=cfg, device=device)
    if seed_globals:
        init_seed()
    case = inputs.make_case('tiny')
    U, I = case['n_user'], case['n_item']
    trn = sp.coo_matrix((np.ones(len(case['rows']), dtype=np.float32), (case['rows'], case['cols'])), shape=(U, I))
    rs = np.random.RandomState(0)
    val = sp.coo_matrix((np.ones(200), (rs.randint(0, U, 200), rs.randint(0, I, 200))), shape=(U, I))
    dh = DataHandlerGeneralCF(trn, val, val)
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + name)
    m = [getattr(mod, a) for a in dir(mod) if a.lower() == name][0](dh).to(device)
    tr = Trainer(dh)
    tr.create_optimizer(m)
    return m, tr, dh


def _save(tmp_path, key='lightgcn', **kw):
    m, tr, dh = make_run(key, **kw)
    path = str(tmp_path / 'resume.pth')
    tr.save_checkpoint(m, path)
    return path, m, tr


def test_round_trip_of_host_state(tmp_path):
    from sslrec_b200.data_handler import HostBatchLoader
    path, m, tr = _save(tmp_path, 'ncl')
    loader = tr.data_handler.train_dataloader
    assert isinstance(loader, HostBatchLoader)
    for _ in range(3):
        m._seeds.next()
    loader.dataset.epoch_flag_counter = 7
    tr.epoch_done = 4
    with torch.no_grad():
        m.user_embeds.mul_(2)
    tr.save_checkpoint(m, path)
    want = (dict(m.state_dict()), m._seeds.state, m._seeds.count, np.random.get_state()[1].copy(), torch.get_rng_state())
    saved = {k: v.clone() for k, v in want[0].items()}

    m2, tr2, _ = make_run('ncl', seed_globals=False)
    np.random.seed(11)
    torch.manual_seed(11)
    assert tr2.load_checkpoint(m2, path) == 5
    for k, v in m2.state_dict().items():
        assert torch.equal(v, saved[k]), k
    assert (m2._seeds.state, m2._seeds.count) == (want[1], want[2])
    assert np.array_equal(np.random.get_state()[1], want[3]) and torch.equal(torch.get_rng_state(), want[4])
    assert tr2.data_handler.train_dataloader.dataset.epoch_flag_counter == 7
    assert not hasattr(m2, 'user2cluster')                   # saved before the first clustering: the first step clusters
    ck = torch.load(path, weights_only=True)                 # plain data: loads without unpickling code
    assert all(t.device.type == 'cpu' for t in ck['model'].values())
    assert type(ck['model_resume']['seeds']['state']) is int


def test_another_model_is_refused(tmp_path):
    path, _, _ = _save(tmp_path, 'simgcl')
    m, tr, _ = make_run('sgl')
    with pytest.raises(ValueError, match='another run.*model: saved .simgcl., now .sgl.'):
        tr.load_checkpoint(m, path)


@pytest.mark.parametrize('section,change,what', [
    ('model', dict(embedding_size=16), 'embedding_size saved 32, now 16'),
    ('train', dict(batch_size=64), 'batch_size: saved 128, now 64'),
    ('train', dict(deterministic=True), 'deterministic: saved False, now True'),
    ('train', dict(seed=7), 'seed: saved 2023, now 7'),
    ('optimizer', dict(weight_decay=1e-4), 'weight_decay saved 0, now 0.0001'),
])
def test_changed_settings_are_refused(tmp_path, section, change, what):
    path, _, _ = _save(tmp_path)
    kw = {'train': change} if section == 'train' else {'model': change} if section == 'model' else {}
    m, tr, _ = make_run('lightgcn', **kw)
    if section == 'optimizer':
        from sslrec_b200.config import configs
        configs['optimizer'].update(change)
    with pytest.raises(ValueError, match=what):
        tr.load_checkpoint(m, path)


def test_extended_run_is_accepted(tmp_path):
    """train.epoch, patience, test_step and the test section may change between the runs."""
    path, _, _ = _save(tmp_path)
    m, tr, _ = make_run('lightgcn', train=dict(epoch=9, patience=3, test_step=2), test=dict(k=[20], metrics=['ndcg']))
    assert tr.load_checkpoint(m, path) == 0


def test_multi_gpu_is_refused_both_ways(tmp_path):
    from sslrec_b200.trainer import Trainer
    path, m, tr = _save(tmp_path)
    sharded = Trainer(tr.data_handler, grad_sync=object())
    sharded.optimizer = tr.optimizer
    for call in (sharded.save_checkpoint, sharded.load_checkpoint):
        with pytest.raises(RuntimeError, match='single-GPU'):
            call(m, path)
    m.shard_to(types.SimpleNamespace(shard_propagation=False))
    for call in (tr.save_checkpoint, tr.load_checkpoint):
        with pytest.raises(RuntimeError, match='single-GPU'):
            call(m, path)


def test_failed_write_leaves_the_previous_checkpoint(tmp_path, monkeypatch):
    path, m, tr = _save(tmp_path)
    before = open(path, 'rb').read()
    real_save = torch.save

    def save_half(obj, f, *a, **kw):
        real_save(obj, f, *a, **kw)
        f.seek(0)
        f.truncate(f.tell() + 100)
        raise OSError('disk full')

    saved = m.user_embeds.detach().clone()
    with torch.no_grad():
        m.user_embeds.add_(1)
    monkeypatch.setattr(torch, 'save', save_half)
    with pytest.raises(OSError, match='disk full'):
        tr.save_checkpoint(m, path)
    monkeypatch.undo()
    assert open(path, 'rb').read() == before
    assert os.listdir(tmp_path) == ['resume.pth']           # no temporary file left behind
    m2, tr2, _ = make_run('lightgcn')
    tr2.load_checkpoint(m2, path)
    assert torch.equal(m2.user_embeds, saved)


def test_torch_dataloader_cannot_checkpoint(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    m, tr, _ = make_run('lightgcn', train=dict(torch_dataloader=True, checkpoint_step=1))
    with pytest.raises(RuntimeError, match='DataLoader does not expose its iterator state'):
        tr.train(m)
    with pytest.raises(RuntimeError, match='DataLoader does not expose its iterator state'):
        tr.save_checkpoint(m, str(tmp_path / 'x.pth'))
    assert not os.path.exists(tmp_path / 'checkpoint')


def test_checkpoint_path_follows_save_model():
    from sslrec_b200.config import configs
    m, tr, _ = make_run('lightgcn')
    assert tr.checkpoint_path() == './checkpoint/lightgcn/lightgcn-synthetic-resume.pth'
    configs['tune'] = {'enable': True, 'now_para_str': 'x'}
    assert tr.checkpoint_path() == './checkpoint/lightgcn/tune/lightgcn-synthetic-resume.pth'
