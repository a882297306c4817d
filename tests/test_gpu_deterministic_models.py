"""train.deterministic for all seven models: a training step is a pure function of (parameters, optimizer state, batch, seeds).
On batches with deliberately repeated users and items and FusedAdam at lr 1e-2 (which amplifies any last-bit difference):
two fresh runs give bit-identical losses, parameters and NCL clusterings; a GraphedStep replay equals the eager loop bit for
bit (HCCF: the eager loop on the graph-safe path of ``GraphedStep.eager``); step 0 stays within the golden tolerances; two
Trainer runs (epochs + evaluate, host and device loader) give identical epoch losses and metrics; the multi-GPU combinations raise."""
import types

import numpy as np
import pytest
import torch

from oracle import inputs, replay
import ssl_test_helpers as H
from test_gpu_models import CASES as GOLDEN_CASES, _run

pytestmark = pytest.mark.gpu

CASES = [('lightgcn', 'tiny'), ('lightgcn', 'small'), ('simgcl', 'tiny'), ('simgcl', 'small'), ('sgl', 'tiny'), ('sgl_nd', 'tiny'),
         ('ncl', 'tiny'), ('ncl_k50', 'small'), ('hccf', 'tiny'), ('hccf_h128', 'small'), ('lightgcl', 'tiny'), ('lightgcl', 'small'),
         ('directau', 'tiny'), ('directau', 'small')]
FLAGGED = {0, 3}             # NCL: re-cluster on the first batch and on a later one


@pytest.fixture
def E():
    from sslrec_b200 import engine
    engine.DETERMINISTIC = True
    yield engine
    engine.DETERMINISTIC = None


def _model(key, size):
    g = replay.load_golden(key, size)
    case = inputs.make_case(size)
    torch.manual_seed(0)                    # same parameter init, and the same generator for k-means / svd_lowrank, in every run
    np.random.seed(0)
    model, dh = H.make_model(key, case, g['hp'])
    model.load_state_dict({'user_embeds': case['user_e'], 'item_embeds': case['item_e']}, strict=False)
    return model, case


def _batches(case, ncl, n=6):
    """Half of every batch drawn from three training pairs and a handful of negatives: users and items repeat many times."""
    rs = np.random.RandomState(5)
    B, n_edges = case['batch'], len(case['rows'])
    out = []
    for k in range(n):
        pick = np.where(rs.rand(B) < 0.5, rs.randint(0, min(3, n_edges), size=B), rs.randint(0, n_edges, size=B))
        negs = np.where(rs.rand(B) < 0.5, rs.randint(0, min(4, case['n_item']), size=B), rs.randint(0, case['n_item'], size=B))
        b = [torch.from_numpy(np.asarray(a)).long().cuda() for a in (case['rows'][pick], case['cols'][pick], negs)]
        if ncl:
            f = torch.zeros(B, dtype=torch.int64)
            f[0] = int(k in FLAGGED)
            b.append(f.cuda())
        out.append(b)
    return out


def _train(key, size, graphed):
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    name = key.split('_')[0]
    ncl = name == 'ncl'
    model, case = _model(key, size)
    batches = _batches(case, ncl)
    opt = FusedAdam(model.parameters(), lr=1e-2)
    losses = []
    if graphed:
        step = GraphedStep(model, opt, batches[0], warmup=2, recluster=0 in FLAGGED)
        losses += [None, None]
        for k, b in enumerate(batches[1:], start=1):
            loss, parts = step(b, recluster=k in FLAGGED)
            losses.append((loss.clone(), {k_: torch.as_tensor(v, device='cuda').clone() for k_, v in parts.items()}))
        step.close()
    else:
        model._graph_mode = name == 'hccf'         # the path GraphedStep takes (and GraphedStep.eager)
        for b in [batches[0]] * 2 + batches[1:]:
            opt.zero_grad()
            loss, parts = model.cal_loss(b)
            loss.backward()
            opt.step()
            losses.append((loss.detach().clone(), {k_: torch.as_tensor(v, device='cuda').detach().clone() for k_, v in parts.items()}))
        model._graph_mode = False
    torch.cuda.synchronize()
    params = {n: p.detach().clone() for n, p in model.named_parameters()}
    clusters = (model.user2cluster.clone(), model.item2cluster.clone()) if ncl else None
    return losses, params, clusters


def _assert_same(a, b, what, first=0):
    for k, (x, y) in enumerate(zip(a[0][first:], b[0][first:])):
        assert torch.equal(x[0], y[0]), (what, 'loss', k, x[0].item(), y[0].item())
        for t in x[1]:
            assert torch.equal(x[1][t], y[1][t]), (what, t, k)
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), (what, n, (a[1][n] - b[1][n]).abs().max().item())
    if a[2] is not None:
        assert torch.equal(a[2][0], b[2][0]) and torch.equal(a[2][1], b[2][1]), (what, 'clusters')


@pytest.mark.parametrize('key,size', CASES)
def test_two_runs_and_graph_replay_are_bit_identical(E, key, size):
    first, second = _train(key, size, False), _train(key, size, False)
    assert len(first[0]) >= 5
    _assert_same(first, second, 'eager run 2')
    _assert_same(_train(key, size, True), first, 'graph replay', first=2)


@pytest.mark.parametrize('model_key,case_name', GOLDEN_CASES)
def test_step0_within_golden_tolerances(E, model_key, case_name):
    g, case, model, batch = _run(model_key, case_name)
    loss, parts = model.cal_loss(batch)
    loss.backward()
    H.golden_loss_grads_close(g, loss, parts, model.named_parameters(), 'deterministic ')


def _trainer_run(name, loader):
    import importlib
    import scipy.sparse as sp
    from sslrec_b200.config import default_config, load_config
    from sslrec_b200.data_handler import DataHandlerGeneralCF
    from sslrec_b200.trainer import Trainer, init_seed
    case = inputs.make_case('small')
    hp = dict(layer_num=2, embedding_size=32, reg_weight=1e-6, keep_rate=0.8, cl_weight=1e-2, temperature=0.2, eps=0.2, hyper_num=32,
              mult=1.0, leaky=0.5)
    cfg = default_config(name, **hp)
    cfg['train'].update(batch_size=1024, epoch=2, loss='pairwise', deterministic=True, device_loader=loader == 'device')
    cfg['optimizer']['lr'] = 1e-2
    cfg['test']['batch_size'] = 256
    load_config(base=cfg, device='cuda')
    init_seed()
    U, I = case['n_user'], case['n_item']
    trn = sp.coo_matrix((np.ones(len(case['rows']), dtype=np.float32), (case['rows'], case['cols'])), shape=(U, I))
    rs = np.random.RandomState(0)
    val = sp.coo_matrix((np.ones(400), (rs.randint(0, U, 400), rs.randint(0, I, 400))), shape=(U, I))
    dh = DataHandlerGeneralCF(trn, val, val)
    dh.load_data()
    mod = importlib.import_module('sslrec_b200.general_cf.' + name)
    model = [getattr(mod, a) for a in dir(mod) if a.lower() == name][0](dh).cuda()
    tr = Trainer(dh)
    tr.create_optimizer(model)
    losses = [tr.train_epoch(model, e) for e in range(2)]
    return losses, tr.evaluate(model)


@pytest.mark.parametrize('loader', ['host', 'device'])
@pytest.mark.parametrize('name', ['simgcl', 'hccf'])
def test_trainer_runs_with_the_key_are_identical(name, loader):
    from sslrec_b200 import engine
    assert engine.DETERMINISTIC is None                    # the config key alone decides
    a, b = _trainer_run(name, loader), _trainer_run(name, loader)
    for (la, da), (lb, db) in zip(a[0], b[0]):
        assert la == lb and da == db, (la, lb)
    for m in a[1]:
        assert np.array_equal(a[1][m], b[1][m]), m


def test_multi_gpu_combinations_raise(E):
    from sslrec_b200.parallel import RowShard
    from sslrec_b200.trainer import Trainer
    model, _ = _model('lightgcn', 'tiny')
    with pytest.raises(RuntimeError, match='single-GPU'):
        RowShard(None, 0, 2, 100)
    with pytest.raises(RuntimeError, match='single-GPU'):
        model.shard_to(types.SimpleNamespace(shard_propagation=False))
    tr = Trainer(types.SimpleNamespace(train_dataloader=None), grad_sync=object())
    with pytest.raises(RuntimeError, match='single-GPU'):
        tr.train_epoch(model, 0)
