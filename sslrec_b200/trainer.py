"""Trainer -- mirror of the base ``Trainer`` of trainer/trainer.py:39-162 for the surface the hot
path needs: ``create_optimizer`` (Adam only, :45-49; here the fused kernel), ``train_epoch`` (:51-84,
same loop: sample_negs, zero_grad, cal_loss, loss.item(), backward, step, per-term float()) and
``evaluate`` (:139-152 + metrics.py:82-127 with the native top-k)."""
from __future__ import annotations

import os
import tempfile
import time
from copy import deepcopy

import numpy as np
import torch

from . import engine as E
from ._lib import check, lib
from .config import configs
from .optim import FusedAdam

# Trainer.evaluate ranks with model.predict_topk (no [Bt, I] score matrix) from this many items on, below it with full_predict + topk; both
# give the same ids.  On an H100 80GB HBM3 (400 W and 700 W, profiles/r06_predict_topk.md) the fused call runs at 0.55-0.91x the pair's
# speed at 19 747-83 761 items and 1.3-1.5x it at 1 000 000 items (256- and 1024-user batches); the crossover in between is not measured.
FUSED_TOPK_MIN_ITEMS = 1_000_000


def init_seed():
    """trainer/trainer.py:26-36."""
    t = configs.get('train', {})
    if t.get('reproducible', False):
        seed = t['seed']
        np.random.seed(seed)
        torch.manual_seed(seed)
        if torch.cuda.is_available():
            torch.cuda.manual_seed_all(seed)


def _summary_writer():
    """The optional TensorBoard writer of trainer.py:20-23 (``train.tensorboard: true`` -> SummaryWriter('runs')); None otherwise."""
    if not configs.get('train', {}).get('tensorboard', False):
        return None
    from torch.utils.tensorboard import SummaryWriter
    return SummaryWriter(log_dir='runs')


CHECKPOINT_FORMAT = 1         # version of the dict Trainer.save_checkpoint writes


def _to_cpu(obj):
    """A copy of a nest of dicts / lists / tuples with every tensor moved to the CPU."""
    if isinstance(obj, torch.Tensor):
        return obj.detach().cpu()
    if isinstance(obj, dict):
        return {k: _to_cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to_cpu(v) for v in obj)
    return obj


def _numpy_rng_state() -> dict:
    """numpy's global generator as plain values and one tensor, so the checkpoint loads with ``weights_only=True``."""
    s = np.random.get_state(legacy=False)
    return {'bit_generator': s['bit_generator'], 'key': torch.from_numpy(s['state']['key'].astype(np.int64)), 'pos': int(s['state']['pos']),
            'has_gauss': int(s['has_gauss']), 'gauss': float(s['gauss'])}


def _set_numpy_rng_state(s: dict) -> None:
    np.random.set_state({'bit_generator': s['bit_generator'], 'state': {'key': s['key'].numpy().astype(np.uint32), 'pos': s['pos']},
                         'has_gauss': s['has_gauss'], 'gauss': s['gauss']})


def _atomic_save(obj, path: str) -> None:
    """torch.save to a temporary file in the target's directory, flushed and fsync'ed, then renamed over ``path``: readers see the
    old file or the new one, never a partial write."""
    directory = os.path.dirname(os.path.abspath(path))
    os.makedirs(directory, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix='.' + os.path.basename(path) + '.', suffix='.tmp', dir=directory)
    try:
        with os.fdopen(fd, 'wb') as f:
            torch.save(obj, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    dfd = os.open(directory, os.O_RDONLY)          # the rename itself survives a crash once the directory is on disk
    try:
        os.fsync(dfd)
    finally:
        os.close(dfd)


def _describe_difference(key, saved, now) -> str:
    if isinstance(saved, dict) and isinstance(now, dict):
        keys = sorted((k for k in saved.keys() | now.keys() if saved.get(k) != now.get(k)), key=str)
        return '{}: {}'.format(key, ', '.join(f'{k} saved {saved.get(k)!r}, now {now.get(k)!r}' for k in keys))
    return f'{key}: saved {saved!r}, now {now!r}'


class Trainer(object):
    def __init__(self, data_handler, logger=None, grad_sync=None):
        self.data_handler = data_handler
        self.logger = logger
        self.grad_sync = grad_sync     # parallel.BatchShard: data-parallel ranks average gradients before the step
        if grad_sync is not None:
            E.NegSpec.from_config().refuse_multi_gpu(sharded=False)
        self._graphed = None           # graphed.GraphedStep when train.cuda_graph is set
        self._writer = None            # created on first use: the scalars 'Loss/train' and 'HR/test' of trainer.py:78,144
        self.epoch_done = -1           # the last epoch train_epoch finished (a training checkpoint resumes after it)
        self.early_stop_state = None   # train() with patience: {'waited', 'best_epoch', 'best_metric', 'best_state'}

    def _scalar(self, tag, value, step):
        if self._writer is None and configs.get('train', {}).get('tensorboard', False):
            self._writer = _summary_writer()
        if self._writer is not None:
            self._writer.add_scalar(tag, value, step)

    def create_optimizer(self, model):
        optim_config = configs['optimizer']
        if optim_config['name'] == 'adam':
            self.optimizer = FusedAdam(model.parameters(), lr=optim_config['lr'], weight_decay=optim_config['weight_decay'])
        else:
            raise NotImplementedError("only 'adam' is supported (trainer.py:47)")

    def train_epoch(self, model, epoch_idx):
        """Same loop and same logged numbers as trainer.py:51-84.  The reference reads ``loss.item()`` and
        ``float(v)`` for every loss term right after ``cal_loss`` (:66, :72), i.e. 1 + n_terms blocking device
        syncs per step; here the step's scalars are copied device->pinned host asynchronously and summed when
        the copy has landed (one step later), so the host keeps enqueueing while the GPU works."""
        if self.grad_sync is not None and E.deterministic():
            raise RuntimeError('train.deterministic is single-GPU: the gradient all-reduce of grad_sync sums in an order of its own')
        train_dataloader = self.data_handler.train_dataloader
        train_dataloader.dataset.sample_negs()
        if hasattr(train_dataloader.sampler, 'set_epoch'):
            train_dataloader.sampler.set_epoch(epoch_idx)
        loss_log_dict = {}
        ep_loss = 0
        model.train()
        reader = LossReader(configs['device'])
        use_graph = bool(configs['train'].get('cuda_graph', False))       # optional key: replay the step as ONE CUDA graph launch
        if use_graph and self.grad_sync is not None:
            raise RuntimeError('train.cuda_graph captures a single-GPU step (no gradient exchange inside)')
        for _, tem in enumerate(train_dataloader):
            recluster = _recluster_flag(train_dataloader, tem) if use_graph else False
            batch_data = list(map(lambda x: x.long().to(configs['device'], non_blocking=True), tem))
            if use_graph:
                loss, loss_dict = self._graph_step(model, batch_data, recluster)
            else:
                self.optimizer.zero_grad()
                loss, loss_dict = model.cal_loss(batch_data)
                loss.backward()
                if self.grad_sync is not None:
                    self.grad_sync.average_gradients(model.parameters())
                self.optimizer.step()
            for done in reader.push(loss, loss_dict):
                ep_loss += done[0]
                for loss_name, val in done[1].items():
                    loss_log_dict[loss_name] = loss_log_dict.get(loss_name, 0.0) + val / len(train_dataloader)
        for done in reader.flush():
            ep_loss += done[0]
            for loss_name, val in done[1].items():
                loss_log_dict[loss_name] = loss_log_dict.get(loss_name, 0.0) + val / len(train_dataloader)
        steps = len(train_dataloader.dataset) // configs['train']['batch_size']                   # trainer.py:60,78
        self._scalar('Loss/train', ep_loss / max(steps, 1), epoch_idx)
        if self.logger is not None:
            self.logger.log_loss(epoch_idx, loss_log_dict, save_to_log=configs['train'].get('log_loss', True))
        self.epoch_done = epoch_idx
        return ep_loss, loss_log_dict

    def _graph_step(self, model, batch_data, recluster=False):
        """The step through graphed.GraphedStep: the first full-size batch is stepped eagerly (that is the capture's warm-up -- every
        batch is trained on exactly once, like the eager loop) and captured; later full-size batches replay the graph; a batch of
        another size (the epoch's last) runs eagerly with the same device-resident seeds.  ``recluster``: the batch carries NCL's
        k-means flag (decided on the host), so the model re-clusters before the step, outside the graph."""
        from .graphed import GraphedStep
        g = self._graphed
        if g is not None and g.model is not model:
            g.close()
            g = self._graphed = None
        if g is None:
            g = self._graphed = GraphedStep(model, self.optimizer, batch_data, warmup=1, recluster=recluster)
            return g.warm_result
        if all(a.shape == b.shape for a, b in zip(batch_data, g.static_batch)):
            return g(batch_data, recluster=recluster)
        return g.eager(batch_data, recluster=recluster)

    def train(self, model):
        """trainer.py:86-137: plain run (evaluate every ``test_step`` epochs, then test + save) or, when the YAML
        carries ``patience`` (configurator sets ``early_stop``), tracking of the best first-metric@k[0] with the
        best ``state_dict`` restored into a freshly built model before the final evaluate / test / save.

        Optional keys (single GPU): ``train.checkpoint_step: n`` writes a training checkpoint (``save_checkpoint``) to
        ``checkpoint_path()`` after every n-th epoch; ``train.resume_path: path`` loads one (``load_checkpoint``) and continues at
        the epoch after it, with the early-stop counters and best state it holds."""
        self.create_optimizer(model)
        cfg = configs['train']
        start, self.early_stop_state = 0, None
        if cfg.get('resume_path'):
            start = self.load_checkpoint(model, cfg['resume_path'])
        if cfg.get('checkpoint_step'):
            self._single_gpu(model, 'train.checkpoint_step')       # refused now rather than at the first checkpoint
            self._train_loader('train.checkpoint_step')
        if not cfg.get('early_stop', False):
            for epoch_idx in range(start, cfg['epoch']):
                self.train_epoch(model, epoch_idx)
                if epoch_idx % cfg['test_step'] == 0:
                    self.evaluate(model, epoch_idx)
                self._checkpoint_after(model, epoch_idx)
            self.test(model)
            self.save_model(model)
            return model
        key = configs['test']['metrics'][0]
        es = self.early_stop_state = self.early_stop_state or {'waited': 0, 'best_epoch': 0, 'best_metric': -1e9, 'best_state': None}
        for epoch_idx in range(start, cfg['epoch']):
            if es['waited'] >= cfg['patience']:           # resumed from the checkpoint of the epoch that stopped the run
                break
            self.train_epoch(model, epoch_idx)
            if epoch_idx % cfg['test_step'] == 0:
                score = self.evaluate(model, epoch_idx)[key][0]
                if score > es['best_metric']:
                    es.update(waited=0, best_epoch=epoch_idx, best_metric=score, best_state=deepcopy(model.state_dict()))
                    self._log('Validation score increased.  Copying the best model ...')
                else:
                    es['waited'] += 1
                    self._log(f"Early stop counter: {es['waited']} out of {cfg['patience']}")
            self._checkpoint_after(model, epoch_idx)
            if es['waited'] >= cfg['patience']:
                break
        self._log('Best Epoch {}'.format(es['best_epoch']))
        if es['best_state'] is not None:
            model = self._rebuild(model, es['best_state'])
        self.evaluate(model)
        self.test(model)
        self.save_model(model)
        return model

    def _log(self, msg):
        if self.logger is not None:
            self.logger.log(msg)

    def _rebuild(self, model, state_dict):
        """The reference re-creates the model with build_model(data_handler) and loads the best parameters
        (trainer.py:129-131); here the same class is re-instantiated on the same data handler."""
        fresh = type(model)(self.data_handler).to(configs['device'])
        fresh.comm = getattr(model, 'comm', None)
        fresh.load_state_dict(state_dict)
        return fresh

    def test(self, model):
        """trainer.py:152-160: metrics on the test split."""
        if not hasattr(self.data_handler, 'test_dataloader'):
            raise NotImplementedError('data handler has no test_dataloader')
        self._in_test = True                 # the reference's test() writes no TensorBoard scalar (trainer.py:152-160)
        try:
            return self.evaluate(model, loader=self.data_handler.test_dataloader, data_type='Test set')
        finally:
            self._in_test = False

    def save_model(self, model):
        """trainer.py:162-186: ./checkpoint/{model}/{model}-{data}-{timestamp}.pth (tune runs: ./checkpoint/{model}/tune/
        {model}-{data}-{now_para_str}.pth) when train.save_model is set.  Returns the path or None."""
        if not configs['train'].get('save_model', False):
            return None
        model_name, data_name = configs['model']['name'], configs['data']['name']
        tune = configs.get('tune', {}).get('enable', False)
        save_dir = './checkpoint/{}{}'.format(model_name, '/tune' if tune else '')
        os.makedirs(save_dir, exist_ok=True)
        tag = configs['tune']['now_para_str'] if tune else int(time.time())
        path = '{}/{}-{}-{}.pth'.format(save_dir, model_name, data_name, tag)
        torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, path)
        self._log('Save model parameters to {}'.format(path))
        return path

    def load_model(self, model):
        """trainer.py:188-196."""
        if 'pretrain_path' not in configs['train']:
            raise KeyError("No pretrain_path in configs['train']")
        path = configs['train']['pretrain_path']
        model.load_state_dict(torch.load(path, map_location=configs['device']))
        self._log('Load model parameters from {}'.format(path))
        return model

    # ---- training checkpoints: everything a run needs to continue as if it had never stopped ---------------------------
    def checkpoint_path(self) -> str:
        """./checkpoint/{model}/{model}-{data}-resume.pth (tune runs: ./checkpoint/{model}/tune/...), the directory of save_model."""
        model_name, data_name = configs['model']['name'], configs['data']['name']
        tune = configs.get('tune', {}).get('enable', False)
        return './checkpoint/{}{}/{}-{}-resume.pth'.format(model_name, '/tune' if tune else '', model_name, data_name)

    def _checkpoint_after(self, model, epoch_idx):
        n = configs['train'].get('checkpoint_step')
        if n and (epoch_idx + 1) % n == 0:
            path = self.save_checkpoint(model, self.checkpoint_path())
            self._log('Save training checkpoint to {}'.format(path))

    def _single_gpu(self, model, what):
        if self.grad_sync is not None or getattr(model, 'comm', None) is not None:
            raise RuntimeError(f'{what}: training checkpoints are single-GPU (a multi-GPU run shards its optimizer and table state)')

    def _train_loader(self, what):
        """-> (kind, loader) for the train loaders whose position a checkpoint can hold."""
        from .data_handler import DeviceLoader, HostBatchLoader
        loader = self.data_handler.train_dataloader
        if isinstance(loader, HostBatchLoader):
            return 'host', loader
        if isinstance(loader, DeviceLoader):
            return 'device', loader
        raise RuntimeError(f'{what}: the train loader {type(loader).__name__} does not expose its iterator state, so a resumed run '
                           'would train on other batches; use the default HostBatchLoader (no train.torch_dataloader) or train.device_loader')

    def _resume_record(self, model, kind):
        """What a checkpoint must agree on with the run that loads it.  train.epoch, patience, test_step and the test section may
        differ (a run can be extended)."""
        t = configs['train']
        record = {'model': configs['model']['name'], 'data': configs['data']['name'], 'user_num': int(model.user_num),
                  'item_num': int(model.item_num), 'model_config': deepcopy(configs['model']), 'optimizer_config': deepcopy(configs['optimizer']),
                  'batch_size': t['batch_size'], 'seed': t.get('seed'), 'loader': kind, 'deterministic': E.deterministic()}
        record.update(E.NegSpec.from_config().record())
        return record

    def save_checkpoint(self, model, path):
        """Write a training checkpoint at an epoch boundary: parameters, the model's other training state (``resume_state``), the
        optimizer with its step count, the kernel seed stream, numpy's, torch's and CUDA's global generators, the train loader's
        position, the last finished epoch, the early-stop state and a record of the run it belongs to.  Every tensor is stored on
        the CPU.  The file is replaced atomically: a crash while writing leaves the previous checkpoint intact.  Returns ``path``."""
        self._single_gpu(model, 'save_checkpoint')
        kind, loader = self._train_loader('save_checkpoint')
        g = self._graphed
        if g is not None and g._primed:
            # the seeds of the graph's first replay are drawn but unused; a resumed run could not draw them again, so this run
            # drops them too and captures afresh at its next step, as the resumed run does
            g.close()
            self._graphed = None
        self.optimizer.sync_host_step()
        es = self.early_stop_state
        ckpt = {
            'format': CHECKPOINT_FORMAT,
            'record': self._resume_record(model, kind),
            'model': _to_cpu(model.state_dict()),
            'model_resume': _to_cpu(model.resume_state()),
            'optimizer': _to_cpu(self.optimizer.state_dict()),
            'rng': {'numpy': _numpy_rng_state(), 'torch': torch.get_rng_state(), 'cuda': [s.cpu() for s in torch.cuda.get_rng_state_all()]},
            'loader': loader.state(),
            'trainer': {'epoch': int(self.epoch_done),
                        'early_stop': None if es is None else {'waited': int(es['waited']), 'best_epoch': int(es['best_epoch']),
                                                              'best_metric': float(es['best_metric']),
                                                              'best_state': _to_cpu(es['best_state'])}},
        }
        _atomic_save(ckpt, path)
        return path

    def load_checkpoint(self, model, path) -> int:
        """Restore a ``save_checkpoint`` file into ``model``, this trainer's optimizer (created if missing), the generators and the
        train loader.  Raises when the checkpoint belongs to another run (model, data, sizes, the model and optimizer sections,
        batch size, seed, loader kind, train.deterministic) or to a multi-GPU one.  Returns the epoch to continue at."""
        self._single_gpu(model, 'load_checkpoint')
        kind, loader = self._train_loader('load_checkpoint')
        ckpt = torch.load(path, map_location='cpu', weights_only=True)
        if not isinstance(ckpt, dict) or ckpt.get('format') != CHECKPOINT_FORMAT:
            raise ValueError(f'{path}: not a training checkpoint of format {CHECKPOINT_FORMAT} (save_checkpoint writes one)')
        saved, now = ckpt['record'], self._resume_record(model, kind)
        diff = [_describe_difference(k, saved.get(k), now.get(k)) for k in list(now) + [k for k in saved if k not in now]
                if saved.get(k) != now.get(k)]
        if diff:
            raise ValueError(f'{path}: the checkpoint belongs to another run: ' + '; '.join(diff))
        if self._graphed is not None:                  # captured around the old state: the next step captures afresh
            self._graphed.close()
            self._graphed = None
        if not hasattr(self, 'optimizer'):
            self.create_optimizer(model)
        model.load_state_dict(ckpt['model'])
        model.load_resume_state(ckpt['model_resume'])
        self.optimizer.load_state_dict(ckpt['optimizer'])
        rng = ckpt['rng']
        _set_numpy_rng_state(rng['numpy'])
        torch.set_rng_state(rng['torch'])
        for i, s in enumerate(rng['cuda'][:torch.cuda.device_count()]):
            torch.cuda.set_rng_state(s, i)
        loader.load_state(ckpt['loader'])
        tr = ckpt['trainer']
        self.epoch_done = tr['epoch']
        es = tr['early_stop']
        if es is not None and es['best_state'] is not None:
            es['best_state'] = {k: v.to(configs['device']) for k, v in es['best_state'].items()}
        self.early_stop_state = es
        self._log('Load training checkpoint from {} (epoch {})'.format(path, self.epoch_done))
        return self.epoch_done + 1

    @torch.no_grad()
    def evaluate(self, model, epoch_idx=None, loader=None, data_type=None):
        """All-rank evaluation: full_predict -> top-max(k) on device (one fused predict_topk call when the model has it and the catalogue
        has at least FUSED_TOPK_MIN_ITEMS items) -> recall / ndcg / precision / mrr on host
        (metrics.py:11-45, :82-127).  Validation split when the handler has one, else the test split
        (trainer.py:139-150)."""
        seeds = getattr(model, '_seeds', None)
        if seeds is None:
            return self._evaluate(model, epoch_idx, loader, data_type)
        with seeds.host_draws():         # between CUDA-graph replays too, the forward pass takes the next seeds of the host sequence
            return self._evaluate(model, epoch_idx, loader, data_type)

    def _evaluate(self, model, epoch_idx, loader, data_type):
        model.eval()
        if loader is None:
            if hasattr(self.data_handler, 'valid_dataloader'):
                loader, data_type = self.data_handler.valid_dataloader, 'Validation set'
            elif hasattr(self.data_handler, 'test_dataloader'):
                loader, data_type = self.data_handler.test_dataloader, 'Test set'
            else:
                raise NotImplementedError('data handler has neither valid_dataloader nor test_dataloader')
        ks = configs['test']['k']
        metrics = configs['test']['metrics']
        unknown = [m for m in metrics if m not in ('recall', 'ndcg', 'precision', 'mrr')]
        if unknown:
            raise ValueError(f'unknown test metrics {unknown} (metrics.py knows recall, ndcg, precision, mrr)')
        per_user = {m: [] for m in metrics}
        ds = loader.dataset
        n_users = len(ds.test_users)
        ptr, flat = truth_csr(ds)
        seen = 0
        for tem in _eval_batches(loader):
            if not isinstance(tem, (list, tuple)):
                tem = [tem]
            users = tem[0].numpy().astype(np.int64)
            batch_data = list(map(lambda x: x.long().to(configs['device']), tem))
            if len(batch_data) == 1:
                batch_data.append('train')                   # dataset built with dense_mask=False: mask from the device CSR
            if hasattr(model, 'predict_topk') and getattr(model, 'item_num', 0) >= FUSED_TOPK_MIN_ITEMS:     # the same ids either way
                top = model.predict_topk(batch_data, max(ks))
            else:
                top = topk(model.full_predict(batch_data), max(ks))
            seen += top.shape[0]
            top = top.cpu().numpy()
            rows = batch_metric_rows(top, users, ptr, flat, ks, metrics)
            for m in metrics:
                per_user[m].append(rows[m])
        assert seen == n_users, 'evaluation did not cover every test user (metrics.py:113)'
        # one sum over all users in loader order: the result does not depend on how the users were batched
        result = {m: (np.concatenate(per_user[m]).sum(0) / n_users if per_user[m] else np.zeros(len(ks))) for m in metrics}
        if not getattr(self, '_in_test', False):
            self._scalar('HR/test', float(result[metrics[0]][0]), epoch_idx)                       # trainer.py:144,148 (evaluate only, not test)
        if self.logger is not None:
            self.logger.log_eval(result, ks, data_type=data_type or 'Validation set', epoch_idx=epoch_idx)
        return result


def _recluster_flag(loader, tem) -> bool:
    """Whether a training batch carries NCL's k-means flag (its 4th tensor, datasets_general_cf.py:28-44), without a device read:
    host loaders hold the flags in host memory; a DeviceTrnData knows on the host which batch got a set flag (its loader reads
    where pair 0 landed once per epoch)."""
    if len(tem) < 4:
        return False
    flags = tem[3]
    if not flags.is_cuda:
        return bool(flags.any())
    return bool(getattr(loader.dataset, 'last_flag', False))


def _eval_batches(loader):
    """The loader's batches.  A sequential torch DataLoader over a lean AllRankTstData (user ids only: ``dense_mask=False``) is served as
    slices of ``test_users`` -- the same batches without 76 k ``__getitem__`` calls and collates per amazon-sized evaluation."""
    from .data_handler import AllRankTstData
    import torch.utils.data as tdata
    ds = getattr(loader, 'dataset', None)
    if (isinstance(loader, tdata.DataLoader) and isinstance(ds, AllRankTstData) and not ds.dense_mask and loader.batch_size
            and isinstance(loader.sampler, tdata.SequentialSampler) and not loader.drop_last):
        users = torch.from_numpy(np.ascontiguousarray(ds.test_users))
        return (users[lo:lo + loader.batch_size] for lo in range(0, users.numel(), loader.batch_size))
    return iter(loader)


def truth_csr(ds):
    """The held-out positives of an AllRankTstData (``user_pos_lists``, datasets_general_cf.py:52-58) as one flat CSR (ptr int64
    [n_user + 1], items int64 ascending inside a user's list), built once per dataset."""
    cached = getattr(ds, '_truth_csr', None)
    if cached is None:
        import itertools
        lists = ds.user_pos_lists
        lens = np.fromiter((len(x) for x in lists), dtype=np.int64, count=len(lists))
        ptr = np.zeros(len(lists) + 1, dtype=np.int64)
        np.cumsum(lens, out=ptr[1:])
        flat = np.fromiter(itertools.chain.from_iterable(lists), dtype=np.int64, count=int(ptr[-1]))
        owner = np.repeat(np.arange(len(lists), dtype=np.int64), lens)
        flat = flat[np.lexsort((flat, owner))]                # ascending inside every user's list: a batch's (row, item) keys come out sorted
        cached = ds._truth_csr = (ptr, flat)
    return cached


def batch_metric_rows(top, users, ptr, flat, ks, metrics):
    """recall / ndcg / precision / mrr of metrics.py:11-45 for one evaluation batch, one value per row and cut-off, without the
    per-user Python loop (82 us per user on the host: 6 s per amazon-sized evaluation against 0.1-0.4 s of GPU work).

    top   [n, max(ks)] item ids, best first (the top-k of full_predict's masked scores)
    users [n] the rows' user ids; (ptr, flat): ``truth_csr`` of the held-out positives
    -> {metric: float64 [n, len(ks)]}; the caller sums over all test users and divides by their number (metrics.py:122-124)."""
    top = np.asarray(top, dtype=np.int64)
    users = np.asarray(users, dtype=np.int64)
    n, kmax = top.shape
    lens = ptr[users + 1] - ptr[users]
    total = int(lens.sum())
    # (row, item) keys of the batch's ground truth; a hit is a top-k entry whose key is among them (np.isin per row in the loop form)
    first = np.cumsum(lens) - lens
    within = np.arange(total, dtype=np.int64) - np.repeat(first, lens)
    truth_items = flat[np.repeat(ptr[users], lens) + within]
    base = int(max(top.max(initial=0), truth_items.max(initial=0))) + 1
    truth_keys = np.repeat(np.arange(n, dtype=np.int64), lens) * base + truth_items      # ascending (rows ascending, items ascending per row)
    top_keys = np.arange(n, dtype=np.int64)[:, None] * base + top
    if total:
        pos = np.minimum(np.searchsorted(truth_keys, top_keys), total - 1)
        hit = (truth_keys[pos] == top_keys).astype(np.float64)
    else:
        hit = np.zeros(top.shape)
    disc = 1.0 / np.log2(np.arange(2, kmax + 2))              # 1 / log2(rank + 1)
    ideal = np.cumsum(disc)                                   # idcg of a user with j + 1 positives at a cut-off >= j + 1
    denom = np.maximum(lens, 1)
    out = {m: np.zeros((n, len(ks))) for m in metrics}
    for ki, k in enumerate(ks):
        h = hit[:, :k]
        right = h.sum(1)
        if 'recall' in out:
            out['recall'][:, ki] = right / denom
        if 'precision' in out:
            out['precision'][:, ki] = right / k
        if 'ndcg' in out:
            out['ndcg'][:, ki] = (h * disc[:k]).sum(1) / ideal[np.minimum(k, denom) - 1]
        if 'mrr' in out:                                      # metrics.py:24-29: sum of hit / rank over the top k
            out['mrr'][:, ki] = (h / np.arange(1, k + 1)).sum(1)
    return out


class LossReader:
    """Device -> pinned-host reads of a step's loss scalars without blocking the enqueueing thread: ``push``
    starts the copy of this step's values and returns the steps whose copies have already landed."""

    def __init__(self, device, depth: int = 2):
        self.device, self.depth, self.queue = device, depth, []
        self._free = []            # pinned staging buffers are recycled: cudaHostAlloc per step costs milliseconds

    def _staging(self, n):
        for k, h in enumerate(self._free):
            if h.numel() >= n:
                return self._free.pop(k)
        return torch.empty(max(n, 8), dtype=torch.float32, pin_memory=True)

    def push(self, loss, loss_dict):
        names = list(loss_dict)
        vals = torch.stack([loss.detach()] + [torch.as_tensor(loss_dict[n]).detach().to(loss.device).reshape(()) for n in names])
        buf = self._staging(vals.numel())
        host = buf[:vals.numel()]
        host.copy_(vals, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.queue.append((ev, host, names, buf))
        out = []
        while len(self.queue) > self.depth or (self.queue and self.queue[0][0].query()):
            out.append(self._pop())
        return out

    def _pop(self):
        ev, host, names, buf = self.queue.pop(0)
        ev.synchronize()
        v = host.tolist()
        self._free.append(buf)
        return v[0], dict(zip(names, v[1:]))

    def flush(self):
        out = []
        while self.queue:
            out.append(self._pop())
        return out


def topk(preds: torch.Tensor, k: int, return_values: bool = False):
    """The k largest scores per row, descending, ties -> lower item id (replaces torch.topk at
    metrics.py:108)."""
    if not preds.is_cuda:
        raise RuntimeError('sslrec_b200.topk: CUDA tensors only')
    preds = preds.contiguous()
    n_b, n_item = preds.shape
    idx = torch.empty(n_b, k, device=preds.device, dtype=torch.int64)
    val = torch.empty(n_b, k, device=preds.device, dtype=torch.float32)
    with torch.cuda.device(preds.device):
        check(lib.ssl_topk(preds.data_ptr(), n_b, n_item, k, idx.data_ptr(), val.data_ptr(),
                           torch.cuda.current_stream(preds.device).cuda_stream), 'ssl_topk')
    return (idx, val) if return_values else idx
