"""Data side of the plugin surface: mirror of data_utils/data_handler_general_cf.py and
data_utils/datasets_general_cf.py for graphs given as arrays (synthetic or loaded pickles).

``DataHandlerGeneralCF(trn_mat, val_mat, tst_mat)`` exposes what models and trainer read from the
reference's handler: ``torch_adj`` (sparse COO fp32 on ``configs['device']``), ``trn_mat``, the three
dataloaders, and it sets ``configs['data']['user_num'/'item_num']`` in ``load_data`` (:81)."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import torch
import torch.utils.data as data

from .config import configs


def normalized_adjacency(trn_mat: sp.coo_matrix):
    """(rows, cols, vals, N) of D^-1/2 [[0,R],[R^T,0]] D^-1/2, deg = rowsum + 1e-10 in float64, fp32
    values (data_handler_general_cf.py:37-73).  Vectorised; no scipy matrix products."""
    n_user, n_item = trn_mat.shape
    trn_mat = sp.coo_matrix(trn_mat)
    key = np.unique(trn_mat.row.astype(np.int64) * n_item + trn_mat.col.astype(np.int64))
    ur, ic = key // n_item, key % n_item + n_user
    n = n_user + n_item
    rows = np.concatenate([ur, ic])
    cols = np.concatenate([ic, ur])
    deg = np.bincount(rows, minlength=n).astype(np.float64) + 1e-10
    dinv = np.power(deg, -0.5)
    dinv[np.isinf(dinv)] = 0.0
    vals = (dinv[cols] * dinv[rows]).astype(np.float32)
    return rows, cols, vals, n


class PairwiseTrnData(data.Dataset):
    """(user, pos item, neg item) triples; negatives re-drawn every epoch by uniform rejection
    sampling against the user's training positives (datasets_general_cf.py:6-26), vectorised."""

    def __init__(self, coomat):
        self.rows = coomat.row.astype(np.int32)
        self.cols = coomat.col.astype(np.int32)
        self.n_item = coomat.shape[1]
        self._pos_keys = np.unique(self.rows.astype(np.int64) * self.n_item + self.cols.astype(np.int64))
        self.negs = np.zeros(len(self.rows)).astype(np.int32)

    def sample_negs(self, chunk: int = 8192):
        """The reference's loop (datasets_general_cf.py:13-20: per pair, ``np.random.randint(item_num)`` until the item is not one of the user's
        positives) reproduced DRAW FOR DRAW from numpy's global generator -- same negatives, same generator state afterwards -- without the per-pair
        Python loop: ``randint(n, size=k)`` yields the same stream as k scalar calls, so a chunk of pairs takes the next draws in order and the
        (rare) rejected draw only shifts the pairs after it."""
        rows64 = self.rows.astype(np.int64)
        n, keys = len(self.rows), self._pos_keys
        negs = np.zeros(n, dtype=np.int64)

        def is_positive(users, items):
            k = users * self.n_item + items
            pos = np.minimum(np.searchsorted(keys, k), keys.shape[0] - 1)
            return keys[pos] == k if keys.shape[0] else np.zeros(len(k), dtype=bool)

        for lo in range(0, n, chunk):
            hi = min(n, lo + chunk)
            i = lo                                             # next pair without a negative
            stream = np.zeros(0, dtype=np.int64)
            p = 0                                              # next unused draw of ``stream``
            while i < hi:
                if p == len(stream):                           # exactly as many new draws as there are pairs left: nothing is drawn that the loop would not draw
                    stream, p = np.random.randint(self.n_item, size=hi - i).astype(np.int64), 0
                k = min(hi - i, len(stream) - p)
                cand = stream[p:p + k]
                hit = np.flatnonzero(is_positive(rows64[i:i + k], cand))
                if hit.size == 0:
                    negs[i:i + k] = cand
                    i, p = i + k, p + k
                else:                                          # the pairs before the first rejected draw keep theirs; that pair retries with the next draw
                    t = int(hit[0])
                    negs[i:i + t] = cand[:t]
                    i, p = i + t, p + t + 1
        self.negs = negs.astype(np.int32)

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, idx):
        return self.rows[idx], self.cols[idx], self.negs[idx]


class PairwiseWEpochFlagTrnData(PairwiseTrnData):
    """NCL: a flag that is 1 on the very first sample and once every ``epoch_period`` epochs
    (datasets_general_cf.py:28-44)."""

    def __init__(self, coomat):
        super().__init__(coomat)
        self.epoch_flag_counter = -1
        self.epoch_period = configs['model']['epoch_period']

    def __getitem__(self, idx):
        flag = 0
        if self.epoch_flag_counter == -1:
            flag = 1
            self.epoch_flag_counter = 0
        if idx == 0:
            self.epoch_flag_counter += 1
            if self.epoch_flag_counter % self.epoch_period == 0:
                flag = 1
        anc, pos, neg = super().__getitem__(idx)
        return anc, pos, neg, flag

    def flags_for(self, idx: np.ndarray) -> np.ndarray:
        """The flags ``__getitem__`` would return for the samples ``idx`` served in this order (same counter updates)."""
        flags = np.zeros(len(idx), dtype=np.int64)
        if len(idx) and self.epoch_flag_counter == -1:
            flags[0] = 1
            self.epoch_flag_counter = 0
        for p in np.flatnonzero(idx == 0):
            self.epoch_flag_counter += 1
            if self.epoch_flag_counter % self.epoch_period == 0:
                flags[p] = 1
        return flags


class HostBatchLoader:
    """``DataLoader(trn_data, batch_size, shuffle=True, num_workers=0)`` of data_handler_general_cf.py:95, batch for batch: the same
    draws from torch's global generator (the iterator's base seed, then the RandomSampler's seed of a fresh generator whose
    ``randperm`` orders the epoch), the same tensors (int32 pairs and negatives, int64 flags), but a batch is three array gathers
    instead of 4096 ``__getitem__`` calls and a collate (1.5 s -> 0.7 s per amazon-sized epoch of the training loop).
    ``.dataset`` / ``len()`` / iteration are what the trainer uses (trainer.py:52-54,62)."""

    def __init__(self, dataset: PairwiseTrnData, batch_size: int):
        self.dataset, self.batch_size = dataset, int(batch_size)
        self.sampler = None

    def __len__(self):
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        ds, n = self.dataset, len(self.dataset)
        torch.empty((), dtype=torch.int64).random_()                               # _BaseDataLoaderIter._base_seed
        seed = int(torch.empty((), dtype=torch.int64).random_().item())            # RandomSampler.__iter__
        gen = torch.Generator()
        gen.manual_seed(seed)
        perm = torch.randperm(n, generator=gen).numpy()
        with_flags = isinstance(ds, PairwiseWEpochFlagTrnData)
        for lo in range(0, n, self.batch_size):
            idx = perm[lo:lo + self.batch_size]
            out = [torch.from_numpy(ds.rows[idx]), torch.from_numpy(ds.cols[idx]), torch.from_numpy(ds.negs[idx])]
            if with_flags:
                out.append(torch.from_numpy(ds.flags_for(idx)))
            yield out


class DeviceTrnData:
    """The training pairs and their per-epoch negatives resident on the device: ``sample_negs`` is one launch of
    ``ssl_sample_negs`` (rejection sampling against the sorted training CSR; a pure function of seed, epoch and pair)
    instead of the host loop of datasets_general_cf.py:13-26 followed by a host->device copy per batch."""

    def __init__(self, coomat, device, seed: int = 2023, epoch_period=None):
        from ._lib import check, lib                     # raises if the CUDA library is missing: no host fallback here
        self._check, self._lib = check, lib
        coomat = sp.coo_matrix(coomat)
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('DeviceTrnData needs a CUDA device (use PairwiseTrnData + DataLoader on the host)')
        csr = sp.csr_matrix((np.ones(coomat.nnz, dtype=np.float32), (coomat.row, coomat.col)), shape=coomat.shape)
        csr.sum_duplicates()
        csr.sort_indices()
        self.n_item = coomat.shape[1]
        self.rows = torch.from_numpy(coomat.row.astype(np.int64)).to(self.device)
        self.cols = torch.from_numpy(coomat.col.astype(np.int64)).to(self.device)
        self.negs = torch.zeros_like(self.rows)
        self._rowptr = torch.from_numpy(csr.indptr.astype(np.int32)).to(self.device)
        self._csr_cols = torch.from_numpy(csr.indices.astype(np.int32)).to(self.device)
        self.seed, self.epoch = int(seed), 0
        self.epoch_period = epoch_period                 # NCL: pairwise_with_epoch_flag (datasets_general_cf.py:28-44)
        self.epoch_flag_counter = -1

    def sample_negs(self):
        with torch.cuda.device(self.device):
            self._check(self._lib.ssl_sample_negs(self.rows.data_ptr(), self.rows.numel(), self._rowptr.data_ptr(),
                                                  self._csr_cols.data_ptr(), self.n_item, self.seed, self.epoch, self.negs.data_ptr(),
                                                  torch.cuda.current_stream(self.device).cuda_stream), 'ssl_sample_negs')
        self.epoch += 1

    def __len__(self):
        return self.rows.numel()

    def batch(self, idx: torch.Tensor, has_pair0: bool = False):
        """``has_pair0``: the batch contains training pair 0 (the loader knows; no device sync here)."""
        out = [self.rows[idx], self.cols[idx], self.negs[idx]]
        if self.epoch_period is not None:
            # the flag of datasets_general_cf.py:35-44: 1 on the very first sample served, and on sample 0 once
            # every ``epoch_period`` visits of it
            flags = torch.zeros_like(idx)
            self.last_flag = False          # whether this batch carries a set flag, known on the host (graphed NCL steps read it)
            if self.epoch_flag_counter == -1:
                flags[0] = 1
                self.epoch_flag_counter = 0
                self.last_flag = True
            if has_pair0:
                self.epoch_flag_counter += 1
                if self.epoch_flag_counter % self.epoch_period == 0:
                    flags = flags | (idx == 0).long()
                    self.last_flag = True
            out.append(flags)
        return out


class DeviceLoader:
    """``DataLoader(trn_data, batch_size, shuffle=True)`` (data_handler_general_cf.py:95) for a DeviceTrnData: a fresh
    device permutation per epoch, batches gathered on the device.  ``rank`` / ``world`` give each data-parallel
    rank a disjoint share of the same permutation (every rank seeds the same generator)."""

    def __init__(self, dataset: DeviceTrnData, batch_size: int, rank: int = 0, world: int = 1, seed: int = 2023):
        self.dataset, self.batch_size, self.rank, self.world = dataset, int(batch_size), rank, world
        self.sampler = None
        self._gen = torch.Generator(device=dataset.device)
        self._gen.manual_seed(seed)

    def _share(self) -> int:
        return (len(self.dataset) + self.world - 1) // self.world

    def __len__(self):
        return (self._share() + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        perm = torch.randperm(len(self.dataset), device=self.dataset.device, generator=self._gen)
        if self.world > 1:
            share = self._share()
            perm = torch.cat([perm, perm[:share * self.world - perm.numel()]])[self.rank::self.world]   # padded like DistributedSampler
        at0 = -1
        if self.dataset.epoch_period is not None:            # one read per epoch: where pair 0 landed in this rank's share
            hit = (perm == 0).nonzero()
            at0 = int(hit[0]) if hit.numel() else -1
        for lo in range(0, perm.numel(), self.batch_size):
            yield self.dataset.batch(perm[lo:lo + self.batch_size], lo <= at0 < lo + self.batch_size)


class AllRankTstData(data.Dataset):
    """Test users with their held-out positives and a dense train-mask row (datasets_general_cf.py:46-68)."""

    def __init__(self, coomat, trn_mat, dense_mask: bool = True):
        """dense_mask = False: yield only the user id; the model masks from its device CSR of the training matrix
        (``full_predict([users, 'train'])``) instead of a dense float64 [I] row per user built on the host."""
        self.dense_mask = dense_mask
        self.csrmat = (sp.csr_matrix(trn_mat) != 0) * 1.0
        coomat = sp.coo_matrix(coomat)
        order = np.argsort(coomat.row, kind='stable')
        rows, cols = coomat.row[order], coomat.col[order]
        self.user_pos_lists = [list() for _ in range(coomat.shape[0])]
        bounds = np.flatnonzero(np.diff(rows)) + 1
        for u, chunk in zip(rows[np.concatenate([[0], bounds])] if len(rows) else [], np.split(cols, bounds) if len(rows) else []):
            self.user_pos_lists[int(u)] = chunk.tolist()
        self.test_users = np.unique(rows)

    def __len__(self):
        return len(self.test_users)

    def __getitem__(self, idx):
        pck_user = self.test_users[idx]
        if not self.dense_mask:
            return pck_user
        pck_mask = np.reshape(self.csrmat[pck_user].toarray(), [-1])
        return pck_user, pck_mask


class DataHandlerGeneralCF:
    """``DataHandlerGeneralCF()`` -- no arguments, as the reference builds it (build_data_handler.py) -- loads
    ./datasets/general_cf/sparse_{yelp,gowalla,amazon}/{train,valid,test}_mat.pkl chosen by ``configs['data']['name']``
    (data_handler_general_cf.py:11-35); ``DataHandlerGeneralCF(trn_mat, val_mat, tst_mat)`` takes the matrices directly
    (synthetic graphs, tests)."""

    def __init__(self, trn_mat=None, val_mat=None, tst_mat=None):
        if trn_mat is None:
            name = configs['data']['name']
            if name not in ('yelp', 'gowalla', 'amazon'):
                raise ValueError(f"data.name '{name}': the general_cf handler knows yelp, gowalla, amazon (data_handler_general_cf.py:12-17)")
            predir = './datasets/general_cf/sparse_{}/'.format(name)
            self.trn_file, self.val_file, self.tst_file = predir + 'train_mat.pkl', predir + 'valid_mat.pkl', predir + 'test_mat.pkl'
            self._mats = None
        else:
            self.trn_file = self.val_file = self.tst_file = None
            self._mats = (sp.coo_matrix(trn_mat), val_mat, tst_mat)

    def _load_one_mat(self, file):
        """data_handler_general_cf.py:21-35: pickled scipy matrix -> binary float32 COO."""
        import pickle
        with open(file, 'rb') as fs:
            mat = (pickle.load(fs) != 0).astype(np.float32)
        return sp.coo_matrix(mat)

    def _make_torch_adj(self, mat):
        rows, cols, vals, n = normalized_adjacency(mat)
        idxs = torch.from_numpy(np.vstack([rows, cols]).astype(np.int64))
        adj = torch.sparse_coo_tensor(idxs, torch.from_numpy(vals), (n, n), check_invariants=False)
        return adj.to(configs['device'])

    def load_data(self):
        if self._mats is None:
            self._mats = (self._load_one_mat(self.trn_file), self._load_one_mat(self.val_file), self._load_one_mat(self.tst_file))
        trn_mat, val_mat, tst_mat = self._mats
        trn_mat = sp.coo_matrix((trn_mat != 0).astype(np.float32))
        self.trn_mat = trn_mat
        configs['data']['user_num'], configs['data']['item_num'] = trn_mat.shape
        self.torch_adj = self._make_torch_adj(trn_mat)
        if configs['train']['loss'] == 'pairwise':
            trn_data = PairwiseTrnData(trn_mat)
        elif configs['train']['loss'] == 'pairwise_with_epoch_flag':
            trn_data = PairwiseWEpochFlagTrnData(trn_mat)
        else:
            raise NotImplementedError(configs['train']['loss'])
        if configs['train'].get('device_loader', False):
            # optional key: pairs, negative sampling and batching on the device (no per-sample host collate, no H2D per batch)
            period = configs['model']['epoch_period'] if configs['train']['loss'] == 'pairwise_with_epoch_flag' else None
            seed = configs['train'].get('seed', 2023)
            self.train_dataloader = DeviceLoader(DeviceTrnData(trn_mat, configs['device'], seed, period), configs['train']['batch_size'], seed=seed)
        else:
            # the reference's DataLoader(shuffle=True) batch for batch, without the per-sample collate (optional key train.torch_dataloader: true
            # keeps torch's DataLoader itself)
            if configs['train'].get('torch_dataloader', False):
                self.train_dataloader = data.DataLoader(trn_data, batch_size=configs['train']['batch_size'], shuffle=True, num_workers=0)
            else:
                self.train_dataloader = HostBatchLoader(trn_data, configs['train']['batch_size'])
        # optional key test.dense_mask: true = the reference's dense float64 [I] train-mask row per test user, built on the host and shipped per
        # batch (datasets_general_cf.py:64-68; 686 MB per 1024-user batch at the amazon shape); default: the model masks from its device CSR
        dense = configs['test'].get('dense_mask', False)
        if val_mat is not None:
            self.valid_dataloader = data.DataLoader(AllRankTstData(val_mat, trn_mat, dense), batch_size=configs['test']['batch_size'], shuffle=False, num_workers=0)
        if tst_mat is not None:
            self.test_dataloader = data.DataLoader(AllRankTstData(tst_mat, trn_mat, dense), batch_size=configs['test']['batch_size'], shuffle=False, num_workers=0)
