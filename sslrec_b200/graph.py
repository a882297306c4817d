"""Adjacency plan: the reference's ``data_handler.torch_adj`` (an uncoalesced, column-sorted COO
fp32 tensor, data_utils/data_handler_general_cf.py:53-73) converted ONCE to the int32 CSR the
sm_90a propagation kernel walks.  The structure and the values are symmetric (D^-1/2 A D^-1/2
of an undirected bipartite graph), so the same CSR serves the forward SpMM and the transposed
SpMM of the backward pass; only an *injected* edge mask needs the reverse-entry permutation.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


class GraphPlan:
    """CSR of (a row shard of) the normalised adjacency + the native work lists.

    rows/cols/vals : COO triplets in ANY order (numpy or torch, host or device).
    n             : number of nodes N = |U| + |I| (matrix is N x N).
    row_ranges    : ((a0, a1), (b0, b1)) global rows owned by this plan (row-sharded multi-GPU: the rank's share
                    of the user rows and of the item rows); ``row_range`` = one range; default all rows.
    ``coo_to_csr`` maps the caller's entry order to CSR positions so masks given in the
    reference's COO order (aug_utils.py:25-30) can be injected.
    """

    def __init__(self, rows, cols, vals, n: int, device: torch.device, row_range=None, need_rev: bool = False, side_split: int = 0,
                 row_ranges=None):
        n = int(n)
        sharded = row_range is not None or row_ranges is not None
        ranges = _ranges(n, row_range, row_ranges)
        rowptr, rows_s, cols_s, vals_s, order = local_csr(rows, cols, vals, ranges)
        if not sharded:
            self.coo_to_csr_full = np.empty_like(order)
            self.coo_to_csr_full[order] = np.arange(order.shape[0])
        rev = None
        if need_rev:
            if sharded:
                raise ValueError('injected masks (rev) are a single-GPU debugging aid')
            key = rows_s * n + cols_s
            keyt = cols_s * n + rows_s
            pos = np.searchsorted(key, keyt)
            if not np.array_equal(key[pos], keyt):
                raise ValueError('adjacency structure is not symmetric')
            rev = torch.from_numpy(pos.astype(np.int32)).to(device)
        self._setup(np.ascontiguousarray(rowptr.astype(np.int32)), torch.from_numpy(cols_s.astype(np.int32)).to(device),
                    torch.from_numpy(vals_s).to(device), n, torch.device(device), ranges, rev, side_split)

    @classmethod
    def from_csr(cls, h_rowptr, colidx: torch.Tensor, vals: torch.Tensor, n: int, row_ranges=None, side_split: int = 0) -> 'GraphPlan':
        """From a ready CSR of the owned rows: host int32 rowptr over the local rows (range a then range b), device
        int32 global column ids (ascending inside a row) and device fp32 values -- no host sort (BASELINE config 4)."""
        self = cls.__new__(cls)
        self._setup(np.ascontiguousarray(np.asarray(h_rowptr, dtype=np.int32)), colidx.contiguous(), vals.contiguous(), int(n),
                    colidx.device, _ranges(int(n), None, row_ranges), None, side_split)
        return self

    def _setup(self, h_rowptr, colidx, vals, n, device, ranges, rev, side_split):
        (a0, a1), (b0, b1) = ranges
        self.n, self.device, self.ranges = n, torch.device(device), ranges
        self.row_offset, self.n_rows = a0, (a1 - a0) + (b1 - b0)      # row_offset: first owned row (single-range plans)
        self.entry_lo = 0
        self.h_rowptr, self.colidx, self.vals, self.rev = h_rowptr, colidx, vals, rev
        self.nnz = int(colidx.shape[0])
        if colidx.dtype != torch.int32 or vals.dtype != torch.float32 or h_rowptr.shape[0] != self.n_rows + 1:
            raise ValueError('CSR arrays must be int32 colidx, fp32 vals, rowptr of n_rows + 1 entries')
        self._handle = C.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib.ssl_plan_create_ranges(
                C.byref(self._handle), self.h_rowptr.ctypes.data, self.colidx.data_ptr(), self.vals.data_ptr(),
                self.rev.data_ptr() if self.rev is not None else None,
                self.n_rows, self.n, self.nnz, a0, a1, b0, b1, int(side_split), stream), 'ssl_plan_create_ranges')

    def rowptr_dev(self) -> torch.Tensor:
        """The owned rows' CSR row pointer on the device (int32 [n_rows + 1]; the propagation kernel walks its own work list and never
        reads it -- only the exact-order evaluation SpMM does)."""
        if getattr(self, '_rowptr_dev', None) is None:
            self._rowptr_dev = torch.from_numpy(np.ascontiguousarray(self.h_rowptr)).to(self.device)
        return self._rowptr_dev

    def owned_rows(self) -> torch.Tensor:
        """Global ids of the owned rows in local order (host int64)."""
        (a0, a1), (b0, b1) = self.ranges
        return torch.cat([torch.arange(a0, a1), torch.arange(b0, b1)])

    @classmethod
    def from_torch_adj(cls, adj: torch.Tensor, device=None, need_rev: bool = False, side_split: int = 0) -> 'GraphPlan':
        """From the reference's sparse COO tensor (any device).  side_split = |U| orders the work list side by side."""
        idx = adj._indices() if adj.layout == torch.sparse_coo else adj.to_sparse_coo()._indices()
        val = adj._values() if adj.layout == torch.sparse_coo else adj.to_sparse_coo()._values()
        device = device if device is not None else adj.device
        return cls(idx[0].cpu().numpy(), idx[1].cpu().numpy(), val.cpu().numpy(), adj.shape[0], device, need_rev=need_rev, side_split=side_split)

    @property
    def handle(self):
        return self._handle

    def stats(self):
        out = (C.c_int64 * 4)()
        _lib.check(_lib.lib.ssl_plan_stats(self._handle, out))
        return dict(items=out[0], split_rows=out[1], segments=out[2], max_row_nnz=out[3])

    def mask_to_csr(self, mask_in_caller_order) -> torch.Tensor:
        """uint8 keep-mask given in the order of the COO triplets passed to the constructor ->
        device uint8 tensor in CSR entry order (what edge_mode 2 reads)."""
        if not hasattr(self, 'coo_to_csr_full'):
            raise ValueError('injected masks are a single-GPU debugging aid (row-sharded plans keep no COO map)')
        m = _np(mask_in_caller_order).astype(np.uint8)
        out = np.empty_like(m)
        out[self.coo_to_csr_full] = m
        return torch.from_numpy(out[self.entry_lo:self.entry_lo + self.nnz].copy()).to(self.device)

    def __del__(self):
        try:
            if getattr(self, '_handle', None) is not None and self._handle.value:
                _lib.lib.ssl_plan_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def local_csr(rows, cols, vals, ranges):
    """Host part of a (sharded) plan: the COO entries whose row lies in ``ranges`` = ((a0, a1), (b0, b1)), sorted into CSR
    order over the local rows (range a, then range b).  -> (rowptr int64 [n_local + 1], global rows, cols, vals of the
    kept entries in CSR order, and ``order``: positions of those entries in the caller's arrays)."""
    rows = _np(rows).astype(np.int64)
    cols = _np(cols).astype(np.int64)
    vals = _np(vals).astype(np.float32)
    (a0, a1), (b0, b1) = ranges
    keep = np.flatnonzero(((rows >= a0) & (rows < a1)) | ((rows >= b0) & (rows < b1)))
    order = keep[np.lexsort((cols[keep], rows[keep]))]          # CSR order: row, then col (range a precedes range b)
    rows_s, cols_s, vals_s = rows[order], cols[order], vals[order]
    rows_l = np.where(rows_s < a1, rows_s - a0, rows_s - b0 + (a1 - a0))
    n_rows = (a1 - a0) + (b1 - b0)
    rowptr = np.zeros(n_rows + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum(np.bincount(rows_l, minlength=n_rows))
    if rows_l.shape[0] >= 2 ** 31 - 1:
        raise ValueError('a plan holds at most 2^31-2 entries; shard the rows')
    return rowptr, rows_s, cols_s, vals_s, order


def _ranges(n, row_range, row_ranges):
    if row_ranges is not None:
        (a0, a1), (b0, b1) = row_ranges
        if b1 == b0:
            b0 = b1 = a1
        return (int(a0), int(a1)), (int(b0), int(b1))
    r0, r1 = (0, n) if row_range is None else (int(row_range[0]), int(row_range[1]))
    return (r0, r1), (r1, r1)


def _np(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return np.asarray(x)
