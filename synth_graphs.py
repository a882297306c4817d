"""Synthetic bipartite interaction graphs with the shape statistics of the reference's datasets
(SURVEY.md section 8d): user degree ~ lognormal(sigma = 1) scaled to the requested mean and clipped
to [1, 1e4], items drawn by Zipf(alpha) popularity over a random permutation of the item ids,
duplicates removed, exactly ``n_edge`` unique (user, item) pairs.  numpy PCG64, fixed seed."""
from __future__ import annotations

import numpy as np

# |U|, |I|, E of the reference's bundled train matrices (SURVEY.md section 8) and BASELINE.json config 4
SHAPES = {
    'gowalla': (25557, 19747, 294983),
    'yelp': (42712, 26822, 182357),
    'amazon': (76469, 83761, 966680),
    'synthetic-xl': (5_000_000, 1_000_000, 150_000_000),       # config 4: the whole graph trains on one 80 GB GPU
    'synthetic-xl-8th': (625_000, 125_000, 18_750_000),      # one GPU's eighth of config 4 (same degree statistics)
}
# item-popularity exponent: 0.5 reproduces the bundled datasets' head (max item degree ~1e3 at
# amazon's size; the real matrices have 841 / 309 / 1018); 1.0 is BASELINE.json config 4's generator
ZIPF = {'gowalla': 0.5, 'yelp': 0.5, 'amazon': 0.5, 'synthetic-xl': 1.0, 'synthetic-xl-8th': 1.0}


def named_graph(name: str, seed: int = 2023):
    n_user, n_item, n_edge = SHAPES[name]
    rows, cols = bipartite_graph(n_user, n_item, n_edge, seed, ZIPF[name])
    return rows, cols, n_user, n_item


def _merge_unique(keys: np.ndarray, new: np.ndarray) -> np.ndarray:
    """sorted-unique union of a sorted-unique array with arbitrary new values (one sort of ``new`` only)."""
    new.sort()
    if new.size:
        new = new[np.concatenate([[True], new[1:] != new[:-1]])]
    if keys.size == 0:
        return new
    pos = np.searchsorted(keys, new)
    fresh = (pos == keys.size) | (keys[np.minimum(pos, keys.size - 1)] != new)
    return np.insert(keys, pos[fresh], new[fresh])


def bipartite_graph(n_user: int, n_item: int, n_edge: int, seed: int = 2023, zipf_alpha: float = 1.0):
    rng = np.random.Generator(np.random.PCG64(seed))
    deg = rng.lognormal(mean=0.0, sigma=1.0, size=n_user)
    deg = np.clip(deg * (n_edge / deg.sum()), 1, 1e4)
    deg = np.maximum(1, np.round(deg * (n_edge / deg.sum()))).astype(np.int64)
    pop = 1.0 / np.arange(1, n_item + 1, dtype=np.float64) ** zipf_alpha
    cdf = np.cumsum(pop)
    cdf /= cdf[-1]
    perm = rng.permutation(n_item)
    keys = np.empty(0, dtype=np.int64)
    want = deg.copy()
    for it in range(12):
        users = np.repeat(np.arange(n_user, dtype=np.int64), want)
        if it < 2:          # popularity-driven draws; later passes fill the collision losses uniformly
            items = perm[np.searchsorted(cdf, rng.random(users.shape[0]), side='right').clip(0, n_item - 1)]
        else:
            items = rng.integers(0, n_item, size=users.shape[0], dtype=np.int64)
        keys = _merge_unique(keys, users * n_item + items)
        if keys.shape[0] >= n_edge:
            break
        missing = n_edge - keys.shape[0]
        have = np.bincount(keys // n_item, minlength=n_user)
        want = np.maximum(deg - have, 0)
        short = missing - int(want.sum())
        if short > 0:       # rounding of the degree targets: spread the remainder over random users
            want = want + np.bincount(rng.integers(0, n_user, size=int(short * 1.05) + 1), minlength=n_user)
    if keys.shape[0] > n_edge:
        keys = np.sort(rng.choice(keys, size=n_edge, replace=False))
    if keys.shape[0] != n_edge:
        raise RuntimeError('could not place %d unique edges' % n_edge)
    return (keys // n_item).astype(np.int64), (keys % n_item).astype(np.int64)


# --------------------------------------------------------------------------------------------------
# The same family of graphs generated ON THE DEVICE (torch CUDA ops), for BASELINE.json config 4
# (5 M x 1 M nodes, 150 M edges): the numpy path above needs minutes and tens of GB of host memory
# at that size, the device path a few seconds.  Same distributions (lognormal user degrees, Zipf item
# popularity over a random permutation, duplicates removed, exactly n_edge pairs), torch's Philox
# generator with a fixed seed -- NOT bit-identical to the numpy generator.
# --------------------------------------------------------------------------------------------------

def bipartite_keys_device(n_user: int, n_item: int, n_edge: int, seed: int, zipf_alpha: float, device):
    """Sorted unique int64 keys u * n_item + i of exactly ``n_edge`` (user, item) pairs, on ``device``."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    deg = torch.exp(torch.randn(n_user, device=device, dtype=torch.float64, generator=g))
    deg = (deg * (n_edge / deg.sum())).clamp_(1, 1e4)
    deg = torch.round(deg * (n_edge / deg.sum())).clamp_(min=1).to(torch.int64)
    pop = 1.0 / torch.arange(1, n_item + 1, device=device, dtype=torch.float64) ** zipf_alpha
    cdf = torch.cumsum(pop, 0)
    cdf /= cdf[-1].clone()
    perm = torch.randperm(n_item, device=device, generator=g)
    arange_u = torch.arange(n_user, device=device, dtype=torch.int64)
    keys = torch.empty(0, device=device, dtype=torch.int64)
    want = deg.clone()
    for it in range(16):
        users = torch.repeat_interleave(arange_u, want)
        if it < 2:
            r = torch.rand(users.shape[0], device=device, dtype=torch.float64, generator=g)
            items = perm[torch.searchsorted(cdf, r, right=True).clamp_(max=n_item - 1)]
            del r
        else:
            items = torch.randint(0, n_item, (users.shape[0],), device=device, generator=g)
        new = users * n_item + items
        del users, items
        keys = torch.unique(torch.cat([keys, new]))
        del new
        if keys.shape[0] >= n_edge:
            break
        missing = n_edge - keys.shape[0]
        have = torch.bincount(keys // n_item, minlength=n_user)
        want = (deg - have).clamp_(min=0)
        short = missing - int(want.sum())
        if short > 0:
            extra = torch.randint(0, n_user, (int(short * 1.05) + 1,), device=device, generator=g)
            want = want + torch.bincount(extra, minlength=n_user)
    if keys.shape[0] < n_edge:
        raise RuntimeError('could not place %d unique edges' % n_edge)
    if keys.shape[0] > n_edge:
        keep = torch.randperm(keys.shape[0], device=device, generator=g)[:n_edge]
        keys = keys[keep].sort().values
    return keys


def normalized_csr_device(keys, n_user: int, n_item: int, ranges=None):
    """CSR (host int32 rowptr, device int32 colidx, device fp32 vals) of the rows ``ranges`` = ((a0, a1), (b0, b1)) of
    D^-1/2 [[0, R], [R^T, 0]] D^-1/2 (deg = rowsum + 1e-10 in float64, fp32 values: the formula of
    sslrec_b200.data_handler.normalized_adjacency / data_handler_general_cf.py:37-73), from the sorted unique edge keys.
    Range a must lie in the user rows, range b in the item rows (global ids |U| + i); default = every row."""
    import torch
    dev = keys.device
    n = n_user + n_item
    if ranges is None:
        ranges = ((0, n_user), (n_user, n))
    (a0, a1), (b0, b1) = ranges
    assert 0 <= a0 <= a1 <= n_user and n_user <= b0 <= b1 <= n
    ku, ki = keys // n_item, keys % n_item
    deg_u = torch.bincount(ku, minlength=n_user)
    deg_i = torch.bincount(ki, minlength=n_item)
    dinv = torch.pow(torch.cat([deg_u, deg_i]).to(torch.float64) + 1e-10, -0.5)
    # user rows [a0, a1): the keys are sorted by (u, i) -> a contiguous slice, already in CSR order
    lo, hi = torch.searchsorted(keys, torch.tensor([a0 * n_item, a1 * n_item], device=dev, dtype=torch.int64)).tolist()
    col_a = (ki[lo:hi] + n_user)
    val_a = (dinv[col_a] * dinv[ku[lo:hi]]).to(torch.float32)
    rp_a = torch.cumsum(deg_u[a0:a1], 0)
    # item rows [b0, b1): entries (i, u) sorted by (i, u)
    i0, i1 = b0 - n_user, b1 - n_user
    sel = (ki >= i0) & (ki < i1)
    kt = (ki[sel] - i0) * n_user + ku[sel]
    del sel
    kt = kt.sort().values
    col_b = kt % n_user
    row_b = kt // n_user + b0
    val_b = (dinv[col_b] * dinv[row_b]).to(torch.float32)
    del kt, row_b
    rp_b = torch.cumsum(deg_i[i0:i1], 0) + (hi - lo)
    rowptr = torch.cat([torch.zeros(1, device=dev, dtype=torch.int64), rp_a, rp_b])
    colidx = torch.cat([col_a, col_b]).to(torch.int32)
    vals = torch.cat([val_a, val_b])
    if int(rowptr[-1]) != colidx.shape[0] or colidx.shape[0] >= 2 ** 31 - 1:
        raise RuntimeError('bad CSR assembly')
    return rowptr.to(torch.int32).cpu().numpy(), colidx, vals
