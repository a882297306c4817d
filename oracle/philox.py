"""TEST INFRASTRUCTURE (oracle) -- numpy restatement of the counter-based draws the CUDA path evaluates
in-kernel (sslrec_b200/csrc/common.cuh), so tests can check them bit for bit instead of statistically.

The reference draws its masks / noise / negatives from torch's and numpy's global generators
(aug_utils.py:28,49,129; datasets_general_cf.py:20); those streams cannot be reproduced inside a kernel,
so the product keys Philox4x32-10 by (seed, stream, row, col).  What must match the reference is the
USE of the uniforms -- ``floor(U + keep)`` for EdgeDrop / NodeDrop, ``U[0,1)`` noise, uniform rejection
sampling -- and that is what these functions restate on top of the same Philox blocks.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)
TAG_EDGE, TAG_NODE, TAG_NOISE, TAG_NEGS, TAG_HYPR = 0x45444745, 0x4E4F4445, 0x4E4F4953, 0x4E454753, 0x48595052


def philox4x32_10(c0, c1, c2, c3, seed: int):
    """Four uint32 arrays (broadcast together) -> four uint32 arrays; key = the 64-bit seed (lo, hi)."""
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, dtype=np.uint64) & MASK for c in (c0, c1, c2, c3)))
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2                              # 32 x 32 -> 64 bit products
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK, p1 >> np.uint64(32), p1 & MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def u01(x: np.ndarray) -> np.ndarray:
    """24-bit uniform in [0, 1) as float32 (common.cuh u01)."""
    return (x >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def edge_keep(seed: int, stream: int, rows, cols, keep: float) -> np.ndarray:
    """EdgeDrop mask floor(U + keep) == 1 of the stored entries (rows, cols) (aug_utils.py:28)."""
    r = philox4x32_10(rows, cols, stream, TAG_EDGE, seed)[0]
    return (u01(r) + np.float32(keep)) >= np.float32(1.0)


def node_keep(seed: int, rows, keep: float) -> np.ndarray:
    """NodeDrop mask (aug_utils.py:49)."""
    r = philox4x32_10(rows, 0, 0, TAG_NODE, seed)[0]
    return (u01(r) + np.float32(keep)) >= np.float32(1.0)


def noise_uniform(seed: int, stream: int, n_rows: int, dim: int, row_offset: int = 0) -> np.ndarray:
    """The [n_rows, dim] uniforms of EmbedPerturb (aug_utils.py:129): element (r, 4q + t) is word t of the block
    keyed (r, q, stream)."""
    rows = (np.arange(n_rows, dtype=np.uint64) + np.uint64(row_offset))[:, None]
    quads = np.arange((dim + 3) // 4, dtype=np.uint64)[None, :]
    words = philox4x32_10(rows, quads, stream, TAG_NOISE, seed)
    return np.stack([u01(w) for w in words], axis=-1).reshape(n_rows, -1)[:, :dim]


def hyper_keep(seed: int, stream: int, n: int, h: int, keep: float) -> np.ndarray:
    """The [n, h] keep mask of HCCF's incidence dropout (hccf.py:48-49, ssl_hyper_dropout mode 1): element (r, 4q + t) is
    kept when word t of the block keyed (r, q, stream, HYPR) gives floor(U + keep) == 1, evaluated in float32."""
    rows = np.arange(n, dtype=np.uint64)[:, None]
    quads = np.arange(h // 4, dtype=np.uint64)[None, :]
    words = philox4x32_10(rows, quads, stream, TAG_HYPR, seed)
    u = np.stack([u01(w) for w in words], axis=-1).reshape(n, h)
    return (u + np.float32(keep)) >= np.float32(1.0)


def sample_negs(users, trn_rowptr, trn_cols, n_item: int, seed: int, epoch: int) -> np.ndarray:
    """Uniform rejection sampling of one negative per training pair (datasets_general_cf.py:17-23) on the draws
    of ssl_sample_negs: draw t of pair e = word t % 4 of the block keyed (e lo, e hi, t // 4, epoch ^ TAG)."""
    users = np.asarray(users, dtype=np.int64)
    keys = np.asarray(trn_rowptr, dtype=np.int64)
    pos = set()
    for u in np.unique(users):
        for c in trn_cols[keys[u]:keys[u + 1]]:
            pos.add((int(u), int(c)))
    e = np.arange(len(users), dtype=np.uint64)
    negs = np.zeros(len(users), dtype=np.int64)
    todo = np.arange(len(users))
    for blk in range(64):
        if not todo.size:
            break
        words = philox4x32_10(e[todo] & MASK, e[todo] >> np.uint64(32), blk, (epoch ^ TAG_NEGS) & 0xFFFFFFFF, seed)
        live = np.ones(todo.size, dtype=bool)                  # pairs whose draws of this block were all rejected so far
        for t in range(4):
            sel = np.flatnonzero(live)
            cand = ((words[t][sel].astype(np.uint64) * np.uint64(n_item)) >> np.uint64(32)).astype(np.int64)
            negs[todo[sel]] = cand
            hit = np.fromiter(((int(u), int(c)) in pos for u, c in zip(users[todo[sel]], cand)), dtype=bool, count=sel.size)
            live[sel[~hit]] = False
        todo = todo[live]
    return negs
