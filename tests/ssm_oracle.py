"""TEST INFRASTRUCTURE -- restatements of the sampled softmax term (optional key train.ssm_temperature), which has no
counterpart in the reference: the term and its gradients in float64 torch autograd, and the kernels' documented fp32
arithmetic (csrc/ssm.cuh) as a sequential numpy restatement with every FMA emulated exactly."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

EPS = 1e-8                      # x^ = x / sqrt(EPS + |x|^2), the InfoNCE normalisation (loss_utils.py:30-39)


# ---- float64 -------------------------------------------------------------------------------------------------------------------

def scores64(users, items, ancs, poss, cands, tau) -> torch.Tensor:
    """[B, M+1] s_q = u^ . c^_q / tau in the dtype of the tables; column 0 the positive, column 1 + j candidate j."""
    nrm = lambda x: x / torch.sqrt(EPS + (x * x).sum(-1, keepdim=True))
    u = nrm(users[ancs])
    c = nrm(items[torch.cat([poss.view(-1, 1), cands], 1)])
    return torch.einsum('bd,bqd->bq', u, c) / tau


def term64(users, items, ancs, poss, cands, tau) -> torch.Tensor:
    """sum_b lse_q(s_q) - s_0; differentiable in users and items, computed in their dtype."""
    s = scores64(users, items, ancs, poss, cands, tau)
    return (torch.logsumexp(s, 1) - s[:, 0]).sum()


# ---- float32 in the documented order -------------------------------------------------------------------------------------------

def fma32(a, b, c) -> np.ndarray:
    """fmaf(a, b, c) exactly: a * b is exact in float64, the sum is rounded to odd in float64 (TwoSum gives its error), and the
    round-to-odd value rounds to the correctly rounded float32 (53 >= 24 + 2 bits)."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    t = p + c
    bp = t - p
    e = (p - (t - bp)) + (c - bp)
    even = (t.view(np.int64) & 1) == 0
    t = np.where((e != 0) & even & np.isfinite(t), np.nextafter(t, np.where(e > 0, np.inf, -np.inf)), t)
    return t.astype(np.float32)


def group_lanes(d: int) -> int:
    g = 1
    while g * 4 < d:
        g *= 2
    return g


def _tree(v: np.ndarray) -> np.ndarray:
    """The xor butterfly over the last axis (G slots): for o = 1, 2, .. G/2: v_t = v_t + v_(t xor o); -> slot 0's value."""
    G = v.shape[-1]
    t = np.arange(G)
    o = 1
    while o < G:
        v = (v + v[..., t ^ o]).astype(np.float32)
        o *= 2
    return v[..., 0]


def _dot(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """tree over the slots of the per-slot 4-term FMA chains of x . y (broadcast over the leading axes)."""
    d = x.shape[-1]
    x, y = np.broadcast_arrays(x, y)
    xs, ys = x.reshape(x.shape[:-1] + (d // 4, 4)), y.reshape(y.shape[:-1] + (d // 4, 4))
    acc = np.zeros(xs.shape[:-1], np.float32)
    for k in range(4):
        acc = fma32(xs[..., k], ys[..., k], acc)
    v = np.zeros(acc.shape[:-1] + (group_lanes(d),), np.float32)
    v[..., :d // 4] = acc
    return _tree(v)


_libm = C.CDLL('libm.so.6')
for _name in ('expf', 'logf'):
    getattr(_libm, _name).restype = C.c_float
    getattr(_libm, _name).argtypes = [C.c_float]


def libm_expf(x: np.ndarray) -> np.ndarray:
    """The host C library's expf, element by element (the function the host emulation of the kernels calls)."""
    x = np.asarray(x, np.float32)
    return np.array([_libm.expf(float(v)) for v in x.ravel()], np.float32).reshape(x.shape)


def libm_logf(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float32)
    return np.array([_libm.logf(float(v)) for v in x.ravel()], np.float32).reshape(x.shape)


def forward32(u: np.ndarray, c: np.ndarray, tau: float, expf=libm_expf, logf=libm_logf):
    """The forward of csrc/ssm.cuh on gathered rows: u [B, d], c [B, M+1, d] (column 0 the positive) float32 ->
    (loss_b [B], s [B, M+1], w [B, M+1], nrm [B, M+2])."""
    f = np.float32
    tau = f(tau)
    B, Q, d = c.shape
    G = group_lanes(d)
    nu = np.sqrt(f(EPS) + _dot(u, u))
    nq = np.sqrt(f(EPS) + _dot(c, c))
    dt = _dot(u[:, None, :], c)
    den = (nu[:, None] * nq) * tau
    s = (dt / den).astype(f)
    m = np.fmax.reduce(s, axis=1, initial=-np.inf).astype(f)
    ex = expf(s - m[:, None])
    part = np.zeros((B, G), f)
    for q in range(Q):                               # lane t adds q = t, t + G, ... in ascending q
        part[:, q % G] = part[:, q % G] + ex[:, q]
    S = _tree(part)
    loss = ((m + logf(S)) - s[:, 0]).astype(f)
    w = (ex / S[:, None]).astype(f)
    w[:, 0] = w[:, 0] - f(1)
    nrm = np.concatenate([nu[:, None], nq], 1).astype(f)
    return loss, s, w, nrm


def backward32(u: np.ndarray, c: np.ndarray, tau: float, s, w, nrm, g: float):
    """The backward of csrc/ssm.cuh on gathered rows with the upstream scale g (fp32) -> (g_u [B, d], g_c [B, M+1, d]): each
    position's contribution, as the kernel writes it into a -0.0 stage."""
    f = np.float32
    tau, g = f(tau), f(g)
    nu, nq = nrm[:, 0], nrm[:, 1:]
    gw = (g * w).astype(f)
    a = (gw / ((nu[:, None] * nq) * tau)).astype(f)
    e = ((gw * s) / (nq * nq)).astype(f)
    gc = fma32(a[..., None], u[:, None, :], -(e[..., None] * c).astype(f))
    acc = np.zeros_like(u)
    beta = np.zeros(u.shape[0], f)
    for q in range(c.shape[1]):
        acc = fma32(a[:, q, None], c[:, q, :], acc)
        beta = fma32(gw[:, q], s[:, q], beta)
    r = -(beta / (nu * nu)).astype(f)
    return fma32(r[:, None], u, acc), gc
