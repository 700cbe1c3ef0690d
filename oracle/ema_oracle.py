"""fp64 oracle of the EMA codebook (``EMAVectorQuantizer``) -- TEST INFRASTRUCTURE ONLY.

The reference has no EMA quantiser, so there is no reference code to be at parity with.  This file restates the
published algorithm instead: van den Oord et al. 2017, "Neural Discrete Representation Learning", appendix A.1, in the
form Taming Transformers' ``EMAVectorQuantizer`` uses (smoothed cluster sizes, the update applied after the lookup), on
top of the reference's lookup (quantizers.py:38-92: normalised residual, first-minimum argmin, residual depth loop).

Everything is numpy float64.  The statistics are taken over the codes given to them (the kernels' own codes in the
tests): on an fp32 near-tie the fp64 lookup may pick the other code, which says nothing about the statistics.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

NORM_EPS = 1e-12


def norm(x: np.ndarray, use_norm: bool = True) -> np.ndarray:
    """BaseQuantizer.norm (quantizers.py:24): x / max(|x|, 1e-12), or the identity when use_norm is False"""
    x = np.asarray(x, dtype=np.float64)
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), NORM_EPS) if use_norm else x


def lookup(z: np.ndarray, E: np.ndarray, depth: int = 1, use_norm: bool = True) -> np.ndarray:
    """the residual lookup in fp64: z [M, D], E [K, D] -> idx int64 [M, depth] (first minimum)"""
    r = np.asarray(z, dtype=np.float64).copy()
    en = norm(E, use_norm)
    idx = np.empty((r.shape[0], depth), dtype=np.int64)
    for t in range(depth):
        x = norm(r, use_norm)
        d = (x * x).sum(1, keepdims=True) + (en * en).sum(1) - 2.0 * x @ en.T
        idx[:, t] = d.argmin(1)
        r = r - en[idx[:, t]]
    return idx


def compared_vectors(z: np.ndarray, E: np.ndarray, idx: np.ndarray, use_norm: bool = True) -> np.ndarray:
    """x[m, t]: the vector the lookup compared at depth t (the normalised residual), following the given codes"""
    idx = idx.reshape(idx.shape[0], -1)
    r = np.asarray(z, dtype=np.float64).copy()
    en = norm(E, use_norm)
    xs = []
    for t in range(idx.shape[1]):
        xs.append(norm(r, use_norm))
        r = r - en[idx[:, t]]
    return np.stack(xs, 1)


def statistics(z: np.ndarray, E: np.ndarray, idx: np.ndarray, use_norm: bool = True) -> Tuple[np.ndarray, np.ndarray]:
    """n [K] int64 = occurrences of each code over all tokens and depths; s [K, D] = sum of the compared vectors"""
    K, D = E.shape
    x = compared_vectors(z, E, idx, use_norm).reshape(-1, D)
    flat = idx.reshape(-1)
    n = np.bincount(flat, minlength=K).astype(np.int64)
    s = np.zeros((K, D), dtype=np.float64)
    np.add.at(s, flat, x)
    return n, s


def allreduce(stats):
    """the cross-rank reduction: (n, s) summed over the replicas"""
    return sum(st[0] for st in stats), sum(st[1] for st in stats)


def update(cluster_size: np.ndarray, embed_avg: np.ndarray, n: np.ndarray, s: np.ndarray, decay: float,
           eps: float) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """-> (cluster_size, embed_avg, weight) after one update"""
    cs = decay * np.asarray(cluster_size, np.float64) + (1.0 - decay) * np.asarray(n, np.float64)
    ea = decay * np.asarray(embed_avg, np.float64) + (1.0 - decay) * np.asarray(s, np.float64)
    N = cs.sum()
    smoothed = (cs + eps) / (N + len(cs) * eps) * N
    return cs, ea, ea / smoothed[:, None]


def loss(z: np.ndarray, E: np.ndarray, idx: np.ndarray, beta: float = 0.25, use_norm: bool = True) -> float:
    """beta * mean((sg(q) - x)^2) per depth, averaged over the depths; no codebook term"""
    idx = idx.reshape(idx.shape[0], -1)
    x = compared_vectors(z, E, idx, use_norm)
    q = norm(E, use_norm)[idx]
    return float(np.mean([beta * ((q[:, t] - x[:, t]) ** 2).mean() for t in range(idx.shape[1])]))


def grad_z(z: np.ndarray, E: np.ndarray, idx: np.ndarray, g_out: np.ndarray, g_loss: float, beta: float = 0.25,
           use_norm: bool = True, residual: bool = False) -> np.ndarray:
    """gradient at z: the straight-through g_out plus, in plain mode, the commitment term
    g_loss * beta * 2 / (M D) * J_norm(z)^T (norm(z) - q).  In residual mode the residual is built from z.detach()
    (quantizers.py:43): g_out alone."""
    g = np.asarray(g_out, dtype=np.float64).copy()
    if residual:
        return g
    z = np.asarray(z, dtype=np.float64)
    M, D = z.shape
    zn = norm(z, use_norm)
    v = zn - norm(E, use_norm)[idx.reshape(-1)]
    if use_norm:
        nz = np.maximum(np.linalg.norm(z, axis=1, keepdims=True), NORM_EPS)
        v = (v - zn * (zn * v).sum(1, keepdims=True)) / nz
    return g + g_loss * beta * 2.0 / (M * D) * v
