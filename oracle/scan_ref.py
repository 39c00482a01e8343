"""ORACLE (test infrastructure, NOT product code): numpy restatement of psam_voxel_subsample_f32 (csrc/scan.cu) in the order
stated in include/psam_b200.h - quantisation, the cell keys of every level, the level counts, L*, one representative per
cell and the hash thinning.  The hash is mesh_ref's splitmix64 finaliser.  The nearest-key search is checked against
oracle.tokenizer_ref.knn(query, key, 1), the exact C kNN with the device's distance and tie rule."""
from __future__ import annotations

import numpy as np

from oracle.mesh_ref import GOLDEN, U64, splitmix

F32 = np.float32
LEVELS = 22
QMAX = 2 ** 21 - 1


def quantize(xyz):
    """(q [P, 3] int64, valid [P] bool): q_a = clamp(floor(fl(x_a + 1) * 2^20), 0, 2^21 - 1) in fp32; q is 0 where invalid."""
    x = np.asarray(xyz, F32).reshape(-1, 3)
    valid = np.isfinite(x).all(1)
    with np.errstate(all="ignore"):
        t = np.floor((x + F32(1)) * F32(2 ** 20))
        t = np.minimum(np.maximum(t, F32(0)), F32(QMAX))
    return np.where(valid[:, None], t, 0).astype(np.int64), valid


def cell_keys(q: np.ndarray, L: int) -> np.ndarray:
    k = q >> (21 - L)
    return ((k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]).astype(np.int64)


def centre_dist(q: np.ndarray, L: int) -> np.ndarray:
    """e = sum_a (2 q_a + 1 - (2 k_a + 1) 2^(21 - L))^2, exact int64."""
    s = 21 - L
    d = 2 * q + 1 - (2 * (q >> s) + 1) * (1 << s)
    return (d * d).sum(1)


def level_counts(xyz) -> np.ndarray:
    """n_L for L = 0 .. 21: distinct occupied cells of the valid points."""
    q, valid = quantize(xyz)
    u = np.unique(cell_keys(q[valid], 21))  # the occupied level-21 cells; a coarser cell is occupied iff one of them lies in it
    q = np.stack([u >> 42, (u >> 21) & QMAX, u & QMAX], 1)
    return np.array([len(np.unique(cell_keys(q, L))) for L in range(LEVELS)], np.int64)


def key_hash(keys: np.ndarray, seed: int) -> np.ndarray:
    with np.errstate(over="ignore"):
        return splitmix(U64(seed & (2 ** 64 - 1)) + (keys.astype(U64) + U64(1)) * GOLDEN)


def subsample(xyz, S: int, seed: int = 0):
    """(idx [S] int64, ascending then -1; stats [4] int64 = (valid, L*, n_L*, kept)) of psam_voxel_subsample_f32."""
    q, valid = quantize(xyz)
    counts = level_counts(xyz)
    above = np.flatnonzero(counts >= S)
    Ls = int(above[0]) if len(above) else LEVELS - 1
    pts = np.flatnonzero(valid)
    keys = cell_keys(q[pts], Ls)
    e = centre_dist(q[pts], Ls)
    order = np.lexsort((pts, e, keys))  # by key, then (e, index)
    first = np.ones(len(order), bool)
    first[1:] = keys[order][1:] != keys[order][:-1]
    rep, rkey = pts[order][first], keys[order][first]
    n = len(rep)
    if n > S:
        keep = np.lexsort((rkey, key_hash(rkey, seed)))[:S]
        rep = rep[keep]
    out = np.full(S, -1, np.int64)
    out[:len(rep)] = np.sort(rep)
    return out, np.array([int(valid.sum()), Ls, n, min(S, n)], np.int64)
