"""ORACLE (test infrastructure, NOT product code): numpy restatement of the mesh kernels of csrc/mesh.cu in the evaluation
order stated in include/psam_b200.h - face weights, the exact integer CDF, the counter-based hash, face choice, the
barycentric point with its clamp, the texel rule, face centres, mask lifting and the label map.  fp32 arithmetic is done
one numpy operation at a time (each rounded on its own, nothing fused); the hash and mulhi use uint64.  Nearest samples
come from oracle.tokenizer_ref.knn(query, key, 1), the exact C kNN with the device's distance and tie rule."""
from __future__ import annotations

import numpy as np

F32 = np.float32
U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)


def twice_area(v: np.ndarray, faces: np.ndarray):
    """(A2 [F] fp32 with 0 for bad faces, bad [F] bool, bad_index [F] bool)."""
    v = np.asarray(v, F32)
    f = np.asarray(faces, np.int64)
    V = len(v)
    bad_index = ((f < 0) | (f >= V)).any(1)
    fi = np.where(bad_index[:, None], 0, f)
    a, b, c = v[fi[:, 0]], v[fi[:, 1]], v[fi[:, 2]]
    with np.errstate(all="ignore"):
        e1, e2 = b - a, c - a
        nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
        ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
        nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
        A = np.sqrt((nx * nx + ny * ny) + nz * nz)
        bad = bad_index | ~(np.isfinite(A) & (A > 0))
    return np.where(bad, F32(0), A).astype(F32), bad, bad_index


def weights(v, faces):
    """(q [F] uint64 fixed-point weights, stats [3] int64 = (total, bad faces, bad-index faces))."""
    A, bad, bad_index = twice_area(v, faces)
    amax = float(A.max()) if len(A) else 0.0
    if amax > 0:
        _, E = np.frexp(amax)  # amax = m * 2^E, m in [0.5, 1): 2^(E-1) <= amax < 2^E
        q = np.floor(A.astype(np.float64) * np.ldexp(1.0, 32 - int(E))).astype(U64)
    else:
        q = np.zeros(len(A), U64)
    assert int(q.max(initial=0)) <= 2 ** 32 - 1
    cdf = np.cumsum(q, dtype=U64)
    stats = np.array([int(cdf[-1]) if len(cdf) else 0, int(bad.sum()), int(bad_index.sum())], np.int64)
    return q, cdf, stats


def splitmix(x: np.ndarray) -> np.ndarray:
    z = np.asarray(x, U64).copy()
    with np.errstate(over="ignore"):
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def hash_stream(seed: int, s: np.ndarray, j: int) -> np.ndarray:
    s = np.asarray(s, U64)
    with np.errstate(over="ignore"):
        return splitmix(U64(seed & (2 ** 64 - 1)) + (U64(3) * s + U64(j + 1)) * GOLDEN)


def mulhi(a: np.ndarray, b: int) -> np.ndarray:
    """High 64 bits of a * b (a uint64 array, b < 2^64), by 32-bit halves."""
    a = np.asarray(a, U64)
    m = U64(0xFFFFFFFF)
    a_lo, a_hi = a & m, a >> U64(32)
    b_lo, b_hi = U64(b & 0xFFFFFFFF), U64(b >> 32)
    with np.errstate(over="ignore"):
        lo_lo = a_lo * b_lo
        hi_lo = a_hi * b_lo
        lo_hi = a_lo * b_hi
        hi_hi = a_hi * b_hi
        cross = (lo_lo >> U64(32)) + (hi_lo & m) + lo_hi
        return hi_hi + (hi_lo >> U64(32)) + (cross >> U64(32))


def _bary(w0, w1, w2, a, b, c):
    return (w0 * a + w1 * b) + w2 * c


def _fmin(a, b):
    """np.fmin with -0.0 ordered below +0.0 (np.fmin returns its second operand when the two compare equal)."""
    zero = (a == 0) & (b == 0)
    return np.where(zero, np.where(np.signbit(a) | np.signbit(b), F32(-0.0), F32(0.0)), np.fmin(a, b)).astype(F32)


def _fmax(a, b):
    """np.fmax with -0.0 ordered below +0.0."""
    zero = (a == 0) & (b == 0)
    return np.where(zero, np.where(np.signbit(a) & np.signbit(b), F32(-0.0), F32(0.0)), np.fmax(a, b)).astype(F32)


def _clamp3(p, a, b, c):
    return _fmin(_fmax(p, _fmin(_fmin(a, b), c)), _fmax(_fmax(a, b), c))


def texel(t: np.ndarray, n: int) -> np.ndarray:
    """floor(t * n + 0.5) in fp32, clamped into 0 .. n - 1; NaN -> 0."""
    with np.errstate(invalid="ignore"):
        x = np.floor(np.asarray(t, F32) * F32(n) + F32(0.5))
        return np.where(x >= F32(n - 1), n - 1, np.where(x > 0, np.nan_to_num(x), 0)).astype(np.int64)


def sample(v, faces, S: int, seed: int = 0, vertex_colors=None, uv=None, texture=None):
    """(xyz [S, 3], rgb [S, 3], face [S] int32, stats [3] int64) of psam_mesh_sample_f32."""
    v = np.asarray(v, F32)
    f = np.asarray(faces, np.int64)
    _, cdf, stats = weights(v, f)
    total = int(stats[0])
    if total == 0:
        return np.zeros((S, 3), F32), np.zeros((S, 3), F32), np.full(S, -1, np.int32), stats
    s = np.arange(S, dtype=U64)
    u = mulhi(hash_stream(seed, s, 0), total)
    face = np.searchsorted(cdf, u, side="right")  # smallest f with cdf[f] > u
    r1 = (hash_stream(seed, s, 1) >> U64(40)).astype(F32) * F32(2.0 ** -24)
    r2 = (hash_stream(seed, s, 2) >> U64(40)).astype(F32) * F32(2.0 ** -24)
    sq = np.sqrt(r1)
    w0, w1, w2 = (F32(1) - sq)[:, None], (sq * (F32(1) - r2))[:, None], (sq * r2)[:, None]
    i0, i1, i2 = f[face, 0], f[face, 1], f[face, 2]
    a, b, c = v[i0], v[i1], v[i2]
    xyz = _clamp3(_bary(w0, w1, w2, a, b, c), a, b, c).astype(F32)
    if texture is not None:
        uvs = np.asarray(uv, F32)
        tex = np.asarray(texture, np.uint8)
        H, W = tex.shape[:2]
        t = _bary(w0, w1, w2, uvs[i0], uvs[i1], uvs[i2])
        x, y = texel(t[:, 0], W), texel(F32(1) - t[:, 1], H)
        rgb = tex[y, x, :3].astype(F32) / F32(255)
    elif vertex_colors is not None:
        vc = np.asarray(vertex_colors, F32)
        rgb = _clamp3(_bary(w0, w1, w2, vc[i0], vc[i1], vc[i2]), vc[i0], vc[i1], vc[i2]).astype(F32)
    else:
        rgb = np.full((S, 3), F32(0.5))
    return xyz, rgb.astype(F32), face.astype(np.int32), stats


def face_centers(v, faces) -> np.ndarray:
    v = np.asarray(v, F32)
    f = np.asarray(faces, np.int64)
    bad = ((f < 0) | (f >= len(v))).any(1)
    fi = np.where(bad[:, None], 0, f)
    c = ((v[fi[:, 0]] + v[fi[:, 1]]) + v[fi[:, 2]]) / F32(3)
    c[bad] = np.nan
    return c.astype(F32)


def unpack(bits: np.ndarray, n: int) -> np.ndarray:
    """[K, W] int32 / uint32 words -> bool [K, n] (point i = bit i % 32 of word i // 32)."""
    b = np.ascontiguousarray(bits).astype("<u4")
    b = b.view(np.uint8).reshape(b.shape[0], b.shape[1] * 4)
    return np.unpackbits(b, axis=1, bitorder="little")[:, :n].astype(bool)


def pack(m: np.ndarray) -> np.ndarray:
    """bool [K, n] -> [K, ceil(n / 32)] uint32."""
    K, n = m.shape
    W = (n + 31) // 32
    pad = np.zeros((K, W * 32), bool)
    pad[:, :n] = m
    return np.packbits(pad, axis=1, bitorder="little").view("<u4").reshape(K, W)


def lift(bits: np.ndarray, nearest: np.ndarray, S: int):
    """(bits [K, ceil(M/32)] uint32, area [K] int32) of psam_mask_lift."""
    near = np.asarray(nearest, np.int64)
    words = np.ascontiguousarray(bits).astype("<u4")
    ok = (near >= 0) & (near < S)
    n = near[ok]
    m = np.zeros((len(words), len(near)), bool)
    m[:, ok] = (words[:, n >> 5] >> (n & 31).astype(np.uint32)) & 1
    return pack(m), m.sum(1).astype(np.int32)


def label_map(bits: np.ndarray, priority: np.ndarray, N: int) -> np.ndarray:
    """labels [N] int32 of psam_mask_label_map: the containing row of smallest (priority, row), -1 for none."""
    K = len(bits)
    out = np.full(N, -1, np.int32)
    if K == 0:
        return out
    m = unpack(bits, N)
    order = sorted(range(K), key=lambda k: (int(priority[k]), k), reverse=True)  # paint the winner last
    for k in order:
        out[m[k]] = k
    return out
