"""Deterministic synthetic inputs.  Shared by bench.py, the tests and the golden-vector
generator (through oracle/synth.py); pure CPU torch so that every box produces identical tensors."""
from __future__ import annotations

import torch


def make_cloud(n: int, seed: int = 0, cloud_id: int = 0, kind: str = "ball"):
    """xyz [n,3] uniform in the unit ball then reference-normalised (eval_kitti.py:82-88),
    features [n,3] in [-1,1]."""
    g = torch.Generator().manual_seed(seed + cloud_id)
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    r = torch.rand(n, generator=g) ** (1.0 / 3.0)
    xyz = d * r[:, None]
    if kind == "kitti":
        xyz = xyz * torch.tensor([1.0, 1.0, 0.15])
        k = int(0.4 * n)
        xyz[:k, 2] = xyz[:, 2].min()
    elif kind == "grid":  # tie-heavy: quantised to a 1/64 grid with duplicated points
        xyz = torch.round(xyz * 16) / 16
        xyz[n // 2:] = xyz[: n - n // 2].clone()
    xyz = xyz - xyz.mean(dim=0, keepdim=True)
    xyz = xyz / xyz.norm(dim=1).max()
    feats = torch.rand(n, 3, generator=g) * 2 - 1
    return xyz.float().contiguous(), feats.float().contiguous()


def make_batch(b: int, n: int, seed: int = 0, kind: str = "ball"):
    xs, fs = zip(*[make_cloud(n, seed, i, kind) for i in range(b)])
    return torch.stack(xs), torch.stack(fs)


def make_prompts(xyz: torch.Tensor, num_prompts: int, seed: int = 0):
    """prompt p of cloud b = xyz[b, (seed*7919 + 104729*p) mod N]; labels 1,0,1,0..."""
    B, N, _ = xyz.shape
    idx = torch.tensor([(seed * 7919 + 104729 * p) % N for p in range(num_prompts)])
    coords = xyz[:, idx]
    labels = torch.tensor([1 - (p % 2) for p in range(num_prompts)]).expand(B, -1).contiguous()
    return coords.contiguous(), labels


def make_region_masks(xyz: torch.Tensor, num_masks: int = 1) -> torch.Tensor:
    """Ground-truth masks [B, M, N] bool for the evaluation loop (config c3): mask m of cloud b = the points within
    0.45 + 0.05 m of point 997 (m + 1) - a compact region with a border, as the GT prompt sampler requires."""
    B, N, _ = xyz.shape
    return torch.stack([torch.stack([(xyz[b] - xyz[b, (997 * (m + 1)) % N]).norm(dim=-1) < 0.45 + 0.05 * m
                                     for m in range(num_masks)]) for b in range(B)])


def make_sphere(n_lat: int, n_lon: int, center=(0.0, 0.0, 0.0), radius: float = 1.0):
    """A closed UV sphere: (vertices [2 + (n_lat - 1) n_lon, 3] float32, faces [2 n_lon (n_lat - 1), 3] int32)."""
    import numpy as np

    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    ring = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.sin(th), np.sin(ph)), np.repeat(np.cos(th)[:, None], n_lon, 1)], -1)
    v = np.concatenate([[[0, 0, 1]], ring.reshape(-1, 3), [[0, 0, -1]]]) * radius + np.asarray(center)
    i, j = np.meshgrid(np.arange(n_lat - 2), np.arange(n_lon), indexing="ij")
    r = lambda i, j: 1 + i * n_lon + j % n_lon  # noqa: E731
    band = np.stack([np.stack([r(i, j), r(i + 1, j), r(i + 1, j + 1)], -1), np.stack([r(i, j), r(i + 1, j + 1), r(i, j + 1)], -1)], 2)
    jj = np.arange(n_lon)
    last = len(v) - 1
    cap0 = np.stack([np.zeros(n_lon, int), r(0, jj), r(0, jj + 1)], -1)
    cap1 = np.stack([r(n_lat - 2, jj), np.full(n_lon, last), r(n_lat - 2, jj + 1)], -1)
    f = np.concatenate([cap0, band.reshape(-1, 3), cap1])
    return v.astype(np.float32), f.astype(np.int32)


def make_box(n: int, center=(0.0, 0.0, 0.0), half=(1.0, 1.0, 1.0)):
    """The surface of an axis-aligned box, each side an n x n grid of quads split in two: 12 n^2 faces (the sides do not share
    their edge vertices)."""
    import numpy as np

    t = np.linspace(-1, 1, n + 1)
    a, b = np.meshgrid(t, t, indexing="ij")
    q = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    quad = np.stack([q[:-1, :-1], q[1:, :-1], q[1:, 1:], q[:-1, 1:]], -1).reshape(-1, 4)
    tri = np.concatenate([quad[:, [0, 1, 2]], quad[:, [0, 2, 3]]])
    vs, fs = [], []
    for axis in range(3):
        for side in (-1.0, 1.0):
            p = np.zeros(((n + 1) ** 2, 3))
            u, w = [k for k in range(3) if k != axis]
            p[:, axis], p[:, u], p[:, w] = side, a.ravel(), b.ravel()
            fs.append((tri if side > 0 else tri[:, ::-1]) + sum(len(x) for x in vs))
            vs.append(p)
    v = np.concatenate(vs) * np.asarray(half) + np.asarray(center)
    return v.astype(np.float32), np.concatenate(fs).astype(np.int32)


def make_mesh(num_faces: int, seed: int = 0):
    """A scene of four spheres and four boxes of random sizes and positions with about num_faces faces in all:
    (vertices float32, faces int32, vertex_colors float32 in 0..1, one colour per object)."""
    import numpy as np

    rng = np.random.default_rng(seed)
    k = max(3, int(round((num_faces / 16) ** 0.5)))   # a sphere of k x k has about 2 k^2 faces
    n = max(1, int(round((num_faces / 96) ** 0.5)))    # a box of n has 12 n^2 faces
    vs, fs, cs, base = [], [], [], 0
    for o in range(8):
        c = rng.uniform(-2, 2, 3)
        v, f = make_sphere(k, k, c, rng.uniform(0.3, 1.0)) if o % 2 == 0 else make_box(n, c, rng.uniform(0.2, 0.8, 3))
        vs.append(v)
        fs.append(f + base)
        cs.append(np.tile(rng.uniform(0, 1, 3), (len(v), 1)))
        base += len(v)
    return np.concatenate(vs), np.concatenate(fs), np.concatenate(cs).astype(np.float32)


def make_scan(P: int, seed: int = 0):
    """A LiDAR-like scan of P points over the make_mesh scene (about 20k faces): (xyz [P, 3] float32, rgb [P, 3] float32 in
    0..1).  Points are surface samples kept with probability falling off as 1 / (1 + (r / 2)^2) with the distance r from a
    sensor at (0, 0, 3), so the density falls with range; a few rows are NaN and a few are far outliers (up to 50 times the
    scene's size)."""
    import numpy as np

    rng = np.random.default_rng(seed)
    v, f, col = make_mesh(20000, seed)
    a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
    area = 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)
    cdf = np.cumsum(area) / area.sum()
    sensor = np.array([0.0, 0.0, 3.0])
    out_xyz, out_rgb, n = [], [], 0
    while n < P:
        m = max(2 * (P - n), 1024)
        face = np.minimum(np.searchsorted(cdf, rng.random(m)), len(f) - 1)
        r1, r2 = np.sqrt(rng.random(m))[:, None], rng.random(m)[:, None]
        p = (1 - r1) * a[face] + r1 * (1 - r2) * b[face] + r1 * r2 * c[face]
        r = np.linalg.norm(p - sensor, axis=1)
        keep = rng.random(m) < 1.0 / (1.0 + (r / 2.0) ** 2)
        out_xyz.append(p[keep])
        out_rgb.append(col[f[face[keep], 0]])
        n += int(keep.sum())
    xyz = np.concatenate(out_xyz)[:P].astype(np.float32)
    rgb = np.concatenate(out_rgb)[:P].astype(np.float32)
    k = max(1, P // 10000)
    rows = rng.choice(P, min(P, 2 * k), replace=False)
    xyz[rows[:k], rng.integers(0, 3, len(rows[:k]))] = np.nan
    xyz[rows[k:]] = rng.uniform(-1, 1, (len(rows[k:]), 3)).astype(np.float32) * np.float32(200)
    return xyz, rgb
