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
