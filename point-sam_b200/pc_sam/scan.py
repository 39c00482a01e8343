"""Dense scans: segment a LiDAR sweep, an indoor scan or a photogrammetry cloud of 10^6 - 10^8 points with a model whose
input is about 10^4 points, and carry the masks and part labels back to every scan point.  Every step runs on the GPU:

* ``voxel_subsample`` one point per occupied voxel of the coarsest octree level with at least S voxels (the point nearest
  the voxel's centre), thinned to S by a seeded hash of the voxel (``psam_voxel_subsample_f32``).  Deterministic: the
  samples depend only on the coordinates, S and the seed.
* the nearest sample of every scan point comes from the exact grid search ``psam_nn_grid_f32`` (bit for bit the
  brute-force search, at a fraction of its cost), and masks and labels are lifted as for meshes (``pc_sam.mesh``).

``ScanSegmenter`` ties these to a model (``PointCloudSAM`` or ``PointCloudSAMHier``, through its public API): one
subsample, encode and nearest-sample search per scan, then prompted masks or segment-everything with per-point masks and
labels.  Points with a non-finite coordinate are invalid: they are in no mask and get label -1.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from psam_b200 import ops

from .mesh import _SampleSegmenter, nearest_samples
from .utils.ply import read_ply


def voxel_subsample(xyz: torch.Tensor, num_points: int, *, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """At most num_points of the points xyz [P, 3] (a CUDA tensor, normalised coordinates): (index [S'] int64 ascending,
    stats [4] int64 = (valid points, octree level, occupied voxels at that level, S')).  Reads the statistics once."""
    if num_points < 1:
        raise ValueError(f"num_points must be >= 1, got {num_points}")
    idx, stats = ops.voxel_subsample(xyz, int(num_points), seed)
    st = stats.tolist()  # the one host synchronisation
    return idx[: st[3]], stats


def scan_from_ply(path) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """(xyz [P, 3] float32, rgb [P, 3] float32 in 0..1 or None) of a binary PLY point cloud; colours come from red / green /
    blue or R / G / B properties (uchar, or float already in 0..1)."""
    data = read_ply(path)
    names = data.dtype.names
    xyz = np.stack([data["x"], data["y"], data["z"]], axis=1).astype(np.float32)
    for cols in (("red", "green", "blue"), ("R", "G", "B")):
        if all(c in names for c in cols):
            rgb = np.stack([data[c] for c in cols], axis=1)
            if np.issubdtype(rgb.dtype, np.integer):
                return xyz, rgb.astype(np.float32) / np.float32(255)
            return xyz, rgb.astype(np.float32)
    return xyz, None


class ScanSegmenter(_SampleSegmenter):
    """Segment a dense scan with a Point-SAM model: the scan is normalised over its valid points (mean at the origin,
    farthest valid point at distance 1), voxel-subsampled to at most num_points samples that are encoded once, and masks
    over the samples are carried to every scan point through its nearest sample."""

    _setter = "set_scan"

    def __init__(self, model, num_points: int = 32768, seed: int = 0):
        super().__init__(model, num_points, seed)
        self.sample_index = None

    @property
    def point_nearest(self) -> torch.Tensor:
        return self.targets["point"]

    def set_scan(self, xyz, rgb=None):
        """xyz [P, 3] and optional rgb [P, 3] in 0..1 (numpy arrays or CUDA tensors).  Normalises on the device in float64,
        subsamples, encodes the samples (model.set_pointcloud; rgb 0.5 without colour) and finds the nearest sample of every
        point.  The host synchronises once, for one read of the sample count, the subsample's statistics, the shift and
        the scale.  ValueError when no point is valid or the subsample has fewer points than the model's patches."""
        dev = next(self.model.parameters()).device
        x = xyz if torch.is_tensor(xyz) else torch.from_numpy(np.ascontiguousarray(xyz, dtype=np.float32))
        x = x.to(dev).reshape(-1, 3).float()
        if x.shape[0] == 0:
            raise ValueError("the scan has no point")
        x64 = x.double()
        valid = torch.isfinite(x).all(dim=1)
        n = valid.sum()
        shift = torch.where(valid[:, None], x64, 0.0).sum(0) / n
        d = torch.where(valid, (x64 - shift).norm(dim=1), 0.0)
        scale = d.max()
        safe = torch.where(scale > 0, scale, 1.0)
        xn = torch.where(valid[:, None], (x64 - shift) / safe, float("nan")).float().contiguous()
        idx, stats = ops.voxel_subsample(xn, self.num_points, self.seed)
        g = idx.clamp(min=0)
        xs = xn.index_select(0, g)
        if rgb is None:
            cs = torch.full_like(xs, 0.5)
        else:
            c = rgb if torch.is_tensor(rgb) else torch.from_numpy(np.ascontiguousarray(rgb, dtype=np.float32))
            cs = c.to(dev).reshape(-1, 3).float().index_select(0, g)
        head = torch.cat([stats.double(), shift, scale.reshape(1)]).tolist()  # the one host synchronisation
        valid_n, count = int(head[0]), int(head[3])
        if valid_n == 0:
            raise ValueError("the scan has no point with finite coordinates")
        patches = self.model._group_shape()[0]
        if count < patches:
            raise ValueError(f"the subsample has {count} points, fewer than the model's {patches} patches")
        self.shift, self.scale = np.asarray(head[4:7], np.float64), float(head[7])
        self.stats = stats
        self.points = xn
        self.sample_index = idx[:count]
        self.xyz, self.rgb = xs[:count][None].contiguous(), cs[:count][None].contiguous()
        self.model.set_pointcloud(self.xyz, self.rgb)
        self.targets = dict(point=nearest_samples(self.xyz[0], xn))

    def predict_masks(self, prompt_points, prompt_labels, prompt_mask=None, multimask_output: bool = True) -> Dict[str, torch.Tensor]:
        """Prompted masks: prompt_points [Q, 3] in scan coordinates, prompt_labels [Q] (1 foreground, 0 background),
        prompt_mask [1, S] logits over the samples or None.  Returns logits [C, S] and scores [C] over the samples, and
        point_logits [C, P]: each point takes its nearest sample's logits, an invalid point -inf."""
        return super().predict_masks(prompt_points, prompt_labels, prompt_mask, multimask_output)

    def lift_packed(self, out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """generate_packed's output over the samples with the per-point masks and labels added (see generate_packed).
        Nothing here waits for the device."""
        return super().lift_packed(out)

    def _extras(self) -> Dict:
        return dict(sample_index=self.sample_index, shift=self.shift, scale=self.scale)

    def generate_packed(self, generator, **kwargs) -> Dict[str, torch.Tensor]:
        """PointCloudMaskGenerator.generate_packed on the samples (keywords such as min_mask_region_area and the crop_*
        parameters are passed through unchanged), plus
          point_bits [K, ceil(P/32)] int32 and point_area [K] int32: each mask carried to the scan points through their
            nearest sample (an invalid point is in no mask),
          sample_labels [S] int32: the label map over the samples with priority = area (the smallest mask containing a
            sample wins, ties to the earlier mask; -1 in none),
          point_labels [P] int32: the label of each point's nearest sample, -1 for an invalid point,
          sample_index [S] int64: the scan index of each sample,
          shift [3] and scale: normalised = (scan - shift) / scale.
        The lifting and the labels add no host synchronisation to the generator's own."""
        return super().generate_packed(generator, **kwargs)
