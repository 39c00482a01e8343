"""Mesh segmentation: sample points on a mesh's surface, segment them, and carry the masks back to every vertex and face.

Upstream Point-SAM segments a mesh by sampling a point cloud from it, segmenting the cloud and mapping the labels back to
the mesh.  Here every step runs on the GPU:

* ``sample_surface``  area-weighted surface samples (``psam_mesh_sample_f32``): faces are chosen in proportion to their
  area through an exact integer CDF, points are placed with the barycentric rule of the upstream browser demo, and the
  colour comes from vertex colours or from a texture (nearest texel).  The samples depend only on the mesh and the seed.
* ``nearest_samples`` the nearest sample of every target point (``psam_nn_grid_f32``: exact, ties to the lower index, bit
  for bit the brute-force ``psam_nn_distance_f32``).
* ``lift_masks``      bit-packed masks over the samples carried to the targets through their nearest sample (``psam_mask_lift``).
* ``mask_labels``     one part label per point: the smallest mask containing it (``psam_mask_label_map``).

The same lifting serves scans denser than the model's input: ``pc_sam.scan.ScanSegmenter`` subsamples, segments and lifts.

``MeshSegmenter`` ties these to a model (``PointCloudSAM`` or ``PointCloudSAMHier``, through its public API only): one
sampling, encode and nearest-sample search per mesh, then prompted masks (``predict_masks``) or segment-everything
(``generate_packed``) with per-vertex and per-face masks and labels.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from psam_b200 import ops

from .utils.ply import normalize_points, read_ply


def sample_surface(vertices: torch.Tensor, faces: torch.Tensor, num_points: int, *, seed: int = 0,
                   vertex_colors: Optional[torch.Tensor] = None, uv: Optional[torch.Tensor] = None,
                   texture: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """num_points area-weighted samples of a triangle mesh: vertices [V, 3], faces [F, 3] (int32 or int64 vertex indices),
    optional vertex_colors [V, 3] (0..1) or uv [V, 2] with texture [H, W, 3 or 4] uint8, all CUDA tensors.
    Returns (xyz [S, 3], rgb [S, 3] in 0..1 (0.5 without a colour source), face_index [S] int32) on the device.
    Reads the sampler's statistics once: ValueError when a face has a vertex index outside [0, V) or the mesh has no area.
    Faces of zero or non-finite area, and faces smaller than 2^-32 of the largest, are never sampled."""
    if (uv is None) != (texture is None):
        raise ValueError("uv and texture go together")
    if texture is not None and vertex_colors is not None:
        raise ValueError("give vertex_colors or uv + texture, not both")
    if num_points < 1:
        raise ValueError(f"num_points must be >= 1, got {num_points}")
    xyz, rgb, face, stats = ops.mesh_sample(vertices, faces, int(num_points), seed, vertex_colors, uv, texture)
    total, _, bad_index = stats.tolist()  # the one host synchronisation
    if bad_index:
        raise ValueError(f"{bad_index} faces have a vertex index outside [0, {vertices.reshape(-1, 3).shape[0]})")
    if total == 0:
        raise ValueError("the mesh has no face of positive finite area")
    return xyz, rgb, face


def nearest_samples(sample_xyz: torch.Tensor, target_xyz: torch.Tensor) -> torch.Tensor:
    """Index of the nearest sample of every target point (exact squared distance, ties to the lower index): int64 [M].
    A target with a NaN coordinate gets -1, which lift_masks reads as "in no mask"."""
    return ops.nearest_grid(target_xyz, sample_xyz)[1]


def lift_masks(bits: torch.Tensor, nearest: torch.Tensor, S: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Masks over S samples (bits [K, ceil(S/32)] int32) carried to M targets through nearest [M]: (bits [K, ceil(M/32)]
    int32, area [K] int32).  Target t is in mask k when its nearest sample is."""
    return ops.mask_lift(bits, nearest, S)


def mask_labels(bits: torch.Tensor, priority: torch.Tensor, N: int) -> torch.Tensor:
    """One label per point of N: the mask (row of bits [K, ceil(N/32)]) containing it with the smallest priority [K], ties to
    the lower row, -1 in none.  priority = area gives the smallest part containing each point."""
    return ops.mask_label_map(bits, priority, N)


def mesh_from_ply(path) -> Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]:
    """(vertices [V, 3] float32, faces [F, 3] int32, vertex_colors [V, 3] float32 in 0..1 or None) of a binary PLY mesh
    (read_ply(triangular_mesh=True)); vertex colours come from uchar red / green / blue properties."""
    data, faces = read_ply(path, triangular_mesh=True)
    names = data.dtype.names
    vertices = np.stack([data["x"], data["y"], data["z"]], axis=1).astype(np.float32)
    colors = None
    if all(c in names for c in ("red", "green", "blue")):
        colors = np.stack([data["red"], data["green"], data["blue"]], axis=1).astype(np.float32) / np.float32(255)
    return vertices, faces, colors


def _host(x, dtype) -> Optional[np.ndarray]:
    if x is None:
        return None
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=dtype)


class _SampleSegmenter:
    """What MeshSegmenter and ScanSegmenter share: a model encoded once on S samples (self.xyz / self.rgb [1, S, 3]), and
    named sets of target points, each carried by the index of its nearest sample (-1: no sample, so in no mask).
    Subclasses set self.shift / self.scale (normalised = (x - shift) / scale) and self.targets = {name: nearest [M] int64}."""

    def __init__(self, model, num_points: int, seed: int):
        if num_points < 1:
            raise ValueError(f"num_points must be >= 1, got {num_points}")
        self.model = model
        self.num_points = int(num_points)
        self.seed = int(seed)
        self.xyz = self.rgb = None
        self.targets: Dict[str, torch.Tensor] = {}

    def _require(self):
        if self.xyz is None:
            raise RuntimeError(f"call {self._setter}() first")

    def normalize(self, points) -> np.ndarray:
        """Points in input coordinates -> the normalised coordinates of the samples (float64 on the host, then float32)."""
        self._require()
        return ((_host(points, np.float64) - self.shift) / self.scale).astype(np.float32)

    @staticmethod
    def _gather(x: torch.Tensor, near: torch.Tensor, dim: int, fill):
        """x gathered along dim through near; entries with near < 0 take `fill`."""
        got = x.index_select(dim, near.clamp(min=0))
        miss = (near < 0).view([-1 if d == dim else 1 for d in range(x.dim())])
        return got.masked_fill(miss, fill)

    def predict_masks(self, prompt_points, prompt_labels, prompt_mask=None, multimask_output: bool = True) -> Dict[str, torch.Tensor]:
        self._require()
        dev = self.xyz.device
        pts = torch.from_numpy(self.normalize(np.asarray(_host(prompt_points, np.float64)).reshape(-1, 3))).to(dev)[None]
        labels = torch.from_numpy(_host(prompt_labels, np.int64).reshape(1, -1)).to(dev)
        logits, scores, _ = self.model.predict_masks(pts, labels, prompt_mask, multimask_output)
        logits, scores = logits[0], scores[0]
        out = dict(logits=logits, scores=scores)
        for name, near in self.targets.items():
            out[f"{name}_logits"] = self._gather(logits, near, 1, float("-inf"))
        return out

    def lift_packed(self, out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        self._require()
        S = self.xyz.shape[1]
        bits, area = out["bits"], out["area"]
        res = dict(out)
        for name, near in self.targets.items():
            res[f"{name}_bits"], res[f"{name}_area"] = lift_masks(bits, near, S)
        labels = mask_labels(bits, area, S)
        res["sample_labels"] = labels
        for name, near in self.targets.items():
            res[f"{name}_labels"] = self._gather(labels, near, 0, -1)
        res.update(self._extras())
        return res

    def _extras(self) -> Dict:
        return dict(shift=self.shift, scale=self.scale)

    def generate_packed(self, generator, **kwargs) -> Dict[str, torch.Tensor]:
        self._require()
        return self.lift_packed(generator.generate_packed(self.xyz, self.rgb, **kwargs))


class MeshSegmenter(_SampleSegmenter):
    """Segment a triangle mesh with a Point-SAM model: the mesh is normalised (centroid at the origin, farthest vertex at
    distance 1), num_points samples of its surface are encoded once, and masks over the samples are carried to every vertex
    and face through their nearest sample (a face through its centre)."""

    _setter = "set_mesh"

    def __init__(self, model, num_points: int = 32768, seed: int = 0):
        super().__init__(model, num_points, seed)
        self.face_index = None

    @property
    def vertex_nearest(self) -> torch.Tensor:
        return self.targets["vertex"]

    @property
    def face_nearest(self) -> torch.Tensor:
        return self.targets["face"]

    def set_mesh(self, vertices, faces, vertex_colors=None, uv=None, texture=None):
        """vertices [V, 3], faces [F, 3] and the optional colour sources of sample_surface (numpy arrays or tensors).  Samples
        the surface, encodes the samples (model.set_pointcloud) and finds the nearest sample of every vertex and face centre.
        The host synchronises once, to read the sampler's statistics."""
        v = _host(vertices, np.float64)
        if v.ndim != 2 or v.shape[1] != 3 or len(v) == 0:
            raise ValueError(f"vertices must be [V, 3], got {v.shape}")
        if not np.isfinite(v).all():
            raise ValueError("vertices must be finite")
        shift = v.mean(axis=0)
        scale = float(np.max(np.linalg.norm(v - shift, ord=2, axis=1)))
        if not scale > 0:
            raise ValueError("the mesh's vertices all coincide")
        dev = next(self.model.parameters()).device
        vn = torch.from_numpy(normalize_points(v).astype(np.float32)).to(dev)
        f = torch.from_numpy(_host(faces, np.int64).reshape(-1, 3).astype(np.int32)).to(dev)
        up = lambda x, dt: None if x is None else torch.from_numpy(np.ascontiguousarray(_host(x, dt))).to(dev)  # noqa: E731
        xyz, rgb, face = sample_surface(vn, f, self.num_points, seed=self.seed, vertex_colors=up(vertex_colors, np.float32),
                                        uv=up(uv, np.float32), texture=up(texture, np.uint8))
        self.shift, self.scale = shift, scale
        self.vertices, self.faces = vn, f
        self.xyz, self.rgb, self.face_index = xyz[None], rgb[None], face
        self.model.set_pointcloud(self.xyz, self.rgb)
        self.face_centers = ops.mesh_face_centers(vn, f)
        self.targets = dict(vertex=nearest_samples(xyz, vn), face=nearest_samples(xyz, self.face_centers))

    def predict_masks(self, prompt_points, prompt_labels, prompt_mask=None, multimask_output: bool = True) -> Dict[str, torch.Tensor]:
        """Prompted masks: prompt_points [P, 3] in mesh coordinates, prompt_labels [P] (1 foreground, 0 background),
        prompt_mask [1, S] logits over the samples or None.  Returns logits [C, S] and scores [C] over the samples, and
        vertex_logits [C, V] / face_logits [C, F], each element taking its nearest sample's logits."""
        return super().predict_masks(prompt_points, prompt_labels, prompt_mask, multimask_output)

    def lift_packed(self, out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """generate_packed's output over the samples, with the masks and labels of the vertices and faces added (see
        generate_packed).  Nothing here waits for the device."""
        return super().lift_packed(out)

    def generate_packed(self, generator, **kwargs) -> Dict[str, torch.Tensor]:
        """PointCloudMaskGenerator.generate_packed on the samples (keywords such as min_mask_region_area and the crop_*
        parameters are passed through unchanged), plus
          vertex_bits [K, ceil(V/32)] / face_bits [K, ceil(F/32)] int32 and vertex_area / face_area [K] int32: each mask
            carried to the vertices and faces through their nearest sample,
          sample_labels [S] int32: the label map over the samples with priority = area (the smallest mask containing a
            sample wins, ties to the earlier mask; -1 in none),
          vertex_labels [V] / face_labels [F] int32: the label of each element's nearest sample,
          shift [3] and scale: normalised = (mesh - shift) / scale.
        The lifting and the labels add no host synchronisation to the generator's own."""
        return super().generate_packed(generator, **kwargs)
