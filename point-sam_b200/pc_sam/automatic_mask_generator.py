"""Automatic mask generation ("segment everything") for one point cloud: the point-cloud counterpart of segment-anything's
``SamAutomaticMaskGenerator``.

1. Encode the cloud once (``model._encode``).
2. Pick ``points_per_cloud`` prompt points by farthest-point sampling - the point-cloud analogue of SAM's regular grid -
   each a single positive click.
3. Decode them in batches of ``points_per_batch`` with ``multimask_output=True`` (``model._decode_unchecked``); every
   batch reuses the encoder output and the interpolation weights cached on its ``AuxInputs``.
4. After each batch, ``psam_mask_candidates_f32`` bit-packs the masks, computes areas and stability scores and applies
   the predicted-IoU / stability / area filters.
5. ``psam_mask_nms`` removes duplicates by greedy mask-IoU NMS over all candidates of the cloud.
6. With ``min_mask_region_area > 0`` (SAM's post-processing): ``psam_knn_f32`` builds the cloud's kNN graph,
   ``psam_mask_regions`` fills small holes of every kept mask and removes its small islands (connected components of that
   graph), rescores the masks (1 unchanged, 0 changed) and ``psam_mask_nms`` runs again on the result.

Everything runs on the GPU, and the only host synchronisation is the final read of the number of kept masks.  The
default thresholds are SAM's; they are not tuned for Point-SAM.

Memory: each batch of Z = points_per_batch prompts decodes Z rows of N points.  The split-bf16 input of the last
upscaling Linear is Z*N*Du*4 bytes (Du = 256 for PointCloudSAM, 128 for PointCloudSAMHier): about 2 GB at Z = 64,
N = 32768, Du = 256.  Lower points_per_batch to trade speed for memory.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from psam_b200 import engine, ops


class PointCloudMaskGenerator:
    """Segment every part / object of a point cloud without prompts.

    Parameters (names and defaults are SAM's, except that ``points_per_side`` becomes ``points_per_cloud`` and box NMS
    becomes mask NMS):
      points_per_cloud        prompt points per cloud, chosen by farthest-point sampling (at most N are used)
      points_per_batch        prompts decoded together
      pred_iou_thresh         keep masks with predicted IoU > this (filter off when <= 0)
      stability_score_thresh  keep masks with stability score >= this (filter off when <= 0)
      stability_score_offset  logit offset of the stability score: count(logit > +off) / count(logit > -off)
      mask_nms_thresh         drop a mask whose IoU with a higher-scoring kept mask is > this
      min_mask_area           keep masks of at least this many points (an empty mask is never kept)
    generate / generate_packed take SAM's min_mask_region_area as a keyword (default 0: off).
    The model must be in eval mode.  The candidate count points_per_cloud * 3 is limited to 16384."""

    mask_threshold = 0.0  # a point is in the mask when its logit is > 0 (as in predict_masks' callers)
    # neighbours per point of the kNN graph that defines connectivity for min_mask_region_area (the analogue of SAM's
    # 8-connected pixel grid); the graph is undirected, so a point's degree can be higher
    region_neighbors = 8

    def __init__(self, model, points_per_cloud: int = 1024, points_per_batch: int = 64, pred_iou_thresh: float = 0.88,
                 stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0, mask_nms_thresh: float = 0.7,
                 min_mask_area: int = 0):
        if points_per_cloud < 1 or points_per_batch < 1:
            raise ValueError("points_per_cloud and points_per_batch must be >= 1")
        if points_per_cloud * 3 > ops.NMS_MAX_CANDIDATES:
            raise ValueError(f"points_per_cloud * 3 must be <= {ops.NMS_MAX_CANDIDATES}")
        self.model = model
        self.points_per_cloud = int(points_per_cloud)
        self.points_per_batch = int(points_per_batch)
        self.pred_iou_thresh = float(pred_iou_thresh)
        self.stability_score_thresh = float(stability_score_thresh)
        self.stability_score_offset = float(stability_score_offset)
        self.mask_nms_thresh = float(mask_nms_thresh)
        self.min_mask_area = int(min_mask_area)

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _cloud(t: torch.Tensor, name: str) -> torch.Tensor:
        if t.dim() == 2:
            t = t.unsqueeze(0)
        if t.dim() != 3 or t.shape[0] != 1 or t.shape[2] != 3:
            raise ValueError(f"{name} must be [N, 3] or [1, N, 3] (one cloud per call), got {tuple(t.shape)}")
        return t.float().contiguous()

    def _enqueue(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0) -> Dict[str, torch.Tensor]:
        """Enqueue the whole generation on the current stream; nothing here waits for the device."""
        if min_mask_region_area < 0:
            raise ValueError(f"min_mask_region_area must be >= 0, got {min_mask_region_area}")
        region_area = int(min_mask_region_area)
        m = self.model
        if m.training:
            raise NotImplementedError("psam_b200 is an inference-only path: call model.eval() before generating masks")
        xyz, rgb = self._cloud(xyz, "xyz"), self._cloud(rgb, "rgb")
        if xyz.shape[1] != rgb.shape[1]:
            raise ValueError("xyz and rgb must have the same number of points")
        dev, N = xyz.device, xyz.shape[1]
        P, Bp = min(self.points_per_cloud, N), self.points_per_batch
        with torch.no_grad():
            enc = m._encode(xyz, rgb)
            point_index, centers = ops.fps(xyz, P)
            labels = torch.ones((min(Bp, P), 1), dtype=torch.int64, device=dev)
            cand, C = None, None
            for s in range(0, P, Bp):
                e = min(P, s + Bp)
                masks, iou = m._decode_unchecked(enc, centers[0, s:e].unsqueeze(1), labels[: e - s], None, True)
                if cand is None:
                    C = masks.shape[1]
                    K = P * C
                    cand = (torch.empty((K, ops.mask_words(N)), dtype=torch.int32, device=dev),
                            torch.empty(K, dtype=torch.int32, device=dev), torch.empty(K, dtype=torch.float32, device=dev),
                            torch.empty(K, dtype=torch.float32, device=dev))
                ops.mask_candidates(masks, iou, mask_threshold=self.mask_threshold,
                                    stability_offset=self.stability_score_offset, pred_iou_thresh=self.pred_iou_thresh,
                                    stability_thresh=self.stability_score_thresh, min_area=self.min_mask_area, out=cand,
                                    base=s * C)
            bits, area, stab, score = cand
            keep, keep_count = ops.mask_nms(bits, area, score, self.mask_nms_thresh)
            st = dict(bits=bits, area=area, stability=stab, score=score, keep=keep, keep_count=keep_count,
                      point_index=point_index[0], centers=centers[0], slots=C, device=dev)
            if region_area > 0:
                nbr, _ = ops.knn(xyz, xyz, min(self.region_neighbors + 1, N))
                rbits, rarea, rscore = ops.mask_regions(bits, keep, keep_count, nbr, region_area)
                rkeep, rcount = ops.mask_nms(rbits, rarea, rscore, self.mask_nms_thresh)
                st.update(region_bits=rbits, region_area=rarea, region_score=rscore, region_keep=rkeep, region_count=rcount)
        return st

    @staticmethod
    def _finish(st: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """The single host synchronisation: read the kept count together with the out-of-range flag of the prompt
        encoder, then select the kept candidates (on the device).  After the small-region stage the count is the second
        NMS's, its keep list holds ranks of the first, and bits / area come from the post-processed masks."""
        flag = engine.bad_flag(st["device"])
        regions = "region_keep" in st
        n, bad = (int(v) for v in torch.cat([st["region_count" if regions else "keep_count"], flag]).tolist())
        if bad:
            flag.zero_()
            raise ValueError("Input coordinates must be normalized to [-1, 1].")
        if regions:
            rank = st["region_keep"][:n].long()
            sel = st["keep"][rank].long()
            bits, area = st["region_bits"][rank], st["region_area"][rank]
        else:
            sel = st["keep"][:n].long()
            bits, area = st["bits"][sel], st["area"][sel]
        z = torch.div(sel, st["slots"], rounding_mode="floor")
        return dict(bits=bits, area=area, predicted_iou=st["score"][sel],
                    stability_score=st["stability"][sel], point_index=st["point_index"][z], point_coords=st["centers"][z],
                    mask_slot=sel - z * st["slots"])

    def generate_packed(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0) -> Dict[str, torch.Tensor]:
        """Masks of one cloud as device tensors (K = number of kept masks, W = ceil(N / 32)):
        bits [K, W] int32 (point n is bit n % 32 of word n // 32), area [K] int32, predicted_iou [K], stability_score [K],
        point_index [K] int64 (index of the prompt point in the cloud), point_coords [K, 3], mask_slot [K] (0..2: which
        of the three multimask outputs).  xyz / rgb: [N, 3] or [1, N, 3] CUDA tensors, xyz normalised to [-1, 1].

        min_mask_region_area = 0: the masks are in score order (predicted IoU descending).
        min_mask_region_area = A > 0 (SAM's post-processing; connectivity = the kNN graph with ``region_neighbors``
        neighbours per point): every kept mask gets its holes of fewer than A points filled and its islands of fewer than
        A points removed (if no island reaches A, the largest stays), and mask NMS runs again on the results with
        unchanged masks ranked before changed ones (ties in the first order).  So the order is: unchanged masks, then
        changed ones, each in score order.  bits and area are the post-processed ones; predicted_iou and
        stability_score stay the model's."""
        return self._finish(self._enqueue(xyz, rgb, min_mask_region_area=min_mask_region_area))

    def generate(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0) -> List[Dict]:
        """SAM's record list, in the order of generate_packed: segmentation (bool [N] numpy), area, predicted_iou,
        stability_score, point_coords ([[x, y, z]]), point_index."""
        N = self._cloud(xyz, "xyz").shape[1]
        out = {k: v.cpu().numpy() for k, v in self.generate_packed(xyz, rgb, min_mask_region_area=min_mask_region_area).items()}
        seg = np.unpackbits(out["bits"].astype("<i4").view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
        return [dict(segmentation=seg[i], area=int(out["area"][i]), predicted_iou=float(out["predicted_iou"][i]),
                     stability_score=float(out["stability_score"][i]), point_coords=[out["point_coords"][i].tolist()],
                     point_index=int(out["point_index"][i])) for i in range(len(seg))]
