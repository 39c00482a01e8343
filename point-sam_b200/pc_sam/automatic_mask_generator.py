"""Automatic mask generation ("segment everything") for a point cloud or a batch of clouds: the point-cloud counterpart of
segment-anything's ``SamAutomaticMaskGenerator``.

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

Batches of clouds (``generate_packed_batch`` / ``generate_batch``, B clouds of the same N): one encode and one FPS call for
all B clouds; each decode batch covers the same prompt range of every cloud (``plan_decode``), and every candidate, NMS and
small-region launch covers all B clouds, each owning a block of ``points_per_cloud * 3`` candidate slots.  One host read
covers all B kept counts.  Generation on one cloud is the case B = 1 of the same code.

Clouds of different sizes (a sequence of [N_b, 3] tensors) run the same path on a padded batch [B, N_max, 3] with lengths
[B] on the device (``ops.pad_clouds``).  Farthest-point sampling, the kNN searches, the candidate pass and the small-region
pass stay inside each cloud's own points, so every cloud gets generate_packed's masks; cloud b uses min(points_per_cloud,
N_b) prompts as generate_packed does (its other prompt slots score -inf).  Everything between the tokenizer and the mask
dot sees G patches per cloud or independent point rows, and the decoder also computes logits for the padded rows: that
cost grows with B * N_max - sum(N_b).  Group clouds of similar sizes to keep it small.

Crop layers (keyword ``crop_n_layers > 0``, SAM's zoomed crops for large scenes): ``psam_crop_layout_f32`` splits the cloud's
bounding box into 2^i x 2^i x 2^i overlapping boxes on layer i and counts their points; the host reads the counts once.
Layer 0 runs steps 1-5 on the cloud as given.  Every other crop with at least as many points as the tokenizer's first-level
groups (and a box unlike an earlier one of its layer) is gathered and renormalised by ``psam_crop_gather_f32``, runs steps
1-5 with ``points_per_cloud // crop_n_points_downscale_factor^i`` prompts, and, before its NMS, drops the candidates that
touch an interior face of the crop (``psam_crop_edge_filter``).  ``psam_crop_uncrop`` lifts every crop's kept masks to the
whole cloud, and ``psam_mask_nms`` with score = layer and ``crop_nms_thresh`` merges them (smaller crops win).  Step 6
then runs on the merged set.  The host synchronises twice: the counts, and the final read.

Crop layers on a batch of clouds (``generate_packed_batch_crops`` / ``generate_batch_crops``): ``psam_crop_layout_batched_f32``
lays out every cloud's crops at once and the host reads all counts once; layer 0 runs on the B clouds as above; the crops of
each deeper layer, pooled over the clouds, are sorted by size and cut into padded crop batches (``plan_eval_batches``: at
most points_per_batch crops and DECODE_MAX_ROW_TILES * DECODE_ROW_TILE padded points each), and each batch is one
``psam_crop_gather_batched_f32``, steps 1-4 on the padded batch, one ``psam_crop_edge_filter_batched`` and the batched NMS.
One ``psam_crop_uncrop_batched`` lifts every crop into its cloud's set in the cloud's crop order, and the NMS across crops
and step 6 run per cloud in single launches.  The host synchronises twice per call.  Every crop's candidates are held until
the uncrop: 3P * ceil(n/32) * 4 bytes per crop of n points with P prompts (about 23 MB at P = 1024, n = 60000).  The
decoder also computes logits for the padded crop rows, so batching pays off when the encodes it merges outweigh the
padding: 1.12x on 8 clouds of 10000-30000 points with 256 prompts, but 0.88x (slower) on 2 scene-scale clouds of 131072
points with 1024 prompts (DESIGN.md).

Memory: each batch of Z = points_per_batch prompts decodes Z rows of N points (with B clouds, points_per_batch // B
prompts of each cloud; N = N_max for clouds of different sizes).  The split-bf16 input of the last upscaling Linear is Z*N*Du*4 bytes (Du = 256 for PointCloudSAM, 128 for PointCloudSAMHier): about 2 GB at Z = 64,
N = 32768, Du = 256.  Lower points_per_batch to trade speed for memory.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from psam_b200 import engine, ops
from psam_b200.parallel import plan_eval_batches


# the decoder's upscaling GEMM runs on B * Zc * N rows in tiles of DECODE_ROW_TILE, and its grid holds at most
# DECODE_MAX_ROW_TILES of them
DECODE_ROW_TILE, DECODE_MAX_ROW_TILES = 128, 65535


class DecodePlan(NamedTuple):
    rows: int                       # Zc: prompts of each cloud per decode batch
    batches: List[Tuple[int, int]]  # the prompt range [s, e) of every cloud, one entry per decode batch


def plan_decode(B: int, P: int, N: int, points_per_batch: int) -> DecodePlan:
    """Decode batches for B clouds of N points (N_max for a padded batch of clouds of different sizes) with P prompts each.  A batch covers prompts [s, e) of every cloud, row
    b * (e - s) + j of the decoder for prompt s + j of cloud b.  Zc = max(1, points_per_batch // B) keeps points_per_batch
    rows per batch (the memory bound of the module docstring); the last batch may be short.  Raises ValueError when even
    one prompt per cloud needs more than DECODE_MAX_ROW_TILES row tiles (ceil(B * N / 128)): fewer clouds per call fit."""
    if B < 1 or P < 1 or N < 1 or points_per_batch < 1:
        raise ValueError(f"plan_decode: B, P, N and points_per_batch must be >= 1, got {B}, {P}, {N}, {points_per_batch}")
    tiles = -(-B * N // DECODE_ROW_TILE)
    if tiles > DECODE_MAX_ROW_TILES:
        raise ValueError(f"{B} clouds of {N} points need {tiles} row tiles in the decoder even with one prompt per cloud, at "
                         f"most {DECODE_MAX_ROW_TILES}: generate fewer clouds per call")
    Zc = max(1, points_per_batch // B)
    return DecodePlan(Zc, [(s, min(P, s + Zc)) for s in range(0, P, Zc)])


class CropArgs(NamedTuple):
    n_layers: int
    nms_thresh: float
    overlap_ratio: float
    downscale: int


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
      crop_n_layers           crop layers (0: off; at most 3): layer i splits each axis of the bounding box into 2^i crops
      crop_nms_thresh         mask-IoU threshold of the NMS across crops
      crop_overlap_ratio      overlap of neighbouring crops, as a fraction of the bounding box extent per crop count (< 1)
      crop_n_points_downscale_factor  layer i uses points_per_cloud // factor^i prompts per crop
    generate / generate_packed take SAM's min_mask_region_area and the four crop_* parameters above as keywords, with
    SAM's defaults (min_mask_region_area = 0 and crop_n_layers = 0: off).
    The model must be in eval mode.  The candidate count points_per_cloud * 3 is limited to 16384, and with crop layers
    the kept masks of all crops together as well (ValueError at the final read)."""

    mask_threshold = 0.0  # a point is in the mask when its logit is > 0 (as in predict_masks' callers)
    # neighbours per point of the kNN graph that defines connectivity for min_mask_region_area (the analogue of SAM's
    # 8-connected pixel grid); the graph is undirected, so a point's degree can be higher
    region_neighbors = 8
    # a crop's candidate is dropped when it holds a point within this fraction of the bounding box extent of an interior
    # face of the crop (SAM's is_box_near_crop_edge, atol = 20 pixels)
    crop_edge_margin = 0.02

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

    @staticmethod
    def _clouds(t: torch.Tensor, name: str) -> torch.Tensor:
        if t.dim() != 3 or t.shape[0] < 1 or t.shape[2] != 3:
            raise ValueError(f"{name} must be [B, N, 3], got {tuple(t.shape)}")
        return t.float().contiguous()

    @staticmethod
    def _cloud_state(st: Dict, b: int) -> Dict:
        """Cloud b of a batched state: every per-cloud tensor indexed by b, the counts kept as one-element tensors."""
        per_cloud = ("bits", "area", "stability", "score", "keep", "point_index", "centers", "region_bits", "region_area",
                     "region_score", "region_keep")
        return {k: (v[b] if k in per_cloud else v[b:b + 1] if k in ("keep_count", "region_count") else v) for k, v in st.items()}

    def _generate_batch(self, xyz: torch.Tensor, rgb: torch.Tensor, P: int, edge=None,
                        lengths: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Generation on B clouds [B, N, 3] (whole clouds, or one crop's renormalised cloud, B = 1): one encode, P FPS
        prompts per cloud, multimask decode in the batches of plan_decode with one candidate launch each, the crop's edge
        filter when `edge` is given ([W] for one crop, B = 1; [B, W] for a padded batch of crops, one launch), mask NMS per
        cloud in one go.  Cloud b owns candidate slots b * P * C .. of
        bits [B, P*C, W]; keep [B, P*C] holds slots within the cloud, keep_count [B].  lengths [B] (device): padded clouds,
        cloud b's first lengths[b] points with min(P, lengths[b]) prompts."""
        m, dev, (B, N, _) = self.model, xyz.device, xyz.shape
        plan = plan_decode(B, P, N, self.points_per_batch)
        enc = m._encode(xyz, rgb) if lengths is None else m._encode(xyz, rgb, lengths)
        point_index, centers = ops.fps(xyz, P, lengths=lengths)
        labels = torch.ones((B * plan.rows, 1), dtype=torch.int64, device=dev)
        cand, C = None, None
        for s, e in plan.batches:
            rows = B * (e - s)
            masks, iou = m._decode_unchecked(enc, centers[:, s:e].reshape(rows, 1, 3), labels[:rows], None, True)
            if cand is None:
                C = masks.shape[1]
                K = P * C
                cand = (torch.empty((B, K, ops.mask_words(N)), dtype=torch.int32, device=dev),
                        torch.empty((B, K), dtype=torch.int32, device=dev), torch.empty((B, K), dtype=torch.float32, device=dev),
                        torch.empty((B, K), dtype=torch.float32, device=dev))
            ops.mask_candidates_batched(masks, iou, B, mask_threshold=self.mask_threshold,
                                        stability_offset=self.stability_score_offset, pred_iou_thresh=self.pred_iou_thresh,
                                        stability_thresh=self.stability_score_thresh, min_area=self.min_mask_area, out=cand,
                                        base=s * C, lengths=lengths, num_prompts=P)
        bits, area, stab, score = cand
        if edge is not None and edge.dim() == 1:
            ops.crop_edge_filter(bits[0], score[0], edge)
        elif edge is not None:
            ops.crop_edge_filter_batched(bits, score, edge)
        keep, keep_count = ops.mask_nms_batched(bits, area, score, self.mask_nms_thresh)
        return dict(bits=bits, area=area, stability=stab, score=score, keep=keep, keep_count=keep_count,
                    point_index=point_index, centers=centers, slots=C, device=dev)

    def _generate_one(self, xyz: torch.Tensor, rgb: torch.Tensor, P: int, edge=None) -> Dict[str, torch.Tensor]:
        """_generate_batch on one cloud [1, N, 3], as that cloud's state (bits [K, W], keep [K], keep_count [1], ...)."""
        return self._cloud_state(self._generate_batch(xyz, rgb, P, edge), 0)

    def _regions(self, xyz: torch.Tensor, bits: torch.Tensor, keep: torch.Tensor, keep_count: torch.Tensor,
                 area: int, lengths: Optional[torch.Tensor] = None, min_points: int = 0) -> Dict[str, torch.Tensor]:
        """The small-region stage on B clouds xyz [B, N, 3]: kept masks keep [B, K] (keep_count [B]) of bits [B, K', W];
        one kNN launch, one region launch, then mask NMS per cloud in one go.  lengths [B] (device): padded clouds, the
        smallest of min_points points."""
        k1 = min(self.region_neighbors + 1, xyz.shape[1] if lengths is None else min_points)
        nbr, _ = ops.knn(xyz, xyz, k1, lengths=lengths)
        rbits, rarea, rscore = ops.mask_regions_batched(bits, keep, keep_count, nbr, area, lengths=lengths)
        rkeep, rcount = ops.mask_nms_batched(rbits, rarea, rscore, self.mask_nms_thresh)
        return dict(region_bits=rbits, region_area=rarea, region_score=rscore, region_keep=rkeep, region_count=rcount)

    @staticmethod
    def _crop_args(crop_n_layers, crop_nms_thresh, crop_overlap_ratio, crop_n_points_downscale_factor) -> CropArgs:
        if not 0 <= crop_n_layers <= ops.CROP_MAX_LAYERS:
            raise ValueError(f"crop_n_layers must be in 0..{ops.CROP_MAX_LAYERS}, got {crop_n_layers}")
        if not 0 <= crop_overlap_ratio < 1:
            raise ValueError(f"crop_overlap_ratio must be in [0, 1), got {crop_overlap_ratio}")
        if crop_n_points_downscale_factor < 1:
            raise ValueError(f"crop_n_points_downscale_factor must be >= 1, got {crop_n_points_downscale_factor}")
        if not 0 <= crop_nms_thresh <= 1:
            raise ValueError(f"crop_nms_thresh must be in [0, 1], got {crop_nms_thresh}")
        return CropArgs(int(crop_n_layers), float(crop_nms_thresh), float(crop_overlap_ratio), int(crop_n_points_downscale_factor))

    def _crop_prompts(self, factor: int, layer: int, count: int) -> int:
        return min(max(1, self.points_per_cloud // factor ** layer), count)

    def _enqueue_crops(self, xyz: torch.Tensor, rgb: torch.Tensor, crop: CropArgs, keep_states: bool) -> Dict[str, torch.Tensor]:
        """Crop layers: the layout, one host read of the crop point counts, generation per crop (layer 0 = the cloud as
        given), every crop's kept masks lifted to the cloud, then mask NMS across crops (score = layer).  st["crops"] lists
        the crops that ran (crop, layer, points, prompts); with keep_states, also each crop's generation state (candidates,
        keep list, FPS prompts) and its global point indices, which otherwise are freed as soon as the crop is lifted."""
        dev, N = xyz.device, xyz.shape[1]
        boxes, counts = ops.crop_layout(xyz, crop.n_layers, crop.overlap_ratio)
        counts_h = counts.tolist()  # the first of the two host synchronisations
        min_points = self.model._group_shape()[0]
        runs, first, n = [(0, 0, N)], 1, 8  # (crop, layer, points)
        for layer in range(1, crop.n_layers + 1):
            runs += [(t, layer, counts_h[t]) for t in range(first, first + n) if counts_h[t] >= min_points]
            first, n = first + n, n * 8
        crops, lifted = [], None
        offsets = torch.zeros(len(runs) + 1, dtype=torch.int32, device=dev)
        overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        for k, (t, layer, count) in enumerate(runs):
            P = self._crop_prompts(crop.downscale, layer, count)
            if layer == 0:
                idx = torch.arange(N, dtype=torch.int32, device=dev)
                cs = self._generate_one(xyz, rgb, P)
            else:
                idx, cx, cr, edge = ops.crop_gather(xyz, rgb, boxes, t, count, self.crop_edge_margin)
                cs = self._generate_one(cx, cr, P, edge)
            if lifted is None:
                C = cs["slots"]
                cap = min(ops.NMS_MAX_CANDIDATES, C * sum(self._crop_prompts(crop.downscale, l, c) for _, l, c in runs))
                W = ops.mask_words(N)
                lifted = (torch.empty((cap, W), dtype=torch.int32, device=dev), torch.empty(cap, dtype=torch.int32, device=dev),
                          torch.empty(cap, dtype=torch.float32, device=dev), torch.empty(cap, dtype=torch.float32, device=dev),
                          torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, dtype=torch.int32, device=dev),
                          torch.empty(cap, dtype=torch.int32, device=dev),
                          torch.full((cap,), float("-inf"), dtype=torch.float32, device=dev))
            ops.crop_uncrop((cs["bits"], cs["area"], cs["stability"], cs["score"]), cs["keep"], cs["keep_count"], idx,
                            cs["point_index"], cs["slots"], t, float(layer), offsets, k, lifted, overflow, N)
            info = dict(crop=t, layer=layer, points=count, prompts=P)
            crops.append(dict(cs, idx=idx, **info) if keep_states else info)
        gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore = lifted
        if len(runs) > 1:
            keep, keep_count = ops.mask_nms(gbits, garea, gscore, crop.nms_thresh)
        else:
            keep = torch.arange(gbits.shape[0], dtype=torch.int32, device=dev)
            keep_count = torch.clamp(offsets[1:], max=gbits.shape[0])
        return dict(bits=gbits, area=garea, score=giou, stability=gstab, keep=keep, keep_count=keep_count, prompt=gprompt,
                    mask_slot=gslot, crop=gcrop, crop_score=gscore, crop_boxes=boxes, crop_counts=counts, crops=crops,
                    overflow=overflow, lifted_count=offsets[-1:], xyz=xyz[0], device=dev)

    def _enqueue_crops_batch(self, xyz: torch.Tensor, rgb: torch.Tensor, crop: CropArgs, sizes: List[int],
                             lengths: Optional[torch.Tensor], keep_states: bool) -> Dict[str, torch.Tensor]:
        """_enqueue_crops on B clouds [B, N, 3] (lengths [B] on the device for a padded batch, sizes on the host): the
        batched layout, one host read of every cloud's crop counts, layer 0 as _generate_batch on the B clouds, the crops of
        every deeper layer pooled over the clouds and cut into padded crop batches (plan_eval_batches: sorted by size, at most
        points_per_batch crops and DECODE_MAX_ROW_TILES * DECODE_ROW_TILE padded points per batch), each gathered in one
        batched launch pair and run through _generate_batch with the batched edge filter; then one batched uncrop of every
        crop into its cloud's lifted set [B, cap, W] (crop order within the cloud) and the merge NMS per cloud.  A cloud on
        which only layer 0 ran keeps every lifted mask, as _enqueue_crops does.  st["crops"][b] lists cloud b's crops (with
        keep_states, also their gathered clouds and generation states); st["crop_batches"] lists (layer, pairs, n_max) of
        every crop batch."""
        dev, (B, N, _) = xyz.device, xyz.shape
        boxes, counts = ops.crop_layout_batched(xyz, crop.n_layers, crop.overlap_ratio, lengths)
        counts_h = counts.tolist()  # the first of the two host synchronisations
        min_points = self.model._group_shape()[0]
        runs = []  # per cloud: (crop, layer, points), in crop order
        for b in range(B):
            r, first, n = [(0, 0, sizes[b])], 1, 8
            for layer in range(1, crop.n_layers + 1):
                r += [(t, layer, counts_h[b][t]) for t in range(first, first + n) if counts_h[b][t] >= min_points]
                first, n = first + n, n * 8
            runs.append(r)
        state: Dict[Tuple[int, int], Dict] = {}  # (cloud, crop) -> the crop's generation state, held until the uncrop

        def add(b, t, layer, cs, i, idx, extra):
            state[b, t] = dict(cand=(cs["bits"][i], cs["area"][i], cs["stability"][i], cs["score"][i]), keep=cs["keep"][i],
                               keep_count=cs["keep_count"][i:i + 1], idx=idx, prompt_index=cs["point_index"][i], slots=cs["slots"],
                               crop=t, layer=layer, cloud=b, **extra)

        s0 = self._generate_batch(xyz, rgb, min(self.points_per_cloud, N), lengths=lengths)
        arange = torch.arange(N, dtype=torch.int32, device=dev)
        for b in range(B):
            add(b, 0, 0, s0, b, arange[:sizes[b]], {})
        crop_batches = []
        for layer in range(1, crop.n_layers + 1):
            pool = [(b, t, c) for b in range(B) for t, lay, c in runs[b] if lay == layer]
            P = max(1, self.points_per_cloud // crop.downscale ** layer)
            for batch in plan_eval_batches([c for _, _, c in pool], [layer] * len(pool), self.points_per_batch,
                                           DECODE_MAX_ROW_TILES * DECODE_ROW_TILE):
                pairs = [pool[i] for i in batch]
                n_max = max(c for _, _, c in pairs)
                idx, cx, cr, edge, clen = ops.crop_gather_batched(xyz, rgb, boxes, pairs, self.crop_edge_margin, lengths)
                cs = self._generate_batch(cx, cr, min(P, n_max), edge=edge, lengths=clen)
                for i, (b, t, c) in enumerate(pairs):
                    extra = dict(xyz=cx[i, :c], rgb=cr[i, :c], edge=edge[i, :ops.mask_words(c)]) if keep_states else {}
                    add(b, t, layer, cs, i, idx[i, :c], extra)
                crop_batches.append((layer, pairs, n_max))
        C = s0["slots"]
        caps = [min(ops.NMS_MAX_CANDIDATES, C * sum(self._crop_prompts(crop.downscale, lay, c) for _, lay, c in r)) for r in runs]
        cap, W = max(caps), ops.mask_words(N)
        lifted = (torch.empty((B, cap, W), dtype=torch.int32, device=dev), torch.empty((B, cap), dtype=torch.int32, device=dev),
                  torch.empty((B, cap), dtype=torch.float32, device=dev), torch.empty((B, cap), dtype=torch.float32, device=dev),
                  torch.empty((B, cap), dtype=torch.int64, device=dev), torch.empty((B, cap), dtype=torch.int32, device=dev),
                  torch.empty((B, cap), dtype=torch.int32, device=dev),
                  torch.full((B, cap), float("-inf"), dtype=torch.float32, device=dev))
        order = [dict(state[b, t], capacity=caps[b]) for b in range(B) for t, _, _ in runs[b]]
        lifted_count, overflow = ops.crop_uncrop_batched(order, lifted, N)
        gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore = lifted
        if any(len(r) > 1 for r in runs):
            keep, keep_count = ops.mask_nms_batched(gbits, garea, gscore, crop.nms_thresh)
        else:
            keep, keep_count = torch.empty((B, cap), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev)
        for b in range(B):
            if len(runs[b]) == 1:  # only layer 0 ran: no merge
                keep[b].copy_(arange[:cap] if cap <= N else torch.arange(cap, dtype=torch.int32, device=dev))
                keep_count[b:b + 1] = torch.clamp(lifted_count[b:b + 1], max=caps[b])
        crops = []
        for b in range(B):
            crops.append([])
            for t, lay, c in runs[b]:
                info = dict(crop=t, layer=lay, points=c, prompts=self._crop_prompts(crop.downscale, lay, c))
                if keep_states:
                    s = state[b, t]
                    bits, area, stab, score = s["cand"]
                    info.update({k: v for k, v in s.items() if k not in ("cand", "crop", "layer", "cloud", "prompt_index")},
                                bits=bits, area=area, stability=stab, score=score, point_index=s["prompt_index"])
                crops[b].append(info)
        return dict(bits=gbits, area=garea, score=giou, stability=gstab, keep=keep, keep_count=keep_count, prompt=gprompt,
                    mask_slot=gslot, crop=gcrop, crop_score=gscore, crop_boxes=boxes, crop_counts=counts, crops=crops,
                    crop_batches=crop_batches, capacity=caps, overflow=overflow, lifted_count=lifted_count, xyz=xyz, device=dev)

    @staticmethod
    def _region_area(min_mask_region_area: int) -> int:
        if min_mask_region_area < 0:
            raise ValueError(f"min_mask_region_area must be >= 0, got {min_mask_region_area}")
        return int(min_mask_region_area)

    def _check_model(self):
        if self.model.training:
            raise NotImplementedError("psam_b200 is an inference-only path: call model.eval() before generating masks")

    @staticmethod
    def _same_points(xyz: torch.Tensor, rgb: torch.Tensor):
        if xyz.shape[:2] != rgb.shape[:2]:
            raise ValueError("xyz and rgb must have the same number of clouds and points")

    def _enqueue_clouds(self, xyz: torch.Tensor, rgb: torch.Tensor, region_area: int, lengths: Optional[torch.Tensor] = None,
                        sizes: Optional[List[int]] = None) -> Dict[str, torch.Tensor]:
        """Generation and (region_area > 0) the small-region stage on B validated clouds [B, N, 3], batched state.  lengths
        (device) and sizes (host): a padded batch of clouds of N_b = sizes[b] points."""
        with torch.no_grad():
            st = self._generate_batch(xyz, rgb, min(self.points_per_cloud, xyz.shape[1]), lengths=lengths)
            if region_area > 0:
                st.update(self._regions(xyz, st["bits"], st["keep"], st["keep_count"], region_area, lengths=lengths,
                                        min_points=min(sizes) if sizes else 0))
        if sizes is not None:
            st["sizes"] = sizes
        return st

    def _enqueue(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0, crop_n_layers: int = 0,
                 crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                 crop_n_points_downscale_factor: int = 1, keep_crop_states: bool = False) -> Dict[str, torch.Tensor]:
        """Enqueue the whole generation of one cloud on the current stream.  Without crop layers nothing here waits for the
        device (it is cloud 0 of _enqueue_batch); with them, the crop point counts are read once.  keep_crop_states keeps
        every crop's generation state in st["crops"] (for inspection; it holds each crop's candidate masks until the state
        is dropped)."""
        region_area = self._region_area(min_mask_region_area)
        crop = self._crop_args(crop_n_layers, crop_nms_thresh, crop_overlap_ratio, crop_n_points_downscale_factor)
        self._check_model()
        xyz, rgb = self._cloud(xyz, "xyz"), self._cloud(rgb, "rgb")
        self._same_points(xyz, rgb)
        if crop.n_layers == 0:
            return self._cloud_state(self._enqueue_clouds(xyz, rgb, region_area), 0)
        with torch.no_grad():
            st = self._enqueue_crops(xyz, rgb, crop, keep_crop_states)
            if region_area > 0:
                st.update(self._cloud_state(self._regions(xyz, st["bits"][None], st["keep"][None], st["keep_count"], region_area), 0))
        return st

    def _enqueue_batch(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]], *,
                       min_mask_region_area: int = 0) -> Dict[str, torch.Tensor]:
        """Enqueue the generation of B clouds [B, N, 3], or of a sequence of B clouds [N_b, 3] as one padded batch, on the
        current stream; nothing here waits for the device."""
        region_area = self._region_area(min_mask_region_area)
        self._check_model()
        xyz, rgb, sizes, lengths = self._batch_clouds(xyz, rgb)
        return self._enqueue_clouds(xyz, rgb, region_area, lengths, sizes)

    def _batch_clouds(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]],
                      padded_checks: bool = False) -> Tuple[torch.Tensor, torch.Tensor, Optional[List[int]], Optional[torch.Tensor]]:
        """The checked batch of a batched call: (xyz, rgb [B, N, 3], sizes, lengths).  [B, N, 3] tensors give sizes = None
        (padded_checks: the checks of varlen_clouds all the same, and sizes = [N] * B) and lengths = None; sequences of
        [N_b, 3] clouds are checked by varlen_clouds and padded (ops.pad_clouds, lengths on the device)."""
        if torch.is_tensor(xyz):
            xyz, rgb = self._clouds(xyz, "xyz"), self._clouds(rgb, "rgb")
            self._same_points(xyz, rgb)
            return xyz, rgb, self.model.varlen_clouds(list(xyz), list(rgb)) if padded_checks else None, None
        if torch.is_tensor(rgb):
            raise ValueError("xyz and rgb must both be [B, N, 3] tensors or both sequences of [N_b, 3] tensors")
        sizes = self.model.varlen_clouds(xyz, rgb)
        if any(t.shape[1] != 3 for t in rgb):
            raise ValueError("rgb must hold [N_b, 3] tensors")
        xyz, rgb, lengths = ops.pad_clouds(xyz, rgb)
        return xyz, rgb, sizes, lengths

    def _enqueue_batch_crops(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]],
                             *, min_mask_region_area: int = 0, crop_n_layers: int = 1, crop_nms_thresh: float = 0.7,
                             crop_overlap_ratio: float = 512 / 1500, crop_n_points_downscale_factor: int = 1,
                             keep_crop_states: bool = False) -> Dict[str, torch.Tensor]:
        """Enqueue generate_packed_batch_crops on the current stream: the keywords are checked first, then the model and the
        clouds.  crop_n_layers = 0 is _enqueue_batch; otherwise the crop counts are read once (_enqueue_crops_batch).  Crop
        batches are padded batches of clouds of different sizes, so the checks of varlen_clouds apply to every input."""
        region_area = self._region_area(min_mask_region_area)
        crop = self._crop_args(crop_n_layers, crop_nms_thresh, crop_overlap_ratio, crop_n_points_downscale_factor)
        self._check_model()
        if crop.n_layers == 0:
            return self._enqueue_batch(xyz, rgb, min_mask_region_area=region_area)
        xyz, rgb, sizes, lengths = self._batch_clouds(xyz, rgb, padded_checks=True)
        with torch.no_grad():
            st = self._enqueue_crops_batch(xyz, rgb, crop, sizes, lengths, keep_crop_states)
            if region_area > 0:
                st.update(self._regions(xyz, st["bits"], st["keep"], st["keep_count"], region_area, lengths=lengths,
                                        min_points=min(sizes)))
        st["sizes"] = sizes
        return st

    @staticmethod
    def _read_counts(st: Dict[str, torch.Tensor]) -> List[int]:
        """The single host synchronisation: every cloud's kept count (after the small-region stage, the second NMS's), read
        together with the out-of-range flag of the prompt encoder and, with crop layers, the overflow flag."""
        flag = engine.bad_flag(st["device"])
        counts = st["region_count" if "region_keep" in st else "keep_count"]
        crops = "crops" in st
        vals = [int(v) for v in torch.cat([counts, flag] + ([st["overflow"]] if crops else [])).tolist()]
        B = counts.numel()
        if vals[B]:
            flag.zero_()
            raise ValueError("Input coordinates must be normalized to [-1, 1].")
        if crops and vals[B + 1]:
            raise ValueError(f"crop layers: the kept masks of all crops exceed the {st['bits'].shape[0]} lifted slots; "
                             "lower points_per_cloud or crop_n_layers, or raise crop_n_points_downscale_factor")
        return vals[:B]

    @staticmethod
    def _select(st: Dict[str, torch.Tensor], n: int) -> Dict[str, torch.Tensor]:
        """The n kept masks of one cloud's state, selected on the device.  After the small-region stage the keep list is the
        second NMS's and holds ranks of the first, and bits / area come from the post-processed masks."""
        regions, crops = "region_keep" in st, "crops" in st
        if regions:
            rank = st["region_keep"][:n].long()
            sel = st["keep"][rank].long()
            bits, area = st["region_bits"][rank], st["region_area"][rank]
        else:
            sel = st["keep"][:n].long()
            bits, area = st["bits"][sel], st["area"][sel]
        if crops:
            prompt = st["prompt"][sel]
            return dict(bits=bits, area=area, predicted_iou=st["score"][sel], stability_score=st["stability"][sel],
                        point_index=prompt, point_coords=st["xyz"][prompt], mask_slot=st["mask_slot"][sel].long(),
                        crop_box=st["crop_boxes"][st["crop"][sel].long()])
        z = torch.div(sel, st["slots"], rounding_mode="floor")
        return dict(bits=bits, area=area, predicted_iou=st["score"][sel],
                    stability_score=st["stability"][sel], point_index=st["point_index"][z], point_coords=st["centers"][z],
                    mask_slot=sel - z * st["slots"])

    @classmethod
    def _finish(cls, st: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """One cloud's output from its state (_enqueue), after the single host synchronisation."""
        (n,) = cls._read_counts(st)
        return cls._select(st, n)

    @classmethod
    def _finish_batch(cls, st: Dict[str, torch.Tensor]) -> List[Dict[str, torch.Tensor]]:
        """Every cloud's output from a batched state (_enqueue_batch), after one host synchronisation for all of them.  The
        masks of a padded batch keep the ceil(N_b / 32) words of their own cloud (the later ones are zero)."""
        outs = [cls._select(cls._cloud_state(st, b), n) for b, n in enumerate(cls._read_counts(st))]
        for out, n in zip(outs, st.get("sizes", ())):
            out["bits"] = out["bits"][:, :ops.mask_words(n)].contiguous()
        return outs

    @classmethod
    def _finish_batch_crops(cls, st: Dict[str, torch.Tensor]) -> List[Dict[str, torch.Tensor]]:
        """Every cloud's output from _enqueue_crops_batch's state after the second host synchronisation, which reads every
        cloud's kept count, the prompt encoder's out-of-range flag and every cloud's overflow flag together."""
        flag = engine.bad_flag(st["device"])
        counts = st["region_count" if "region_keep" in st else "keep_count"]
        B = counts.numel()
        vals = [int(v) for v in torch.cat([counts, flag, st["overflow"]]).tolist()]
        if vals[B]:
            flag.zero_()
            raise ValueError("Input coordinates must be normalized to [-1, 1].")
        over = [b for b in range(B) if vals[B + 1 + b]]
        if over:
            b = over[0]
            raise ValueError(f"crop layers: cloud {b}: the kept masks of its crops exceed its {st['capacity'][b]} lifted slots; "
                             "lower points_per_cloud or crop_n_layers, or raise crop_n_points_downscale_factor")
        per_cloud = ("bits", "area", "score", "stability", "keep", "prompt", "mask_slot", "crop", "crop_score", "crop_boxes", "xyz",
                     "region_bits", "region_area", "region_score", "region_keep")
        outs = []
        for b, n in enumerate(vals[:B]):
            sb = {k: (v[b] if k in per_cloud else v[b:b + 1] if k in ("keep_count", "region_count") else v) for k, v in st.items()}
            out = cls._select(sb, n)
            out["bits"] = out["bits"][:, :ops.mask_words(st["sizes"][b])].contiguous()
            outs.append(out)
        return outs

    def generate_packed(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0, crop_n_layers: int = 0,
                        crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                        crop_n_points_downscale_factor: int = 1) -> Dict[str, torch.Tensor]:
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
        stability_score stay the model's.

        crop_n_layers > 0: the masks of all crops, in global point indices, merged by mask NMS across crops in which masks
        of deeper layers rank first (then by crop, then by score within the crop); min_mask_region_area then applies to
        the merged set.  An extra field crop_box [K, 6] (x0, y0, z0, x1, y1, z1 in the input's coordinates) gives each
        mask's crop; layer 0's box is the bounding box."""
        return self._finish(self._enqueue(xyz, rgb, min_mask_region_area=min_mask_region_area, crop_n_layers=crop_n_layers,
                                          crop_nms_thresh=crop_nms_thresh, crop_overlap_ratio=crop_overlap_ratio,
                                          crop_n_points_downscale_factor=crop_n_points_downscale_factor))

    def generate_packed_batch(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]],
                              *, min_mask_region_area: int = 0) -> List[Dict[str, torch.Tensor]]:
        """generate_packed on B clouds at once: xyz / rgb [B, N, 3] CUDA tensors, or sequences of B CUDA tensors [N_b, 3] for
        clouds of different sizes; xyz normalised to [-1, 1].  Returns B dicts with generate_packed's fields, dtypes, order
        and meaning for each cloud (bits [K, ceil(N_b / 32)]).  The clouds share one encode, the decode batches
        (points_per_batch // B prompts of every cloud each) and every post-processing launch, and the host synchronises
        once for all of them; a cloud outside [-1, 1] raises ValueError for the whole call.  Clouds of different sizes are
        padded to the largest (module docstring): the decoder's work grows with the padding.  For crop layers use
        generate_packed_batch_crops."""
        return self._finish_batch(self._enqueue_batch(xyz, rgb, min_mask_region_area=min_mask_region_area))

    @staticmethod
    def _records(out: Dict[str, torch.Tensor], N: int) -> List[Dict]:
        out = {k: v.cpu().numpy() for k, v in out.items()}
        seg = np.unpackbits(out["bits"].astype("<i4").view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
        recs = [dict(segmentation=seg[i], area=int(out["area"][i]), predicted_iou=float(out["predicted_iou"][i]),
                     stability_score=float(out["stability_score"][i]), point_coords=[out["point_coords"][i].tolist()],
                     point_index=int(out["point_index"][i])) for i in range(len(seg))]
        if "crop_box" in out:
            for r, box in zip(recs, out["crop_box"]):
                r["crop_box"] = box.tolist()
        return recs

    def generate(self, xyz: torch.Tensor, rgb: torch.Tensor, *, min_mask_region_area: int = 0, crop_n_layers: int = 0,
                 crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                 crop_n_points_downscale_factor: int = 1) -> List[Dict]:
        """SAM's record list, in the order of generate_packed: segmentation (bool [N] numpy), area, predicted_iou,
        stability_score, point_coords ([[x, y, z]]), point_index, and crop_box ([x0, y0, z0, x1, y1, z1]) with crop
        layers."""
        N = self._cloud(xyz, "xyz").shape[1]
        return self._records(self.generate_packed(xyz, rgb, min_mask_region_area=min_mask_region_area, crop_n_layers=crop_n_layers,
                                                  crop_nms_thresh=crop_nms_thresh, crop_overlap_ratio=crop_overlap_ratio,
                                                  crop_n_points_downscale_factor=crop_n_points_downscale_factor), N)

    def generate_batch(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]], *,
                       min_mask_region_area: int = 0) -> List[List[Dict]]:
        """generate on B clouds [B, N, 3], or a sequence of clouds [N_b, 3], at once (see generate_packed_batch): one record
        list per cloud, whose segmentations have the cloud's own N_b points."""
        if torch.is_tensor(xyz):
            sizes = [self._clouds(xyz, "xyz").shape[1]] * xyz.shape[0]
        else:
            sizes = [int(t.shape[0]) for t in xyz]
        outs = self.generate_packed_batch(xyz, rgb, min_mask_region_area=min_mask_region_area)
        return [self._records(out, n) for out, n in zip(outs, sizes)]

    def generate_packed_batch_crops(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]],
                                    *, crop_n_layers: int = 1, crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                                    crop_n_points_downscale_factor: int = 1, min_mask_region_area: int = 0) -> List[Dict[str, torch.Tensor]]:
        """generate_packed with crop layers on B clouds at once: xyz / rgb [B, N, 3] CUDA tensors or sequences of B CUDA
        tensors [N_b, 3], xyz normalised to [-1, 1].  Returns B dicts with generate_packed(cloud_b, same keywords)'s fields,
        dtypes, order and meaning, crop_box included (bits [K, ceil(N_b / 32)]).  Per cloud, the crop boxes and counts, the
        crops that run, each crop's gathered cloud and its FPS prompts are generate_packed's bit for bit; what follows the
        encoder equals it up to the rounding of a batched encode (the split-K of the encoder's GEMMs depends on the batch),
        as for generate_packed_batch.  Each cloud's lifted set has generate_packed's capacity and crop order; an overflow
        raises ValueError naming the cloud, and so does a cloud outside [-1, 1] (for the whole call).  The clouds and the
        crops are padded batches (module docstring), so a Voronoi tokenizer is refused (NotImplementedError) and so is a
        cloud smaller than the first-level group shape.  The host synchronises twice per call whatever B is.
        crop_n_layers = 0 is generate_packed_batch.  Speed: the decoder also runs on the padded crop rows, so this is faster
        than generate_packed per cloud on object-scale clouds (1.12x for 8 clouds of 10000-30000 points, 256 prompts) but
        slower on scene-scale ones (0.88x for 2 clouds of 131072 points, 1024 prompts, points_per_batch 32), where decoding
        dominates; the module docstring bounds the memory held for the crops."""
        st = self._enqueue_batch_crops(xyz, rgb, min_mask_region_area=min_mask_region_area, crop_n_layers=crop_n_layers,
                                       crop_nms_thresh=crop_nms_thresh, crop_overlap_ratio=crop_overlap_ratio,
                                       crop_n_points_downscale_factor=crop_n_points_downscale_factor)
        return self._finish_batch_crops(st) if "crops" in st else self._finish_batch(st)

    def generate_batch_crops(self, xyz: Union[torch.Tensor, Sequence[torch.Tensor]], rgb: Union[torch.Tensor, Sequence[torch.Tensor]],
                             *, crop_n_layers: int = 1, crop_nms_thresh: float = 0.7, crop_overlap_ratio: float = 512 / 1500,
                             crop_n_points_downscale_factor: int = 1, min_mask_region_area: int = 0) -> List[List[Dict]]:
        """generate with crop layers on B clouds at once (see generate_packed_batch_crops): one SAM record list per cloud,
        with crop_box when crop_n_layers > 0."""
        if torch.is_tensor(xyz):
            sizes = [self._clouds(xyz, "xyz").shape[1]] * xyz.shape[0]
        else:
            sizes = [int(t.shape[0]) for t in xyz]
        outs = self.generate_packed_batch_crops(xyz, rgb, crop_n_layers=crop_n_layers, crop_nms_thresh=crop_nms_thresh,
                                                crop_overlap_ratio=crop_overlap_ratio,
                                                crop_n_points_downscale_factor=crop_n_points_downscale_factor,
                                                min_mask_region_area=min_mask_region_area)
        return [self._records(out, n) for out, n in zip(outs, sizes)]
