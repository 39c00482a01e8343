"""ORACLE (test infrastructure, NOT product code).

numpy restatement of the crop layers of automatic mask generation (include/psam_b200.h psam_crop_layout_f32 /
psam_crop_gather_f32 / psam_crop_edge_filter / psam_crop_uncrop, the crop_n_layers path of
pc_sam/automatic_mask_generator.py): segment-anything's generate_crop_boxes / is_box_near_crop_edge / uncrop_masks and the
NMS across crops, restated for an axis-aligned bounding box in 3-D.  Every value is fp32 with each operation rounded on its
own, in the header's evaluation order, and every decision is made on exact values, so the device kernels must match this
module bit for bit.  On top of oracle/amg_ref.py and oracle/amg_regions_ref.py.
"""
from __future__ import annotations

import numpy as np

from . import amg_ref, amg_regions_ref

F = np.float32
EDGE_MARGIN = 0.02          # PointCloudMaskGenerator.crop_edge_margin
OVERLAP_RATIO = 512 / 1500  # SAM's default crop_overlap_ratio


def crop_layers(n_layers: int):
    """[(crop, layer, n, (jx, jy, jz))] in crop order."""
    out = []
    for layer in range(n_layers + 1):
        n = 1 << layer
        for q in range(n ** 3):
            out.append((len(out), layer, n, (q // (n * n), (q // n) % n, q % n)))
    return out


def bounding_box(xyz) -> np.ndarray:
    """(lo, hi) per axis over the non-NaN coordinates, -0.0 ordered below +0.0; an all-NaN axis gives (+inf, -inf)."""
    x = np.asarray(xyz, dtype=F).reshape(-1, 3)
    nan = np.isnan(x)
    lo = np.where(nan, F(np.inf), x).min(0, initial=F(np.inf))
    hi = np.where(nan, F(-np.inf), x).max(0, initial=F(-np.inf))
    # ndarray.min / max return either zero when +0.0 and -0.0 meet, depending on the order of the elements
    neg0, pos0 = ((x == 0) & np.signbit(x)).any(0), ((x == 0) & ~np.signbit(x)).any(0)
    lo = np.where(lo == 0, np.where(neg0, F(-0.0), F(0.0)), lo)
    hi = np.where(hi == 0, np.where(pos0, F(0.0), F(-0.0)), hi)
    return np.concatenate([lo, hi]).astype(F)


def axis_bounds(lo, hi, n, j, r):
    """Crop j of n on one axis: ((r * L) * 2) / n, (L + o * (n - 1)) / n, lo + j * (s - o), that + s (last: hi)."""
    lo, hi, r = F(lo), F(hi), F(r)
    L = F(hi - lo)
    o = F(F(F(r * L) * F(2)) / F(n))
    s = F(F(L + F(o * F(n - 1))) / F(n))
    b0 = F(lo + F(F(j) * F(s - o)))
    b1 = hi if j == n - 1 else F(b0 + s)
    return b0, b1


def layout(xyz, n_layers: int, overlap_ratio: float = OVERLAP_RATIO):
    """(boxes [T, 6] fp32, counts [T] int64 with -1 for a box equal to an earlier one of its layer, layer [T])."""
    x = np.asarray(xyz, dtype=F).reshape(-1, 3)
    bb = bounding_box(x)
    crops = crop_layers(n_layers)
    boxes = np.zeros((len(crops), 6), dtype=F)
    for t, _, n, j in crops:
        for a in range(3):
            boxes[t, a], boxes[t, 3 + a] = axis_bounds(bb[a], bb[3 + a], n, j[a], overlap_ratio)
    counts = np.zeros(len(crops), dtype=np.int64)
    layer = np.array([c[1] for c in crops])
    for t, lay, _, _ in crops:
        earlier = np.nonzero((layer[:t] == lay))[0]
        if any(np.array_equal(boxes[u], boxes[t]) for u in earlier):
            counts[t] = -1
        else:
            counts[t] = int(members(x, boxes[t]).sum())
    return boxes, counts, layer


def members(xyz, box) -> np.ndarray:
    """Closed membership lo <= p <= hi on all three axes (a NaN coordinate is in no box)."""
    x = np.asarray(xyz, dtype=F).reshape(-1, 3)
    b = np.asarray(box, dtype=F)
    return np.all((b[:3] <= x) & (x <= b[3:]), axis=1)


def crop_cloud(xyz, rgb, boxes, crop: int, edge_margin: float = EDGE_MARGIN):
    """(idx int64 ascending, xyz [n, 3] renormalised to the box midpoint and the largest distance, rgb [n, 3], edge bool [n])."""
    x = np.asarray(xyz, dtype=F).reshape(-1, 3)
    c = np.asarray(rgb, dtype=F).reshape(-1, 3)
    box, bb = np.asarray(boxes[crop], dtype=F), np.asarray(boxes[0], dtype=F)
    idx = np.nonzero(members(x, box))[0]
    p = x[idx]
    centre = ((box[:3] + box[3:]).astype(F) * F(0.5)).astype(F)
    d = (p - centre).astype(F)
    d2 = ((d[:, 0] * d[:, 0]).astype(F) + (d[:, 1] * d[:, 1]).astype(F)).astype(F) + (d[:, 2] * d[:, 2]).astype(F)
    scale = np.sqrt(d2.astype(F).max()) if len(idx) else F(0)
    scale = F(scale)
    coords = (d / scale).astype(F) if scale > 0 else np.zeros_like(d)
    return idx, coords, c[idx], edge_flags(p, box, bb, edge_margin)


def edge_flags(p, box, bb, edge_margin: float = EDGE_MARGIN) -> np.ndarray:
    """Points within edge_margin * L_a (L_a of the bounding box) of an interior face (a face not on the bounding box)."""
    p = np.asarray(p, dtype=F).reshape(-1, 3)
    near = np.zeros(len(p), dtype=bool)
    for a in range(3):
        m = F(F(edge_margin) * F(bb[3 + a] - bb[a]))
        if box[a] != bb[a]:
            near |= (p[:, a] - box[a]).astype(F) <= m
        if box[3 + a] != bb[3 + a]:
            near |= (box[3 + a] - p[:, a]).astype(F) <= m
    return near


def edge_filter(bits, score, edge_bits) -> np.ndarray:
    """score with -inf where the mask shares a point with the edge bitset."""
    hit = (np.asarray(bits).astype(np.uint32) & np.asarray(edge_bits).astype(np.uint32)[None, :]).any(1)
    return np.where(hit, amg_ref.NEG_INF, np.asarray(score, dtype=F)).astype(F)


def uncrop(local_bits, idx, N: int) -> np.ndarray:
    """Local masks [K, W] of a crop's points -> global masks [K, ceil(N / 32)]."""
    n = len(idx)
    local = amg_ref.unpack_bits(np.asarray(local_bits).astype(np.uint32), n) if len(local_bits) else np.zeros((0, n), bool)
    full = np.zeros((len(local), N), dtype=bool)
    full[:, np.asarray(idx, dtype=np.int64)] = local
    return amg_ref.pack_bits(full)


def merge(per_crop, N: int, crop_nms_thresh: float, capacity: int):
    """Lift every crop's kept masks (in crop order) and merge them.  per_crop: list of dicts with crop, layer, idx, bits,
    area, score, stability, keep (kept slots in NMS order), point_index (crop-local prompt indices), slots.  Returns dict of
    the lifted set (bits, area, iou, stability, prompt, mask_slot, crop, layer_score), overflow, and keep (the NMS across
    crops with score = layer when more than one crop ran, else every lifted mask)."""
    rows = []
    for c in per_crop:
        keep = np.asarray(c["keep"], dtype=np.int64)
        g = uncrop(np.asarray(c["bits"]).astype(np.uint32)[keep], c["idx"], N)
        for r, s in enumerate(keep):
            z = s // c["slots"]
            rows.append(dict(bits=g[r], area=int(c["area"][s]), iou=F(c["score"][s]), stability=F(c["stability"][s]),
                             prompt=int(np.asarray(c["idx"])[c["point_index"][z]]), mask_slot=int(s - z * c["slots"]),
                             crop=int(c["crop"]), layer_score=F(c["layer"])))
    overflow = len(rows) > capacity
    rows = rows[:capacity]
    W = (N + 31) // 32
    out = dict(bits=np.array([r["bits"] for r in rows], dtype=np.uint32).reshape(len(rows), W), overflow=overflow)
    for k, dt in (("area", np.int32), ("iou", F), ("stability", F), ("prompt", np.int64), ("mask_slot", np.int64),
                  ("crop", np.int64), ("layer_score", F)):
        out[k] = np.array([r[k] for r in rows], dtype=dt)
    if len(per_crop) > 1:
        out["keep"] = amg_ref.nms(out["bits"], out["area"], out["layer_score"], crop_nms_thresh)
    else:
        out["keep"] = np.arange(len(rows), dtype=np.int64)
    return out


def prompts(points_per_cloud: int, factor: int, layer: int, count: int) -> int:
    return min(max(1, points_per_cloud // factor ** layer), count)


def generate_ref(model, xyz, rgb, points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.88, stability_score_thresh=0.95,
                 stability_score_offset=1.0, mask_nms_thresh=0.7, min_mask_area=0, min_mask_region_area=0, crop_n_layers=1,
                 crop_nms_thresh=0.7, crop_overlap_ratio=OVERLAP_RATIO, crop_n_points_downscale_factor=1, min_points=None,
                 edge_margin=EDGE_MARGIN):
    """End-to-end fp32 generator with crop layers on the oracle models: amg_ref.generate_ref per crop (layer 0 on the cloud
    as given, other crops on crop_cloud's renormalised cloud) with the edge filter before the crop's NMS, then merge and the
    small-region stage on the merged set.  min_points = the tokenizer's first-level group count.  xyz / rgb [1, N, 3] CPU
    tensors.  Returns dict of boxes, counts, crops (per crop: crop, layer, idx, and amg_ref.generate_ref's fields with
    score / keep after the edge filter), merged (merge's dict), regions (postprocess_small_regions' dict or None) and
    final (indices into the lifted set, in output order)."""
    import torch

    x, c = xyz[0].numpy(), rgb[0].numpy()
    N = x.shape[0]
    boxes, counts, layer = layout(x, crop_n_layers, crop_overlap_ratio)
    runs = [(0, 0)] + [(t, int(layer[t])) for t in range(1, len(boxes)) if counts[t] >= min_points]
    per_crop, C = [], None
    for t, lay in runs:
        if lay == 0:
            idx, cx, cr, edge = np.arange(N), x, c, None
        else:
            idx, cx, cr, edge = crop_cloud(x, c, boxes, t, edge_margin)
        P = prompts(points_per_cloud, crop_n_points_downscale_factor, lay, len(idx))
        r = amg_ref.generate_ref(model, torch.from_numpy(np.ascontiguousarray(cx))[None], torch.from_numpy(np.ascontiguousarray(cr))[None],
                                 P, points_per_batch, pred_iou_thresh, stability_score_thresh, stability_score_offset,
                                 mask_nms_thresh, min_mask_area)
        if edge is not None:
            r["score"] = edge_filter(r["bits"], r["score"], amg_ref.pack_bits(edge[None], r["bits"].shape[1])[0])
            r["keep"] = amg_ref.nms(r["bits"], r["area"], r["score"], mask_nms_thresh)
        C = r["slots"]
        per_crop.append(dict(r, crop=t, layer=lay, idx=idx, P=P, edge=edge))
    cap = min(16384, C * sum(p["P"] for p in per_crop))
    merged = merge(per_crop, N, crop_nms_thresh, cap)
    regions, final = None, merged["keep"]
    if min_mask_region_area > 0:
        from . import tokenizer_ref

        nbr = tokenizer_ref.knn(x[None], x[None], min(amg_regions_ref.REGION_NEIGHBORS + 1, N))[0][0]
        regions = amg_regions_ref.postprocess_small_regions(merged["bits"], merged["keep"], nbr, min_mask_region_area,
                                                            mask_nms_thresh)
        final = merged["keep"][regions["keep"]]
    return dict(boxes=boxes, counts=counts, crops=per_crop, merged=merged, regions=regions, final=final)
