"""ORACLE (test infrastructure, NOT product code).

numpy / scipy restatement of the small-region post-processing of automatic mask generation (include/psam_b200.h
psam_mask_regions, the min_mask_region_area path of pc_sam/automatic_mask_generator.py): segment-anything's
remove_small_regions / postprocess_small_regions with connectivity given by the cloud's kNN graph instead of an 8-connected
pixel grid.  Components come from scipy.sparse.csgraph.connected_components; every decision is made on exact integer
counts, so the device kernel must match this module exactly on the same masks and graph.
"""
from __future__ import annotations

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from . import amg_ref

REGION_NEIGHBORS = 8  # PointCloudMaskGenerator.region_neighbors


def components(member: np.ndarray, nbr: np.ndarray):
    """Connected components of the points with member[i] (bool [N]) in the undirected graph {i, nbr[i, t]}, i != j, both
    ends members (entries outside 0..N-1 are no edge).  Returns (label [N], -1 outside the set; size [C]; smallest point
    index [C])."""
    member = np.asarray(member, dtype=bool)
    N = member.shape[0]
    nbr = np.asarray(nbr, dtype=np.int64).reshape(N, -1)
    i = np.repeat(np.arange(N), nbr.shape[1])
    j = nbr.ravel()
    ok = (j >= 0) & (j < N)
    i, j = i[ok], j[ok]
    ok = member[i] & member[j] & (i != j)
    g = coo_matrix((np.ones(int(ok.sum()), dtype=np.int8), (i[ok], j[ok])), shape=(N, N)).tocsr()
    _, lab = connected_components(g, directed=False)
    idx = np.nonzero(member)[0]
    _, comp = np.unique(lab[idx], return_inverse=True)
    label = np.full(N, -1, dtype=np.int64)
    label[idx] = comp
    size = np.bincount(comp).astype(np.int64) if len(idx) else np.zeros(0, dtype=np.int64)
    first = np.full(len(size), N, dtype=np.int64)
    np.minimum.at(first, comp, idx)
    return label, size, first


def remove_small_regions(mask: np.ndarray, nbr: np.ndarray, min_area: int, mode: str):
    """SAM's remove_small_regions on a point cloud.  mode "holes": components of the points outside the mask with fewer
    than min_area points join it.  mode "islands": components of the mask with fewer than min_area points leave it; if none
    reaches min_area only the largest stays (equal sizes: the one with the lowest smallest point index).
    Returns (new mask, changed): changed = some component was smaller than min_area."""
    assert mode in ("holes", "islands")
    mask = np.asarray(mask, dtype=bool)
    holes = mode == "holes"
    member = ~mask if holes else mask
    label, size, first = components(member, nbr)
    small = size < min_area
    if not small.any():
        return mask.copy(), False
    if holes:
        return mask | (member & small[np.maximum(label, 0)]), True
    keep = ~small
    if not keep.any():
        keep[np.lexsort((first, -size))[0]] = True
    return member & keep[np.maximum(label, 0)], True


def postprocess_small_regions(bits: np.ndarray, keep: np.ndarray, nbr: np.ndarray, min_area: int, nms_thresh: float):
    """SAM's postprocess_small_regions on the kept masks bits[keep] (uint32 [K, W] candidates, keep = kept slots in NMS
    order), over the kNN graph nbr [N, k1].  Per kept rank p: holes, then islands; score 1 if neither changed the mask, 0
    otherwise; then greedy mask NMS on the results.  Returns dict of bits [P, W] uint32, area [P] int32, score [P] fp32
    (indexed by rank) and keep (the ranks kept by the second NMS, in order)."""
    nbr = np.asarray(nbr, dtype=np.int64)
    N = nbr.shape[0]
    bits = np.asarray(bits).astype(np.uint32)
    keep = np.asarray(keep, dtype=np.int64)
    masks = amg_ref.unpack_bits(bits[keep], N) if len(keep) else np.zeros((0, N), dtype=bool)
    out = np.zeros_like(masks)
    score = np.ones(len(keep), dtype=np.float32)
    for p, m in enumerate(masks):
        m, changed_h = remove_small_regions(m, nbr, min_area, "holes")
        m, changed_i = remove_small_regions(m, nbr, min_area, "islands")
        out[p] = m
        if changed_h or changed_i:
            score[p] = 0.0
    b = amg_ref.pack_bits(out, bits.shape[1])
    area = out.sum(1).astype(np.int32)
    return dict(bits=b, area=area, score=score, keep=amg_ref.nms(b, area, score, nms_thresh))


def generate_ref(model, xyz, rgb, points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.88,
                 stability_score_thresh=0.95, stability_score_offset=1.0, mask_nms_thresh=0.7, min_mask_area=0,
                 min_mask_region_area=0):
    """amg_ref.generate_ref, then (min_mask_region_area > 0) the small-region stage over the C oracle's kNN graph
    (tokenizer_ref.knn, k1 = min(REGION_NEIGHBORS + 1, N)).  Adds nbr, regions (postprocess_small_regions' dict) and
    final_slots = the candidate slot of every output mask, in output order."""
    from . import tokenizer_ref

    want = amg_ref.generate_ref(model, xyz, rgb, points_per_cloud, points_per_batch, pred_iou_thresh, stability_score_thresh,
                                stability_score_offset, mask_nms_thresh, min_mask_area)
    if min_mask_region_area <= 0:
        return dict(want, final_slots=want["keep"])
    N = xyz.shape[1]
    nbr = tokenizer_ref.knn(xyz.numpy(), xyz.numpy(), min(REGION_NEIGHBORS + 1, N))[0][0]
    post = postprocess_small_regions(want["bits"], want["keep"], nbr, min_mask_region_area, mask_nms_thresh)
    return dict(want, nbr=nbr, regions=post, final_slots=want["keep"][post["keep"]])
