"""ORACLE (test infrastructure, NOT product code).

numpy restatement of automatic mask generation (pc_sam/automatic_mask_generator.py, include/psam_b200.h
psam_mask_candidates_f32 / psam_mask_nms): the candidate rules, greedy mask-IoU NMS as a plain loop over the sorted
candidates, and an end-to-end fp32 generator on the oracle models.  Every comparison is made in fp32 on exact integer
counts, so the device kernels must match this module exactly on the same logits.
"""
from __future__ import annotations

import numpy as np
import torch

NEG_INF = np.float32(-np.inf)


def pack_bits(masks: np.ndarray, W: int = None) -> np.ndarray:
    """bool [K, N] -> uint32 [K, W]: point n is bit n % 32 of word n // 32, words past N are zero."""
    K, N = masks.shape
    W = W if W is not None else (N + 31) // 32
    padded = np.zeros((K, W * 32), dtype=bool)
    padded[:, :N] = masks
    return np.packbits(padded, axis=1, bitorder="little").view("<u4").reshape(K, W)


def unpack_bits(bits: np.ndarray, N: int) -> np.ndarray:
    b = np.ascontiguousarray(bits).astype("<u4")
    return np.unpackbits(b.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)


def candidates(logits, iou_preds, mask_threshold=0.0, stability_offset=1.0, pred_iou_thresh=0.0, stability_thresh=0.0,
               min_area=0, W=None):
    """logits [Z, C, N], iou_preds [Z, C] -> dict of bits [Z*C, W] uint32, area int32, stability fp32, score fp32
    (the predicted IoU of a surviving candidate, -inf otherwise)."""
    lg = np.asarray(logits, dtype=np.float32)
    Z, C, N = lg.shape
    lg = lg.reshape(Z * C, N)
    iou = np.asarray(iou_preds, dtype=np.float32).reshape(Z * C)
    thr = np.float32(mask_threshold)
    hi = np.float32(thr + np.float32(stability_offset))
    lo = np.float32(thr - np.float32(stability_offset))
    masks = lg > thr
    area = masks.sum(1).astype(np.int32)
    with np.errstate(divide="ignore", invalid="ignore"):
        stab = (lg > hi).sum(1).astype(np.float32) / (lg > lo).sum(1).astype(np.float32)
    keep = ~np.isnan(iou) & (area >= min_area) & (area >= 1)
    if pred_iou_thresh > 0:
        keep &= iou > np.float32(pred_iou_thresh)
    if stability_thresh > 0:
        keep &= stab >= np.float32(stability_thresh)
    score = np.where(keep, iou, NEG_INF).astype(np.float32)
    return dict(bits=pack_bits(masks, W), area=area, stability=stab.astype(np.float32), score=score)


def sort_order(score: np.ndarray) -> np.ndarray:
    """Valid candidates (score > -inf) by (score descending, index ascending)."""
    s = np.asarray(score, dtype=np.float32)
    idx = np.nonzero(s > NEG_INF)[0]
    return idx[np.lexsort((idx, -s[idx]))]


def intersections(bits: np.ndarray, N: int = None) -> np.ndarray:
    """Pairwise popcount(bits_i & bits_j), exact (fp32 products of 0/1 summed in blocks well below 2^24)."""
    m = unpack_bits(bits, bits.shape[1] * 32).astype(np.float32)
    K = m.shape[0]
    out = np.zeros((K, K), dtype=np.int64)
    step = 1 << 20
    for c in range(0, m.shape[1], step):
        blk = m[:, c:c + step]
        out += (blk @ blk.T).astype(np.int64)
    return out


def nms(bits, area, score, nms_thresh) -> np.ndarray:
    """Greedy mask-IoU NMS: walk the sorted candidates, keep one unless an earlier kept candidate has
    fp32(inter) / fp32(area_i + area_j - inter) > nms_thresh with it.  Returns the kept candidate indices in order.
    The intersections of a kept candidate with the later ones are popcounts of the packed words."""
    order = sort_order(score)
    if len(order) == 0:
        return np.zeros(0, dtype=np.int64)
    b = np.ascontiguousarray(np.asarray(bits).astype(np.uint32)[order])
    a = np.asarray(area, dtype=np.int64)[order]
    thr = np.float32(nms_thresh)
    removed = np.zeros(len(order), dtype=bool)
    kept = []
    for i in range(len(order)):
        if removed[i]:
            continue
        kept.append(order[i])
        j = i + 1 + np.nonzero(~removed[i + 1:])[0]
        it = np.bitwise_count(b[j] & b[i]).sum(1, dtype=np.int64)
        with np.errstate(divide="ignore", invalid="ignore"):
            iou = it.astype(np.float32) / (a[i] + a[j] - it).astype(np.float32)
        removed[j[iou > thr]] = True
    return np.asarray(kept, dtype=np.int64)


def pair_ious(bits, area, idx) -> np.ndarray:
    """fp32 mask IoU of every pair among the candidates `idx` (for margin checks)."""
    b = np.asarray(bits)[idx]
    a = np.asarray(area, dtype=np.int64)[idx]
    inter = intersections(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter.astype(np.float32) / (a[:, None] + a[None, :] - inter).astype(np.float32)


def generate_ref(model, xyz: torch.Tensor, rgb: torch.Tensor, points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.88,
                 stability_score_thresh=0.95, stability_score_offset=1.0, mask_nms_thresh=0.7, min_mask_area=0):
    """End-to-end fp32 generator: oracle model (torch_ref / hier_ref) predict_masks on the FPS prompts of
    tokenizer_ref.fps, then the numpy candidate rules and NMS.  xyz / rgb [1, N, 3] CPU tensors."""
    from . import tokenizer_ref

    N = xyz.shape[1]
    P = min(points_per_cloud, N)
    pidx = tokenizer_ref.fps(xyz.numpy(), P)[0]
    centers = xyz[0, torch.from_numpy(pidx)]
    logits, ious = [], []
    with torch.no_grad():
        for s in range(0, P, points_per_batch):
            e = min(P, s + points_per_batch)
            m, i = model.predict_masks(xyz, rgb, centers[s:e].unsqueeze(1), torch.ones((e - s, 1), dtype=torch.int64), None, True)
            logits.append(m.numpy())
            ious.append(i.numpy())
    logits, ious = np.concatenate(logits), np.concatenate(ious)
    cand = candidates(logits, ious, 0.0, stability_score_offset, pred_iou_thresh, stability_score_thresh, min_mask_area)
    keep = nms(cand["bits"], cand["area"], cand["score"], mask_nms_thresh)
    C = logits.shape[1]
    return dict(logits=logits, iou=ious, point_index=pidx, keep=keep, slots=C, **cand)
