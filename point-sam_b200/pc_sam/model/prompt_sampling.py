"""Ground-truth-driven prompt sampling for PointCloudSAM.forward(is_eval=True)
(/root/reference/pc_sam/model/common.py:287-474: sample_prompts_adapter, sample_fixed_points,
sample_furthest_points_from_border).  

The reference walks (cloud, mask) pairs in Python, compacts foreground/background points, calls torkit3d's chamfer
kernel per region and compares the results on the host.  Here every (cloud, mask, region) is evaluated by one
psam_border_prompt_f32 call (compact, distance sweep, select; no host synchronisation except the single validity check), with the same
distances (chamfer arithmetic) and the same argmax tie-break."""
from __future__ import annotations

from typing import Union

import torch

from psam_b200 import engine, ops


def sample_furthest_points_from_border(coords: torch.Tensor, labels: torch.Tensor, gt: torch.Tensor):
    """Single-mask form kept for API compatibility (common.py:445-474): coords [N,3], labels [N], gt [N]."""
    lab = labels == 1
    if int(lab.sum()) == 0 or int((labels == 0).sum()) == 0:
        return None, None, -1
    fg = coords[lab]
    min_dists = ops.nn_distance(fg, coords[labels == 0])
    center_idx = torch.argmax(min_dists)
    return fg[center_idx][None, ...], gt[lab][center_idx][None, ...], torch.max(min_dists)


@torch.no_grad()
def sample_fixed_points(points, gt_masks, pred_logits, threshold=None, from_error_region=False):
    """points [B,N,3], gt_masks [B,M,N] bool, pred_logits [B*M,N] | None -> ([B*M,1,3], [B*M,1] bool)."""
    B, M, N = gt_masks.shape
    logits = masks = None
    if pred_logits is not None:
        pred_logits = pred_logits.reshape(B * M, N)
        if threshold is None:
            logits = pred_logits  # mask = logit > 0, evaluated inside the kernel
        else:
            masks = pred_logits.sigmoid() > threshold
    xyz, labels, _ = ops.border_prompt(points, gt_masks.bool(), logits, masks, from_error_region,
                                       status=engine.sampler_flag(points.device))
    engine.raise_if_sampler_failed(points.device)  # the one host check per prompt iteration (skipped under graph capture)
    return xyz, labels


@torch.no_grad()
def sample_prompts(points, gt_masks, pred_logits, threshold=None):
    """Random point of the error region (common.py:321-368) - the training-time branch, plain tensor indexing."""
    B, M, N = gt_masks.shape
    if pred_logits is None:
        diff = gt_masks
    else:
        pl = pred_logits.reshape(B, M, N)
        diff = gt_masks != (pl > 0 if threshold is None else pl.sigmoid() > threshold)
    pcs, pls = [], []
    for i in range(B):
        for j in range(M):
            inds = torch.nonzero(diff[i, j]).squeeze(1)
            if inds.numel() == 0:
                inds = torch.nonzero(gt_masks[i, j]).squeeze(1)
            idx = inds[torch.randint(0, len(inds), [1], device=inds.device)]
            pcs.append(points[i][idx])
            pls.append(gt_masks[i, j][idx])
    return torch.stack(pcs), torch.stack(pls)


@torch.no_grad()
def sample_prompts_adapter(points, gt_masks, pred_logits: Union[torch.Tensor, None], threshold=None, is_eval=False):
    """common.py:287-318: first iteration samples inside the ground truth, later ones inside the error regions; the
    random sampler is only used in training once the batch IoU has reached 1."""
    if pred_logits is None:
        return sample_fixed_points(points, gt_masks, pred_logits, threshold, from_error_region=True)
    if not is_eval:
        B, M, N = gt_masks.shape
        g = gt_masks.reshape(B * M, N)
        pm = pred_logits.reshape(B * M, N) > 0 if threshold is None else pred_logits.reshape(B * M, N).sigmoid() > threshold
        if not float((g & pm).sum() / (g | pm).sum()) < 1:
            return sample_prompts(points, gt_masks, pred_logits, threshold)
    return sample_fixed_points(points, gt_masks, pred_logits, threshold, from_error_region=False)
