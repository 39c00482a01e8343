"""/root/reference/pc_sam/model/loss.py: the evaluation metric (compute_iou, :80-98) and the training criterion
(Criterion, :110-158) of mask_decoder fine-tuning.  Criterion's mask loss runs in CUDA (psam_b200.train.mask_loss: per-row
statistics, then dlogits); only the tiny [B*M, C] finalisation (selection, means, MSE) is torch tensor code, with no host
synchronisation."""
from typing import Dict, List

import torch
import torch.nn as nn
import torch.nn.functional as F


def compute_iou(logits: torch.Tensor, targets: torch.Tensor, threshold: float = None):
    assert logits.shape == targets.shape, (logits.shape, targets.shape)
    assert targets.dtype == torch.bool, targets.dtype
    preds = logits > 0 if threshold is None else logits.sigmoid() > threshold
    return (preds & targets).sum(-1) / (preds | targets).sum(-1)


def _first_argmin(x: torch.Tensor) -> torch.Tensor:
    """Index of the row minimum of x [Z, C], the lowest index on ties (torch.min's CPU result), without a host sync."""
    C = x.shape[1]
    m = x.min(dim=1, keepdim=True).values
    ar = torch.arange(C, device=x.device).expand_as(x)
    return torch.where(x == m, ar, C).min(dim=1).values.clamp_max(C - 1)


def _take(x: torch.Tensor, sel: torch.Tensor) -> torch.Tensor:
    """x[z, sel[z], ...] for x [Z, C, ...]."""
    shape = (x.shape[0], 1) + tuple(x.shape[2:])
    return x.gather(1, sel.view((-1, 1) + (1,) * (x.dim() - 2)).expand(shape)).squeeze(1)


class Criterion(nn.Module):
    """The reference's Criterion: per iteration, sigmoid focal loss (alpha=-1, gamma=2) averaged over the points plus
    2 x dice (eps=1e-3) on the mask logits; at iteration 0 the mask of minimum loss is selected (lowest index on ties), later
    iterations have one mask.  loss_iou is the MSE between the selected iou_preds and the hard IoU of the selected mask
    (integer counts, one fp32 division: bit for bit the reference's compute_iou), or with use_soft_iou the soft Jaccard
    (eps=1e-3).  The loss is the mean over iterations; aux holds iou, best_masks, loss_mask and loss_iou per iteration.
    An empty ground truth with an empty prediction has IoU NaN, as in the reference."""

    def __init__(self, use_soft_iou=False):
        super().__init__()
        self.use_soft_iou = use_soft_iou

    def forward(self, outputs: List[Dict[str, torch.Tensor]], gt_masks: torch.Tensor):
        """outputs: PointCloudSAM.forward's list (masks [B*M, C, N], iou_preds [B*M, C]); gt_masks [B*M, N] bool."""
        from psam_b200.train import mask_loss

        gt = gt_masks.bool().contiguous()
        losses, aux_outputs = [], []
        for i, output in enumerate(outputs):
            masks, iou_preds = output["masks"], output["iou_preds"]
            loss_zc, stats, counts = mask_loss(masks, gt)  # [B*M, C]
            if i == 0:
                sel = _first_argmin(loss_zc.detach())
            else:
                if masks.shape[1] != 1:
                    raise ValueError(f"iteration {i}: one mask per prompt expected after the first iteration, got {masks.shape[1]}")
                sel = torch.zeros(masks.shape[0], dtype=torch.long, device=masks.device)
            loss_mask = _take(loss_zc, sel).mean()
            best_masks = _take(masks, sel)
            iou_pred = _take(iou_preds, sel)
            cnt = _take(counts, sel)
            iou = cnt[:, 0].float() / cnt[:, 1].float()
            if self.use_soft_iou:
                st = _take(stats, sel)
                soft_iou = (st[:, 1] + 1e-3) / (st[:, 2] + st[:, 3] - st[:, 1] + 1e-3)
                loss_iou = F.mse_loss(soft_iou, iou_pred)
            else:
                loss_iou = F.mse_loss(iou, iou_pred)
            losses.append(loss_iou + loss_mask)
            aux_outputs.append(dict(iou=iou, best_masks=best_masks, loss_mask=loss_mask, loss_iou=loss_iou))
        return torch.stack(losses).mean(), aux_outputs
