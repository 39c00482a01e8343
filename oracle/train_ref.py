"""ORACLE (not product code): fp64 restatement of mask_decoder fine-tuning - the reference's Criterion
(pc_sam/model/loss.py:58-158, with torchvision's sigmoid_focal_loss restated from its formula), the per-point mask head, and a
teacher-forced training loop over oracle.torch_ref.MaskDecoder.  Pinned to the reference's own code by
tests/golden/train.npz (oracle/make_train_golden.py, tests/test_finetune.py); the GPU tests use it at any size."""
from __future__ import annotations

import zlib
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

from . import torch_ref


# ---------------------------------------------------------------------------------------------------------
# deterministic parameters: every tensor drawn from its own seeded generator (independent of construction order)
# ---------------------------------------------------------------------------------------------------------
def fill_params(module: torch.nn.Module, seed: int) -> torch.nn.Module:
    """Weights ~ N(0, 1/fan_in), biases ~ 0.1 N(0, 1), LayerNorm weights 1 + 0.1 N(0, 1), embeddings N(0, 1)."""
    norms = {id(m.weight) for m in module.modules() if isinstance(m, torch.nn.LayerNorm)}
    with torch.no_grad():
        for name, p in module.named_parameters():
            g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
            r = torch.randn(p.shape, generator=g, dtype=torch.float64)
            if id(p) in norms:
                v = 1.0 + 0.1 * r
            elif name.endswith("bias"):
                v = 0.1 * r
            elif p.dim() == 2 and "embedding" not in name and "token" not in name:
                v = r / np.sqrt(p.shape[1])
            else:
                v = r
            p.copy_(v.to(p.dtype))
    return module


def grad_probe(name: str, g: torch.Tensor, k: int = 16) -> np.ndarray:
    """Compact fingerprint of a gradient: (norm, dot with a seeded probe, k seeded entries), fp64."""
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    flat = g.detach().double().flatten()
    probe = torch.randn(flat.numel(), generator=gen, dtype=torch.float64)
    idx = torch.randint(0, flat.numel(), (k,), generator=gen)
    return np.concatenate([[float(flat.norm()), float(flat @ probe)], flat[idx].numpy()])


# ---------------------------------------------------------------------------------------------------------
# loss (pc_sam/model/loss.py)
# ---------------------------------------------------------------------------------------------------------
def sigmoid_focal_loss(inputs, targets, alpha: float = -1, gamma: float = 2):
    """torchvision.ops.sigmoid_focal_loss(reduction="none") restated from its formula."""
    p = torch.sigmoid(inputs)
    ce = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    loss = ce * ((1 - p_t) ** gamma)
    if alpha >= 0:
        loss = (alpha * targets + (1 - alpha) * (1 - targets)) * loss
    return loss


def dice_loss(inputs, targets, eps: float = 1e-3):
    num = 2 * (inputs * targets).sum(-1)
    den = inputs.square().sum(-1) + targets.sum(-1)
    return 1 - (num + eps) / (den + eps)


def compute_mask_loss(logits, labels, loss_weight_dice: float = 2):
    t = labels.unsqueeze(1).expand_as(logits).to(logits.dtype)
    return sigmoid_focal_loss(logits, t).mean(-1) + loss_weight_dice * dice_loss(logits.sigmoid(), t)


def compute_iou(logits, targets):
    preds = logits > 0
    return (preds & targets).sum(-1) / (preds | targets).sum(-1)


def compute_jaccard(logits, targets, eps: float = 1e-3):
    probs = logits.sigmoid()
    num = (probs * targets).sum(-1)
    return (num + eps) / ((probs.square() + targets.square()).sum(-1) - num + eps)


def criterion(outputs: List[Dict[str, torch.Tensor]], gt_masks, use_soft_iou: bool = False, hard_iou=None):
    """The reference's Criterion.forward (loss.py:115-158); run on the CPU, so loss.min picks the lowest index on ties.
    hard_iou: optional per-iteration IoU targets to use instead of the IoU of the oracle's own masks (teacher forcing of the
    logit > 0 decisions when comparing against an fp32 run)."""
    losses, aux = [], []
    for i, o in enumerate(outputs):
        masks, iou_preds = o["masks"], o["iou_preds"]
        loss_mask = compute_mask_loss(masks, gt_masks)
        if i == 0:
            loss_mask, sel = loss_mask.min(dim=1)
            ar = torch.arange(sel.shape[0])
            best, iou_preds = masks[ar, sel], iou_preds[ar, sel]
        else:
            best, iou_preds = masks.squeeze(1), iou_preds.squeeze(1)
        loss_mask = loss_mask.mean()
        iou = compute_iou(best, gt_masks) if hard_iou is None else hard_iou[i]
        if use_soft_iou:
            with torch.no_grad():
                target = compute_jaccard(best, gt_masks.to(best.dtype))
        else:
            target = iou
        loss_iou = F.mse_loss(target.to(iou_preds.dtype), iou_preds)
        losses.append(loss_iou + loss_mask)
        aux.append(dict(iou=iou, best_masks=best, loss_mask=loss_mask, loss_iou=loss_iou))
    return torch.stack(losses).mean(), aux


# ---------------------------------------------------------------------------------------------------------
# the per-point mask head and the teacher-forced loop
# ---------------------------------------------------------------------------------------------------------
def mask_head(f0, hyper, gamma, beta, eps, w3, b3, idx, w, rep: int):
    """masks [Z,C,N] = hyper . GELU(W3 GELU(LN(interp(f0))) + b3); f0 [Z,G,D] = output_upscaling[0](keys), idx / w [B,N,3]."""
    idx = torch_ref.repeat_interleave(idx, rep, 0)
    w = torch_ref.repeat_interleave(w, rep, 0)
    v = torch_ref.interpolate_features(f0, idx, w)
    u1 = F.gelu(F.layer_norm(v, (v.shape[-1],), gamma, beta, eps))
    u2 = F.gelu(F.linear(u1, w3, b3))
    return hyper @ u2.transpose(-1, -2)


def decoder_loop(md, pc_embeddings, pc_pe, steps, aux):
    """Teacher-forced decoder iterations: steps is a list of (sparse [Z,P,D], dense [Z or B,G,D]) as the model fed them;
    iteration 0 is multimask.  Returns the forward's list of dicts (masks, iou_preds)."""
    outs = []
    for i, (sparse, dense) in enumerate(steps):
        dense = torch_ref.repeat_interleave(dense, sparse.shape[0] // dense.shape[0], 0)
        masks, iou = md(pc_embeddings, pc_pe, sparse, dense, aux_inputs=aux, multimask_output=(i == 0))
        outs.append(dict(masks=masks, iou_preds=iou))
    return outs


def build_decoder(D: int = 256, mlp_dim: int = 2048, seed: int = 0):
    md = torch_ref.MaskDecoder(D, torch_ref.TwoWayTransformer(2, D, 8, mlp_dim))
    return fill_params(md, seed)
