"""ORACLE tooling (NOT product code): mint tests/golden/train.npz from the reference's own MaskDecoder and Criterion
(imported unmodified through make_golden.import_reference) in float64 on CPU.  The hard IoU stays the reference's fp32
division, cast to fp64 for the MSE (see main()).

A fixed decoder (D = 256, seeded parameters from oracle.train_ref.fill_params, non-identity LayerNorms) runs two teacher-forced
iterations (multimask, then single) on fixed decoder-level inputs; the file records the masks, the Criterion's loss and aux,
and a fingerprint of the gradient of every decoder parameter (train_ref.grad_probe: weights are re-created from the seed).

Run here (needs /root/reference):   python -m oracle.make_train_golden
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

from oracle import train_ref  # noqa: E402
from oracle.make_golden import import_reference  # noqa: E402

SEED, D, MLP, B, M, G, N = 11, 256, 256, 2, 2, 32, 96


def make_inputs():
    g = torch.Generator().manual_seed(SEED)
    Z = B * M
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    idx = torch.stack([torch.randperm(G, generator=g)[:3] for _ in range(B * N)]).reshape(B, N, 3)
    w = torch.rand(B, N, 3, generator=g, dtype=torch.float64) + 0.05
    w = w / w.sum(-1, keepdim=True)
    gt = torch.rand(Z, N, generator=g) < 0.4
    gt[:, 0], gt[:, 1] = True, False  # no empty or full mask
    return dict(pc_embeddings=rn(B, G, D), pc_pe=rn(B, G, D), sparse0=rn(Z, 1, D), dense0=rn(1, 1, D).expand(B, G, D).contiguous(),
                sparse1=rn(Z, 2, D), dense1=rn(Z, G, D), interp_index=idx, interp_weight=w, gt=gt)


def run(md, AuxInputs, crit, x):
    aux = AuxInputs(coords=None, features=None, centers=None, interp_index=x["interp_index"], interp_weight=x["interp_weight"])
    outs = []
    for i, (sp, de) in enumerate([(x["sparse0"], x["dense0"]), (x["sparse1"], x["dense1"])]):
        de = de.repeat_interleave(sp.shape[0] // de.shape[0], 0)
        masks, iou = md(x["pc_embeddings"], x["pc_pe"], sp, de, aux_inputs=aux, multimask_output=(i == 0))
        outs.append(dict(masks=masks, iou_preds=iou))
    loss, aux_out = crit(outs, x["gt"])
    loss.backward()
    return outs, loss, aux_out


def main():
    ref = import_reference()
    import pc_sam.model.loss as ref_loss  # the reference's own (sys.path set by import_reference)

    # One substitution: compute_iou divides integer counts into the default dtype (fp32), and F.mse_loss against fp64
    # iou_preds then fails in backward; the fp32 IoU is cast to fp64 (same value) before the MSE.
    iou32 = ref_loss.compute_iou
    ref_loss.compute_iou = lambda logits, targets, threshold=None: iou32(logits, targets, threshold).double()

    torch.manual_seed(0)
    md = ref["dec"].MaskDecoder(D, ref["tr"].TwoWayTransformer(2, D, 8, MLP)).double()
    train_ref.fill_params(md, SEED)
    x = make_inputs()
    outs, loss, aux = run(md, ref["dec"].AuxInputs, ref_loss.Criterion(), x)
    pack = {k: v.numpy() for k, v in x.items()}
    for i, o in enumerate(outs):
        pack[f"masks{i}"] = o["masks"].detach().numpy()
        pack[f"iou_preds{i}"] = o["iou_preds"].detach().numpy()
        for k in ("iou", "best_masks", "loss_mask", "loss_iou"):
            pack[f"aux{i}_{k}"] = aux[i][k].detach().numpy()
    pack["loss"] = loss.detach().numpy()
    names = [n for n, _ in md.named_parameters()]
    pack["grad_names"] = np.array(names)
    pack["grad_probes"] = np.stack([train_ref.grad_probe(n, p.grad) for n, p in md.named_parameters()])
    out = os.path.join(REPO, "tests", "golden", "train.npz")
    np.savez_compressed(out, seed=SEED, dims=np.array([D, MLP, B, M, G, N]), **pack)
    print("wrote", out, "loss", float(loss))


if __name__ == "__main__":
    main()
