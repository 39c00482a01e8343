"""ORACLE tooling (NOT product code): mint tests/golden/hier.npz by running the REFERENCE's own PointCloudSAMHier.forward
(pc_sam.py:377-496) on CPU, with the substitutions of oracle/make_golden.py (C FPS, restated timm), exact-distance cdist,
and its random prompt sampler (pc_sam.py:434) replaced by a stub that returns a stored, seeded prompt sequence.

Run here (needs the reference checkout):   python -m oracle.make_hier_golden
Weights are not stored: they are re-created by ``oracle.hier_ref.build_hier_model(seed=...)`` and pinned by a checksum.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import hier_ref, synth, torch_ref
from oracle.make_golden import REPO, import_reference, state_checksum

HIER_MODEL = dict(B=2, M=2, N=2000, G=(128, 32), K=(32, 16), radius=(0.2, 0.4), encoder="eva02_test_tiny", rounds=3, seed=11)


@torch.no_grad()
def hier_fixture(ref, out_dir):
    h = HIER_MODEL
    B, M, N, R = h["B"], h["M"], h["N"], h["rounds"]
    xyz, feats = synth.make_batch(B, N, h["seed"], "ball")
    g = torch.Generator().manual_seed(h["seed"])
    seq_c, seq_l = [], []
    for _ in range(R):
        idx = torch.randint(0, N, (B, M), generator=g)
        seq_c.append(torch.stack([xyz[b, idx[b]] for b in range(B)]).reshape(B * M, 1, 3))
        seq_l.append(torch.randint(0, 2, (B * M, 1), generator=g).bool())
    oracle = hier_ref.build_hier_model(h["encoder"], h["G"], h["K"], h["radius"], prompt_iters=R, seed=1234 + h["seed"])
    radius = list(h["radius"])
    pe = ref["enc"].PatchEmbedHier(6, 512, list(h["G"]), list(h["K"]), radius)
    enc = ref["enc"].PointCloudEncoder(pe, torch_ref.create_model(h["encoder"]), 256)
    me = ref["prompt"].MaskEncoderHier(256, radius=radius)
    md = ref["dec"].MaskDecoderHier(256, ref["tr"].TwoWayTransformer(2, 256, 8, 2048))
    model = ref["sam"].PointCloudSAMHier(enc, me, md, R).eval()
    model.load_state_dict(oracle.state_dict(), strict=True)  # pins the state-dict key contract
    rounds = iter(range(R))

    def stub_sample_prompts(coords, gt_masks, prompt_masks):
        t = next(rounds)
        return seq_c[t], seq_l[t]

    orig_cdist, orig_sampler = torch.cdist, ref["sam"].sample_prompts
    torch.cdist = lambda a, b, **kw: orig_cdist(a, b, compute_mode="donot_use_mm_for_euclid_dist")
    ref["sam"].sample_prompts = stub_sample_prompts
    try:
        gt = torch.zeros((B, M, N), dtype=torch.bool)  # only its shape is read once the sampler is stubbed
        outs = model(xyz, feats, gt)
        emb, (p1, p2) = model.pc_encoder(xyz, feats)
    finally:
        torch.cdist, ref["sam"].sample_prompts = orig_cdist, orig_sampler
    pack = dict(meta=np.array([B, M, N, *h["G"], *h["K"], R, h["seed"]]), radius=np.array(h["radius"]), encoder=h["encoder"],
                weights_checksum=state_checksum(model.state_dict()), xyz=xyz.numpy(), feats=feats.numpy(),
                centers1=p1["centers"].numpy(), centers2=p2["centers"].numpy(), fps_idx1=p1["fps_idx"].numpy().astype(np.int32),
                knn1_sorted=torch.sort(p1["knn_idx"], -1).values.numpy().astype(np.int32),
                knn2_sorted=torch.sort(p2["knn_idx"], -1).values.numpy().astype(np.int32),
                emb1=p1["embeddings"].numpy(), emb2=p2["embeddings"].numpy(), pc_embeddings=emb.numpy())
    for t, o in enumerate(outs):
        pack[f"prompt_coords{t}"], pack[f"prompt_labels{t}"] = seq_c[t].numpy(), seq_l[t].numpy()
        pack[f"masks{t}"], pack[f"iou{t}"], pack[f"prompt_masks{t}"] = o["masks"].numpy(), o["iou_preds"].numpy(), o["prompt_masks"].numpy()
    np.savez_compressed(os.path.join(out_dir, "hier.npz"), **pack)
    print("hier fixture written:", [tuple(o["masks"].shape) for o in outs])


if __name__ == "__main__":
    torch.set_num_threads(8)
    hier_fixture(import_reference(), os.path.join(REPO, "tests", "golden"))
