"""ORACLE (test infrastructure, NOT product code).

CPU / plain-PyTorch fp32 restatement of the reference's hierarchical model, on top of ``oracle.torch_ref``:

* PointCloudEncoder with a list-returning tokenizer   pc_sam/model/pc_encoder.py:118-145
* MaskEncoderHier                                      pc_sam/model/prompt_encoder.py:136-183
* MaskDecoderHier                                      pc_sam/model/mask_decoder.py:214-370
* PointCloudSAMHier                                    pc_sam/model/pc_sam.py:377-496 (prompts are supplied)

Every class keeps the reference's state-dict key names (strict-load verified in ``oracle/make_hier_golden.py``).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from .torch_ref import (MLP, AuxInputs, PatchEmbedHier, PatchEncoder, PointCloudEncoder, PointCloudSAM, TwoWayTransformer,
                        batch_index_select, compute_interp_weights, create_model, group_with_centers_and_knn,
                        interpolate_features, repeat_interleave)


class PointCloudEncoderHier(PointCloudEncoder):
    """pc_sam/model/pc_encoder.py:118-145 when patch_embed returns a list: the last level feeds the ViT, the list is returned."""

    def forward(self, coords, features):
        patches = self.patch_embed(coords, features)
        last = patches[-1]
        x = self.patch_proj(last["embeddings"]) + self.pos_embed(last["centers"])
        x = self.transformer.pos_drop(x)
        for blk in self.transformer.blocks:
            x = blk(x)
        x = self.transformer.fc_norm(self.transformer.norm(x))
        return self.out_proj(x), patches


class MaskEncoderHier(nn.Module):
    """pc_sam/model/prompt_encoder.py:136-183."""

    def __init__(self, embed_dim, in_channels=4, radius=None):
        super().__init__()
        self.embed_dim, self.in_channels, self.radius = embed_dim, in_channels, radius
        self.patch_encoder1 = PatchEncoder(in_channels, 128, [64, 128])
        self.patch_encoder2 = PatchEncoder(128 + 3, embed_dim, [128, 256])
        self.no_mask_embed = nn.Embedding(1, embed_dim)

    def forward(self, masks, coords, centers1, knn_idx1, centers2, knn_idx2):
        if masks is None:
            return self.no_mask_embed.weight.reshape(1, 1, -1).expand(centers2.shape[0], centers2.shape[1], -1)
        r = self.radius
        x1 = self.patch_encoder1(group_with_centers_and_knn(coords, masks.detach().unsqueeze(-1), centers1, knn_idx1,
                                                           radius=r[0] if r else None))
        x2 = self.patch_encoder2(group_with_centers_and_knn(centers1, x1, centers2, knn_idx2, radius=r[1] if r else None))
        return [x1, x2]


class MaskDecoderHier(nn.Module):
    """pc_sam/model/mask_decoder.py:214-370 (the MaskDecoder transformer and IoU head, two-stage upscaling)."""

    def __init__(self, transformer_dim, transformer, num_multimask_outputs=3, iou_head_depth=3, iou_head_hidden_dim=256,
                 encoder_dim=128):
        super().__init__()
        D = transformer_dim
        self.transformer_dim, self.transformer = D, transformer
        self.num_multimask_outputs = num_multimask_outputs
        self.iou_token = nn.Embedding(1, D)
        self.num_mask_tokens = num_multimask_outputs + 1
        self.mask_tokens = nn.Embedding(self.num_mask_tokens, D)
        self.output_hypernetworks_mlps = nn.ModuleList([MLP(D, D, D // 2, 3) for _ in range(self.num_mask_tokens)])
        self.output_upscaling2 = nn.Sequential(nn.Linear(D + encoder_dim, D), nn.LayerNorm(D), nn.GELU(), nn.Linear(D, D))
        self.output_upscaling1 = nn.Sequential(nn.Linear(D, D // 2), nn.LayerNorm(D // 2), nn.GELU(),
                                               nn.Linear(D // 2, D // 2), nn.GELU())
        self.iou_prediction_head = MLP(D, iou_head_hidden_dim, self.num_mask_tokens, iou_head_depth)

    @staticmethod
    def _upscale(src, aux, concat_feats=False):
        """mask_decoder.py:347-370."""
        if aux.interp_index is None or aux.interp_weight is None:
            with torch.no_grad():
                aux.interp_index, aux.interp_weight = compute_interp_weights(aux.coords, aux.centers)
        rep = src.shape[0] // aux.interp_index.shape[0]
        x = interpolate_features(src, repeat_interleave(aux.interp_index, rep, 0), repeat_interleave(aux.interp_weight, rep, 0))
        if concat_feats:
            x = torch.cat((x, repeat_interleave(aux.features, rep, 0)), dim=-1)
        return x

    def forward(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings, aux_inputs1, aux_inputs2,
                multimask_output):
        mask_slice = slice(1, None) if multimask_output else slice(0, 1)
        out_tokens = torch.cat([self.iou_token.weight, self.mask_tokens.weight], dim=0)
        out_tokens = out_tokens.unsqueeze(0).expand(sparse_prompt_embeddings.size(0), -1, -1)
        tokens = torch.cat((out_tokens, sparse_prompt_embeddings), dim=1)
        rep = tokens.shape[0] // pc_embeddings.shape[0]
        src = repeat_interleave(pc_embeddings, rep, 0) + dense_prompt_embeddings
        hs, src = self.transformer(src, repeat_interleave(pc_pe, rep, 0), tokens)
        up = self.output_upscaling2(self._upscale(src, aux_inputs2, concat_feats=True))
        up = self.output_upscaling1(self._upscale(up, aux_inputs1))
        ids = list(range(self.num_mask_tokens))[mask_slice]
        hyper_in = torch.stack([self.output_hypernetworks_mlps[i](hs[:, 1 + i, :]) for i in ids], dim=1)
        masks = hyper_in @ up.transpose(-1, -2)
        return masks, self.iou_prediction_head(hs[:, 0, :])[:, mask_slice]


class PointCloudSAMHier(PointCloudSAM):
    """pc_sam/model/pc_sam.py:377-496: the forward loop with externally supplied prompts (the reference samples them)."""

    def _encode(self, coords, features):
        pc_embeddings, (p1, p2) = self.pc_encoder(coords, features)
        aux1 = AuxInputs(coords=coords, features=features, centers=p1["centers"])
        aux2 = AuxInputs(coords=p1["centers"], features=p1["embeddings"], centers=p2["centers"])
        return pc_embeddings, p1, p2, aux1, aux2, self.point_encoder.pe_layer(p2["centers"])

    def _round(self, coords, enc, pc, pl, pm, multimask_output):
        pc_embeddings, p1, p2, aux1, aux2, pc_pe = enc
        sparse = self.point_encoder(pc, pl)
        dense = self.mask_encoder(pm, coords, p1["centers"], p1["knn_idx"], p2["centers"], p2["knn_idx"])
        dense = dense[-1] if isinstance(dense, list) else repeat_interleave(dense, sparse.shape[0] // dense.shape[0], 0)
        return self.mask_decoder(pc_embeddings, pc_pe, sparse, dense, aux1, aux2, multimask_output)

    def predict_iterative(self, coords, features, prompt_coords_seq, prompt_labels_seq):
        enc = self._encode(coords, features)
        outs, pm = [], None
        pc, pl = prompt_coords_seq[0][:, :0], prompt_labels_seq[0][:, :0]
        for t in range(len(prompt_coords_seq)):
            pc = torch.cat([pc, prompt_coords_seq[t]], dim=1)
            pl = torch.cat([pl, prompt_labels_seq[t]], dim=1)
            masks, iou = self._round(coords, enc, pc, pl, pm, t == 0)
            if t == 0:
                best = torch.argmax(iou, dim=1)
                pm = batch_index_select(masks, best, dim=1)
            else:
                best = 0
                pm = masks[:, 0]
            outs.append(dict(prompt_coords=pc, prompt_labels=pl, masks=masks, iou_preds=iou, max_iou_pred_ind=best,
                             prompt_masks=pm))
        return outs

    def predict_masks(self, coords, features, prompt_coords, prompt_labels, prompt_masks=None, multimask_output=True):
        """One round of the forward loop body with the given prompts and prompt mask (the reference's inherited
        predict_masks fails on this model)."""
        return self._round(coords, self._encode(coords, features), prompt_coords, prompt_labels, prompt_masks, multimask_output)


def build_hier_model(encoder: str = "eva02_large_patch14_448", G=(2048, 512), K=(32, 32), radius=(0.05, 0.1),
                     prompt_iters=8, seed: Optional[int] = 1234) -> PointCloudSAMHier:
    """Mirror of configs/model/hier.yaml with default torch initialisation."""
    if seed is not None:
        torch.manual_seed(seed)
    radius = list(radius) if radius is not None else None
    pe = PatchEmbedHier(6, 512, list(G), list(K), radius)
    enc = PointCloudEncoderHier(pe, create_model(encoder), 256)
    me = MaskEncoderHier(256, radius=radius)
    md = MaskDecoderHier(256, TwoWayTransformer(2, 256, 8, 2048))
    return PointCloudSAMHier(enc, me, md, prompt_iters).eval()
