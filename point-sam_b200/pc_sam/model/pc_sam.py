"""PointCloudSAM with the reference API (/root/reference/pc_sam/model/pc_sam.py:20-196) plus the
``set_pointcloud`` / 4-argument ``predict_masks`` form that demo/app.py:198-205 calls.

All computation runs in the sm_90a kernels behind ``psam_b200`` (no CPU / PyTorch fallback).  Training mode fine-tunes
mask_decoder on a frozen encoder (psam_b200.train); everything else is inference."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from psam_b200 import engine, ops

from .common import batch_index_select, repeat_interleave
from .mask_decoder import AuxInputs, MaskDecoder
from .pc_encoder import PatchEmbedNN, PointCloudEncoder
from .prompt_encoder import MaskEncoder, PointEncoder


class PointCloudSAM(nn.Module):
    def __init__(self, pc_encoder: PointCloudEncoder, mask_encoder: MaskEncoder, mask_decoder: MaskDecoder,
                 prompt_iters: int, enable_mask_refinement_iterations=True):
        super().__init__()
        self.pc_encoder = pc_encoder
        self.point_encoder = PointEncoder(pc_encoder.embed_dim)
        self.mask_encoder = mask_encoder
        self.mask_decoder = mask_decoder
        self.prompt_iters = prompt_iters
        self.enable_mask_refinement_iterations = enable_mask_refinement_iterations
        self._cloud = None  # cache filled by set_pointcloud
        self._cloud_key = None

    # ------------------------------------------------------------------------------------------
    def _run_encoder(self, coords, features, lengths):
        if lengths is None:
            return self.pc_encoder(coords, features)
        return engine.run_pc_encoder(self.pc_encoder, coords, features, lengths=lengths)

    def _encode(self, coords, features, lengths=None):
        """lengths [B] int32 (device): coords / features are padded clouds (ops.pad_clouds), cloud b its first lengths[b]
        points; the caller has checked every lengths[b] >= the first-level num_groups (varlen_clouds)."""
        pc_embeddings, patches = self._run_encoder(coords, features, lengths)
        centers = patches["centers"]
        aux = AuxInputs(coords=coords, features=features, centers=centers)
        pc_pe = engine.run_pos_embedding(self.point_encoder.pe_layer, centers, check=False)
        return dict(pc_embeddings=pc_embeddings, patches=patches, aux=aux, pc_pe=pc_pe, coords=coords)

    def _decode_unchecked(self, enc, prompt_coords, prompt_labels, prompt_masks, multimask_output, center_idx=None):
        patches = enc["patches"]
        sparse = engine.run_point_encoder(self.point_encoder, prompt_coords, prompt_labels, check=False)
        dense = self.mask_encoder(prompt_masks, enc["coords"], patches["centers"], patches["knn_idx"], center_idx=center_idx)
        if prompt_masks is not None:
            dense = repeat_interleave(dense, sparse.shape[0] // dense.shape[0], 0)
        return self.mask_decoder(enc["pc_embeddings"], enc["pc_pe"], sparse, dense, aux_inputs=enc["aux"],
                                 multimask_output=multimask_output)

    def _decode(self, enc, prompt_coords, prompt_labels, prompt_masks, multimask_output, center_idx=None):
        masks, iou = self._decode_unchecked(enc, prompt_coords, prompt_labels, prompt_masks, multimask_output, center_idx)
        engine.raise_if_out_of_range(masks.device)  # ValueError like prompt_encoder.py:44-46 (one host sync)
        return masks, iou

    def _center_idx(self, enc):
        """FPS indices of the centres, for MaskEncoder(centralize_features=True)."""
        return enc["patches"].get("fps_idx")

    def _group_shape(self) -> tuple:
        g = self.pc_encoder.patch_embed.grouper
        return g.num_groups, g.group_size

    def varlen_clouds(self, coords: Sequence[torch.Tensor], features: Sequence[torch.Tensor]) -> List[int]:
        """Checks a batch of clouds of different sizes without touching the device and returns their sizes N_b: coords and
        features are sequences of B >= 1 tensors [N_b, 3] and [N_b, Cf].  A Voronoi tokenizer (PatchEmbedNN) is refused
        (NotImplementedError: padded points would join its cells' maxima), and so is a cloud smaller than the first-level
        num_groups or group_size (RuntimeError, as for one cloud: its kNN groups would take padded rows as neighbours)."""
        if isinstance(self.pc_encoder.patch_embed, PatchEmbedNN):
            raise NotImplementedError("clouds of different sizes need a kNN tokenizer: the Voronoi tokenizer (PatchEmbedNN) "
                                      "would pool padded points into its cells")
        if torch.is_tensor(coords) or torch.is_tensor(features):
            raise TypeError("coords and features must be sequences of [N_b, 3] / [N_b, C] tensors, one per cloud")
        coords, features = list(coords), list(features)
        if not coords or len(coords) != len(features):
            raise ValueError(f"{len(coords)} coordinate and {len(features)} feature tensors: need the same number >= 1")
        sizes = []
        for b, (c, f) in enumerate(zip(coords, features)):
            if c.dim() != 2 or c.shape[1] != 3 or f.dim() != 2 or f.shape[0] != c.shape[0]:
                raise ValueError(f"cloud {b}: coords {tuple(c.shape)} and features {tuple(f.shape)} must be [N_b, 3] and [N_b, C]")
            sizes.append(int(c.shape[0]))
        num_groups, group_size = self._group_shape()[:2]
        if min(sizes) < num_groups:
            raise RuntimeError("sample_farthest_points: number of points must be >= num_samples")
        if min(sizes) < group_size:
            b = sizes.index(min(sizes))
            raise RuntimeError(f"knn: cloud {b} has {sizes[b]} points, fewer than the group size {group_size} (k nearest "
                               "neighbours need k <= number of points)")
        return sizes

    def _varlen_gt(self, gt_masks: Sequence[torch.Tensor], sizes: List[int]) -> List[torch.Tensor]:
        """Checks per-cloud ground truth against the cloud sizes without touching the device: gt_masks is a sequence of
        [M, N_b] or [N_b] tensors with the same M for every cloud.  Returns them as [M, N_b]."""
        if torch.is_tensor(gt_masks):
            raise TypeError("gt_masks must be a sequence of [M, N_b] / [N_b] tensors, one per cloud")
        gts = [g.unsqueeze(0) if g.dim() == 1 else g for g in gt_masks]
        if len(gts) != len(sizes):
            raise ValueError(f"{len(gts)} ground-truth tensors for {len(sizes)} clouds")
        for b, (g, n) in enumerate(zip(gts, sizes)):
            if g.dim() != 2 or g.shape[1] != n or g.shape[0] != gts[0].shape[0] or g.shape[0] < 1:
                raise ValueError(f"cloud {b}: ground truth {tuple(gt_masks[b].shape)} must be [M, {n}] or [{n}], with the "
                                 f"same M >= 1 for every cloud (cloud 0 has M = {gts[0].shape[0]})")
        return gts

    def forward_varlen(self, coords: Sequence[torch.Tensor], features: Sequence[torch.Tensor],
                       gt_masks: Sequence[torch.Tensor], is_eval: bool = True) -> List[List[Dict[str, torch.Tensor]]]:
        """forward(is_eval=True) on B clouds of different sizes with one encode: coords / features / gt_masks are sequences
        of [N_b, 3], [N_b, C] and [M, N_b] or [N_b] bool tensors (the same M for every cloud).  The clouds are padded to
        N_max = max N_b (ops.pad_clouds) and run through the same `prompt_iters` rounds as forward, with the same host
        checks per round; FPS, kNN and the ground-truth prompt sampler stay inside each cloud, and the decoder also computes
        the padded rows, which are dropped.  Returns B lists; list b has forward's structure for cloud b alone (masks
        [M, C, N_b], prompt_masks [M, N_b], prompt_coords [M, t + 1, 3], ...) as views of the batch outputs.
        Refused before any device work: training mode or is_eval=False (NotImplementedError: the random training sampler
        is not length-aware), the Voronoi tokenizer and clouds below the first-level group shape (varlen_clouds), and
        shape mismatches (ValueError)."""
        if self.training or not is_eval:
            raise NotImplementedError("forward_varlen runs the evaluation loop only: call model.eval() and pass is_eval=True "
                                      "(the random training sampler does not take clouds of different sizes)")
        sizes = self.varlen_clouds(coords, features)
        gts = self._varlen_gt(gt_masks, sizes)
        B, M = len(sizes), gts[0].shape[0]
        xyz, rgb, lengths = ops.pad_clouds(coords, features)
        gt = torch.zeros((B, M, xyz.shape[1]), dtype=torch.bool, device=xyz.device)
        for b, (g, n) in enumerate(zip(gts, sizes)):
            gt[b, :, :n].copy_(g, non_blocking=True)
        enc = self._encode(xyz, rgb, lengths)
        return self._split_varlen(self._eval_loop(enc, xyz, gt, is_eval=True, lengths=lengths), sizes, M)

    @staticmethod
    def _split_varlen(outputs, sizes: List[int], M: int) -> List[List[Dict[str, torch.Tensor]]]:
        """Per-iteration dicts of a padded batch -> one list per cloud, each field a view cut to cloud b."""
        per = []
        for b, n in enumerate(sizes):
            s = slice(b * M, (b + 1) * M)
            per.append([dict(prompt_coords=o["prompt_coords"][s], prompt_labels=o["prompt_labels"][s],
                             masks=o["masks"][s, :, :n], iou_preds=o["iou_preds"][s],
                             max_iou_pred_ind=o["max_iou_pred_ind"][s] if torch.is_tensor(o["max_iou_pred_ind"]) else o["max_iou_pred_ind"],
                             prompt_masks=o["prompt_masks"][s, :n]) for o in outputs])
        return per

    def predict_masks_varlen(self, coords: Sequence[torch.Tensor], features: Sequence[torch.Tensor], prompt_coords: torch.Tensor,
                             prompt_labels: torch.Tensor, prompt_masks: Optional[Sequence[torch.Tensor]] = None,
                             multimask_output: bool = True) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """predict_masks on B clouds of different sizes with one encode and one decode: coords / features are sequences of
        [N_b, 3] tensors, prompt_coords [B, M, Q, 3], prompt_labels [B, M, Q], prompt_masks None or a sequence of [M, N_b]
        tensors.  Returns B pairs (masks [M, C, N_b], iou_preds [M, C]).  The clouds are padded to N_max = max N_b
        (ops.pad_clouds); farthest-point sampling and the kNN grouping stay inside each cloud, and the decoder also computes
        logits for the padded rows, which are dropped: its cost grows with B * N_max - sum(N_b).  Group clouds of similar
        sizes to keep that small."""
        sizes = self.varlen_clouds(coords, features)
        B = len(sizes)
        if prompt_coords.dim() != 4 or prompt_coords.shape[0] != B or prompt_labels.shape != prompt_coords.shape[:3]:
            raise ValueError(f"prompt_coords must be [B={B}, M, Q, 3] and prompt_labels [B, M, Q], got "
                             f"{tuple(prompt_coords.shape)} and {tuple(prompt_labels.shape)}")
        M, Q = prompt_coords.shape[1], prompt_coords.shape[2]
        pm = None
        if prompt_masks is not None:
            prompt_masks = list(prompt_masks)
            if len(prompt_masks) != B or any(t.shape != (M, n) for t, n in zip(prompt_masks, sizes)):
                raise ValueError(f"prompt_masks must be {B} tensors [M={M}, N_b]")
            pm = torch.nn.utils.rnn.pad_sequence([t.transpose(0, 1) for t in prompt_masks], batch_first=True)
            pm = pm.transpose(1, 2).reshape(B * M, -1)
        xyz, rgb, lengths = ops.pad_clouds(coords, features)
        enc = self._encode(xyz, rgb, lengths)
        masks, iou = self._decode(enc, prompt_coords.reshape(B * M, Q, 3), prompt_labels.reshape(B * M, Q), pm,
                                  bool(multimask_output))
        return [(masks[b * M:(b + 1) * M, :, :n], iou[b * M:(b + 1) * M]) for b, n in enumerate(sizes)]

    def _sample_prompts(self, coords, gt_masks, prompt_masks, is_eval, lengths=None):
        from .prompt_sampling import sample_prompts_adapter

        return sample_prompts_adapter(coords, gt_masks, prompt_masks, is_eval=is_eval, lengths=lengths)

    # ------------------------------------------------------------------------------------------
    def set_pointcloud(self, xyz: torch.Tensor, rgb: torch.Tensor):
        """demo/app.py:199 - encode once, keep the embeddings for subsequent prompt decodes."""
        key = (xyz.data_ptr(), xyz._version, tuple(xyz.shape), rgb.data_ptr(), rgb._version) + self._group_shape()
        if self._cloud is not None and self._cloud_key == key:
            return  # same tensors, unmodified: keep the embeddings (the demo calls this on every click)
        with torch.no_grad():
            self._cloud = self._encode(xyz.float().contiguous(), rgb.float().contiguous())
        self._cloud_key = key
        self._cloud_keepalive = (xyz, rgb)  # the key holds data_ptr()s: keep the storages alive so they cannot be recycled

    def predict_masks(self, *args, **kwargs):
        """Two call forms:
        reference (pc_sam.py:37-45): predict_masks(coords, features, prompt_coords, prompt_labels,
            prompt_masks=None, multimask_output=True) -> (masks [B*M,C,N], iou_preds [B*M,C])
        demo (demo/app.py:200-202):  predict_masks(prompt_points [1,P,3], prompt_labels [1,P],
            prompt_mask [1,N] | None, multimask_output) -> (mask, scores, logits) after set_pointcloud()."""
        names = ("coords", "features", "prompt_coords", "prompt_labels", "prompt_masks", "multimask_output")
        demo_form = "prompt_points" in kwargs or "prompt_mask" in kwargs or (
            len(args) >= 2 and torch.is_tensor(args[1]) and args[1].dim() == 2)
        if demo_form:
            dn = ("prompt_points", "prompt_labels", "prompt_mask", "multimask_output")
            a = dict(zip(dn, args))
            a.update(kwargs)
            if self._cloud is None:
                raise RuntimeError("predict_masks(prompt_points, ...) requires set_pointcloud() first")
            with torch.no_grad():
                logits, scores = self._decode(self._cloud, a["prompt_points"], a["prompt_labels"], a.get("prompt_mask"),
                                              bool(a.get("multimask_output", True)))
            return logits, scores, logits
        a = dict(zip(names, args))
        a.update(kwargs)
        enc = self._encode(a["coords"].float().contiguous(), a["features"].float().contiguous())
        return self._decode(enc, a["prompt_coords"], a["prompt_labels"], a.get("prompt_masks"),
                            bool(a.get("multimask_output", True)))

    def make_predictor(self, batch_size: int, num_points: int, num_prompts: int, multimask_output: bool = True,
                       use_graph: bool = True):
        """Fixed-shape predictor that replays the whole path as one CUDA graph (serving entry point)."""
        from psam_b200.predictor import GraphPredictor

        return GraphPredictor(self, batch_size, num_points, num_prompts, multimask_output, use_graph)

    def make_pipelined_predictor(self, batch_size: int, num_points: int, num_prompts: int, depth: int = 3,
                                 multimask_output: bool = True, use_graph: bool = True):
        """`depth` graph predictors on separate streams, used round-robin so consecutive clouds overlap."""
        from psam_b200.predictor import PipelinedPredictor

        return PipelinedPredictor(self, batch_size, num_points, num_prompts, depth, multimask_output, use_graph)

    def make_iterative_predictor(self, batch_size: int, num_masks: int, num_points: int, use_graph: bool = True,
                                 throughput_tiles: bool = False):
        """forward(is_eval=True) - encoder, then `prompt_iters` rounds of (GT prompt sampling, prompt / mask encoders,
        decoder, best-mask feedback) - captured as ONE CUDA graph with no host synchronisation inside.
        throughput_tiles: capture with the SM-time-optimal GEMM tile policy (several predictors in flight on one GPU)."""
        from psam_b200.predictor import IterativeGraphPredictor

        return IterativeGraphPredictor(self, batch_size, num_masks, num_points, use_graph, throughput_tiles=throughput_tiles)

    def make_iterative_predictor_varlen(self, batch_size: int, num_masks: int, max_points: int, use_graph: bool = True,
                                        throughput_tiles: bool = False):
        """forward_varlen as ONE CUDA graph for every batch of up to batch_size clouds of at most max_points points each
        with num_masks ground-truth masks: the lengths live in a device buffer that FPS, kNN and the prompt sampler read,
        so no cloud size is baked into the graph.  Returns forward_varlen's structure (views valid until the next call)."""
        from psam_b200.predictor import IterativeGraphPredictorVarlen

        return IterativeGraphPredictorVarlen(self, batch_size, num_masks, max_points, use_graph, throughput_tiles=throughput_tiles)

    # ------------------------------------------------------------------------------------------
    def predict_iterative(self, coords, features, prompt_coords_seq: List[torch.Tensor],
                          prompt_labels_seq: List[torch.Tensor]) -> List[Dict[str, torch.Tensor]]:
        """Loop body of forward (pc_sam.py:139-194) with externally supplied prompts: iteration t appends
        prompt_coords_seq[t]; multimask only at t=0; the most confident mask is fed back as prompt mask."""
        enc = self._encode(coords.float().contiguous(), features.float().contiguous())
        outs, pm = [], None
        pc, pl = prompt_coords_seq[0][:, :0], prompt_labels_seq[0][:, :0]
        for t in range(len(prompt_coords_seq)):
            pc = torch.cat([pc, prompt_coords_seq[t]], dim=1)
            pl = torch.cat([pl, prompt_labels_seq[t]], dim=1)
            masks, iou = self._decode(enc, pc, pl, pm, t == 0, center_idx=self._center_idx(enc))
            if t == 0:
                best = torch.argmax(iou, dim=1)
                pm = batch_index_select(masks, best, dim=1)
            else:
                best = 0
                pm = masks[:, 0]
            outs.append(dict(prompt_coords=pc, prompt_labels=pl, masks=masks, iou_preds=iou, max_iou_pred_ind=best,
                             prompt_masks=pm))
        return outs

    def forward(self, coords=None, features=None, gt_masks=None, is_eval=False, xyz=None, rgb=None, mask=None):
        """Reference forward (pc_sam.py:90-196); also accepts the xyz/rgb/mask spelling used by
        evaluation/inference.py:67-68.  Prompts are sampled from the ground truth with the reference's
        sampler (pc_sam/model/common.py:287-474) restated in pc_sam.model.prompt_sampling."""
        if self.training:
            self._check_trainable()  # before any device work
        coords = coords if coords is not None else xyz
        features = features if features is not None else rgb
        gt_masks = gt_masks if gt_masks is not None else mask
        if gt_masks.dim() == 2:
            gt_masks = gt_masks.unsqueeze(1)
        gt_masks = gt_masks.bool()
        if self.training:
            return self._train_loop(coords.float().contiguous(), features.float().contiguous(), gt_masks, is_eval)
        enc = self._encode(coords.float().contiguous(), features.float().contiguous())
        return self._eval_loop(enc, coords, gt_masks, is_eval)

    def _check_trainable(self):
        """Training mode fine-tunes mask_decoder on a frozen encoder: every other parameter must have requires_grad=False.
        A block with active dropout or drop-path is refused by the engine's block validation (the frozen encoder runs
        deterministically, as in eval mode)."""
        for name, p in self.named_parameters():
            if p.requires_grad and not name.startswith("mask_decoder."):
                raise NotImplementedError(
                    f"training mode fine-tunes mask_decoder only, but parameter '{name}' has requires_grad=True: freeze "
                    "everything else first with model.requires_grad_(False); model.mask_decoder.requires_grad_(True)")
        engine.validate_transformer(self.pc_encoder.transformer)

    def _train_loop(self, coords, features, gt_masks, is_eval):
        """The reference's training forward (pc_sam.py:112-196) with only mask_decoder differentiable: the encoder, the
        point and mask prompt encoders run through the engine as in eval mode, the decoder through psam_b200.train.  Two
        iterations refine the mask without a new prompt (the last one and one drawn with torch.randint on the global CPU
        generator, as in the reference); the fed-back mask reaches the mask encoder detached."""
        from psam_b200 import train

        B, M = coords.shape[0], gt_masks.shape[1]
        refine = []
        if self.enable_mask_refinement_iterations:
            refine = [self.prompt_iters - 1]
            if self.prompt_iters > 1:
                refine.append(torch.randint(1, self.prompt_iters, (1,)).item())
        with torch.no_grad():
            enc = self._encode(coords, features)
        patches = enc["patches"]
        outputs = []
        pc = coords.new_empty((B * M, 0, 3))
        pl = gt_masks.new_empty((B * M, 0))
        pm = None
        for i in range(self.prompt_iters):
            if i == 0 or i not in refine:
                npc, npl = self._sample_prompts(coords, gt_masks, pm, is_eval)
                pc = torch.cat([pc, npc], dim=1)
                pl = torch.cat([pl, npl], dim=1)
            with torch.no_grad():
                sparse = engine.run_point_encoder(self.point_encoder, pc, pl, check=False)
                dense = self.mask_encoder(None if pm is None else pm.detach(), coords, patches["centers"], patches["knn_idx"],
                                          center_idx=self._center_idx(enc))
            masks, iou = train.run_mask_decoder_train(self.mask_decoder, enc["pc_embeddings"], enc["pc_pe"], sparse, dense,
                                                      enc["aux"], multimask_output=(i == 0))
            engine.raise_if_out_of_range(masks.device)
            if i == 0:
                best = torch.argmax(iou.detach(), dim=1)
                pm = batch_index_select(masks, best, dim=1)
            else:
                best = 0
                pm = masks[:, 0]
            outputs.append(dict(prompt_coords=pc, prompt_labels=pl, masks=masks, iou_preds=iou, max_iou_pred_ind=best,
                                prompt_masks=pm))
        return outputs

    def _eval_loop(self, enc, coords, gt_masks, is_eval, lengths=None):
        """The body of forward after the encode: `prompt_iters` rounds of prompt sampling from the ground truth
        gt_masks [B, M, N] bool, decode and best-mask feedback.  lengths: padded clouds (forward_varlen)."""
        B, M = coords.shape[0], gt_masks.shape[1]
        outputs = []
        pc = coords.new_empty((B * M, 0, 3))
        pl = gt_masks.new_empty((B * M, 0))
        pm = None
        for i in range(self.prompt_iters):
            npc, npl = self._sample_prompts(coords, gt_masks, pm, is_eval, lengths)
            pc = torch.cat([pc, npc], dim=1)
            pl = torch.cat([pl, npl], dim=1)
            masks, iou = self._decode(enc, pc, pl, pm, i == 0, center_idx=self._center_idx(enc))
            if i == 0:
                best = torch.argmax(iou, dim=1)
                pm = batch_index_select(masks, best, dim=1)
            else:
                best = 0
                pm = masks[:, 0]
            outputs.append(dict(prompt_coords=pc, prompt_labels=pl, masks=masks, iou_preds=iou, max_iou_pred_ind=best,
                                prompt_masks=pm))
        return outputs


PointSAM = PointCloudSAM


class PointCloudSAMHier(PointCloudSAM):
    """PointCloudSAMHier (/root/reference/pc_sam/model/pc_sam.py:377-496): PatchEmbedHier tokenizer, MaskEncoderHier and
    MaskDecoderHier; the transformer sees the level-2 patches, the decoder upscales level 2 -> level 1 -> points.

    forward(is_eval=False) is the reference's loop (random prompt of the error region every round, pc_sam.py:434).
    Extensions over the reference, where its inherited methods fail: forward(is_eval=True) uses the ground-truth border
    sampler exactly as PointCloudSAM.forward(is_eval=True) (so the evaluation driver and the iterative graph predictor run
    this model), and predict_masks / predict_iterative / set_pointcloud run one round of the forward loop body with the
    given prompts (the reference's inherited predict_masks indexes the list of patch levels with a string, pc_sam.py:54)."""

    def _encode(self, coords, features, lengths=None):
        pc_embeddings, patches = self._run_encoder(coords, features, lengths)
        p1, p2 = patches
        aux1 = AuxInputs(coords=coords, features=features, centers=p1["centers"])
        aux2 = AuxInputs(coords=p1["centers"], features=p1["embeddings"], centers=p2["centers"])
        engine.hier_embedding_term(self.mask_decoder, aux2)  # per cloud: kept by set_pointcloud across prompts
        pc_pe = engine.run_pos_embedding(self.point_encoder.pe_layer, p2["centers"], check=False)
        return dict(pc_embeddings=pc_embeddings, patches=patches, aux=(aux1, aux2), pc_pe=pc_pe, coords=coords)

    def _decode_unchecked(self, enc, prompt_coords, prompt_labels, prompt_masks, multimask_output, center_idx=None):
        p1, p2 = enc["patches"]
        sparse = engine.run_point_encoder(self.point_encoder, prompt_coords, prompt_labels, check=False)
        dense = self.mask_encoder(prompt_masks, enc["coords"], p1["centers"], p1["knn_idx"], p2["centers"], p2["knn_idx"])
        if isinstance(dense, list):  # pc_sam.py:452-460: the last level, already batched B*M
            dense = dense[-1]
        aux1, aux2 = enc["aux"]
        return self.mask_decoder(enc["pc_embeddings"], enc["pc_pe"], sparse, dense, aux_inputs1=aux1, aux_inputs2=aux2,
                                 multimask_output=multimask_output)

    def _center_idx(self, enc):
        return None  # MaskEncoderHier has no centralize_features

    def _check_trainable(self):
        raise NotImplementedError("training mode of PointCloudSAMHier is not implemented (fine-tuning covers PointCloudSAM's "
                                  "MaskDecoder): call model.eval()")

    def _group_shape(self) -> tuple:
        pe = self.pc_encoder.patch_embed
        return pe.grouper1.num_groups, pe.grouper1.group_size, pe.grouper2.num_groups, pe.grouper2.group_size

    def _sample_prompts(self, coords, gt_masks, prompt_masks, is_eval, lengths=None):
        if is_eval or lengths is not None:
            return super()._sample_prompts(coords, gt_masks, prompt_masks, is_eval, lengths)
        from .prompt_sampling import sample_prompts

        return sample_prompts(coords, gt_masks, prompt_masks)


def build_point_sam(encoder: str = "eva02_large_patch14_448", num_patches: int = 512, patch_size: int = 64,
                    embed_dim: int = 256, prompt_iters: int = 5) -> PointCloudSAM:
    """Dependency-free mirror of configs/model/{base,default,giant}.yaml (hydra/timm are absent offline)."""
    from .eva import create_model
    from .pc_encoder import PatchEmbed
    from .transformer import TwoWayTransformer

    pe = PatchEmbed(6, 512, num_patches, patch_size)
    enc = PointCloudEncoder(pe, create_model(encoder), embed_dim)
    me = MaskEncoder(embed_dim)
    md = MaskDecoder(embed_dim, TwoWayTransformer(2, embed_dim, 8, 2048))
    return PointCloudSAM(enc, me, md, prompt_iters).eval()


def build_point_sam_hier(encoder: str = "eva02_large_patch14_448", num_patches=(2048, 512), patch_size=(32, 32),
                         radius=(0.05, 0.1), prompt_iters: int = 8, embed_dim: int = 256) -> PointCloudSAMHier:
    """Dependency-free mirror of configs/model/hier.yaml."""
    from .eva import create_model
    from .mask_decoder import MaskDecoderHier
    from .pc_encoder import PatchEmbedHier
    from .prompt_encoder import MaskEncoderHier
    from .transformer import TwoWayTransformer

    radius = list(radius) if radius is not None else None
    pe = PatchEmbedHier(6, 512, list(num_patches), list(patch_size), radius)
    enc = PointCloudEncoder(pe, create_model(encoder), embed_dim)
    me = MaskEncoderHier(embed_dim, radius=radius)
    md = MaskDecoderHier(embed_dim, TwoWayTransformer(2, embed_dim, 8, 2048))
    return PointCloudSAMHier(enc, me, md, prompt_iters).eval()
