"""/root/reference/pc_sam/model/mask_decoder.py:12-370."""
from __future__ import annotations

import dataclasses
from typing import Tuple

import torch
from torch import nn

from psam_b200 import engine


@dataclasses.dataclass
class AuxInputs:
    coords: torch.Tensor
    features: torch.Tensor
    centers: torch.Tensor
    interp_index: torch.Tensor = None
    interp_weight: torch.Tensor = None


class MLP(nn.Module):
    def __init__(self, input_dim: int, hidden_dim: int, output_dim: int, num_layers: int, sigmoid_output: bool = False):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))
        self.sigmoid_output = sigmoid_output


class MaskDecoder(nn.Module):
    def __init__(self, transformer_dim: int, transformer: nn.Module, num_multimask_outputs: int = 3,
                 iou_head_depth: int = 3, iou_head_hidden_dim: int = 256) -> None:
        super().__init__()
        if iou_head_depth != 3:
            raise NotImplementedError("the fused decoder implements the released iou_head_depth=3")
        self.transformer_dim = transformer_dim
        self.transformer = transformer
        self.num_multimask_outputs = num_multimask_outputs
        self.iou_token = nn.Embedding(1, transformer_dim)
        self.num_mask_tokens = num_multimask_outputs + 1
        self.mask_tokens = nn.Embedding(self.num_mask_tokens, transformer_dim)
        self.output_hypernetworks_mlps = nn.ModuleList(
            [MLP(transformer_dim, transformer_dim, transformer_dim, 3) for _ in range(self.num_mask_tokens)])
        self.output_upscaling = nn.Sequential(
            nn.Linear(transformer_dim, transformer_dim), nn.LayerNorm(transformer_dim), nn.GELU(),
            nn.Linear(transformer_dim, transformer_dim), nn.GELU())
        self.iou_prediction_head = MLP(transformer_dim, iou_head_hidden_dim, self.num_mask_tokens, iou_head_depth)

    def forward(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings, aux_inputs: AuxInputs,
                multimask_output: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        return engine.run_mask_decoder(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings,
                                       aux_inputs, multimask_output)


class MaskDecoderHier(nn.Module):
    """mask_decoder.py:214-370: the same two-way transformer and heads, upscaled in two stages (patches -> level-1 centres,
    with the tokenizer's level-1 embeddings concatenated -> points).  The hyper-network MLPs end in D/2."""

    def __init__(self, transformer_dim: int, transformer: nn.Module, num_multimask_outputs: int = 3, iou_head_depth: int = 3,
                 iou_head_hidden_dim: int = 256, encoder_dim: int = 128) -> None:
        super().__init__()
        if iou_head_depth != 3:
            raise NotImplementedError("the fused decoder implements the released iou_head_depth=3")
        self.transformer_dim = transformer_dim
        self.transformer = transformer
        self.num_multimask_outputs = num_multimask_outputs
        self.iou_token = nn.Embedding(1, transformer_dim)
        self.num_mask_tokens = num_multimask_outputs + 1
        self.mask_tokens = nn.Embedding(self.num_mask_tokens, transformer_dim)
        self.output_hypernetworks_mlps = nn.ModuleList(
            [MLP(transformer_dim, transformer_dim, transformer_dim // 2, 3) for _ in range(self.num_mask_tokens)])
        self.output_upscaling2 = nn.Sequential(
            nn.Linear(transformer_dim + encoder_dim, transformer_dim), nn.LayerNorm(transformer_dim), nn.GELU(),
            nn.Linear(transformer_dim, transformer_dim))
        self.output_upscaling1 = nn.Sequential(
            nn.Linear(transformer_dim, transformer_dim // 2), nn.LayerNorm(transformer_dim // 2), nn.GELU(),
            nn.Linear(transformer_dim // 2, transformer_dim // 2), nn.GELU())
        self.iou_prediction_head = MLP(transformer_dim, iou_head_hidden_dim, self.num_mask_tokens, iou_head_depth)

    def forward(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings, aux_inputs1: AuxInputs,
                aux_inputs2: AuxInputs, multimask_output: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        """aux_inputs1: points <- level-1 centres; aux_inputs2: level-1 centres <- level-2 centres, with the level-1
        embeddings as features.  Both cache their interpolation weights, as in the reference."""
        return engine.run_mask_decoder(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings,
                                       (aux_inputs1, aux_inputs2), multimask_output)
