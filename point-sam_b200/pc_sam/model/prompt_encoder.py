"""/root/reference/pc_sam/model/prompt_encoder.py:13-133."""
from __future__ import annotations

from typing import List, Optional, Union

import torch
from torch import nn

from psam_b200 import engine

from .common import PatchEncoder


class PositionEmbeddingRandom(nn.Module):
    def __init__(self, num_pos_feats: int = 64, scale: Optional[float] = None) -> None:
        super().__init__()
        if scale is None or scale <= 0.0:
            scale = 1.0
        self.register_buffer("positional_encoding_gaussian_matrix", scale * torch.randn((3, num_pos_feats)))

    def forward(self, coords: torch.Tensor) -> torch.Tensor:
        """Raises ValueError for coordinates outside [-1, 1] like the reference (:44-46)."""
        return engine.run_pos_embedding(self, coords)


class PointEncoder(nn.Module):
    def __init__(self, embed_dim: int):
        super().__init__()
        self.embed_dim = embed_dim
        self.pe_layer = PositionEmbeddingRandom(embed_dim // 2)
        self.num_point_embeddings: int = 2
        self.point_embeddings = nn.ModuleList([nn.Embedding(1, embed_dim) for _ in range(2)])

    def forward(self, points: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        return engine.run_point_encoder(self, points, labels)


class MaskEncoder(nn.Module):
    def __init__(self, embed_dim, in_channels=4, radius=None, centralize_features=False):
        super().__init__()
        self.embed_dim = embed_dim
        self.in_channels = in_channels
        self.radius = radius
        self.centralize_features = centralize_features
        self.patch_encoder = PatchEncoder(in_channels, embed_dim, [128, 512])
        self.no_mask_embed = nn.Embedding(1, embed_dim)

    def forward(self, masks: Union[torch.Tensor, None], coords, centers, knn_idx, center_idx=None) -> torch.Tensor:
        return engine.run_mask_encoder(self, masks, coords, centers, knn_idx, center_idx)


class MaskEncoderHier(nn.Module):
    """/root/reference/pc_sam/model/prompt_encoder.py:136-183 (two-level PointNet++-style mask encoder)."""

    def __init__(self, embed_dim, in_channels=4, radius: Optional[List[float]] = None):
        super().__init__()
        self.embed_dim = embed_dim
        self.in_channels = in_channels
        self.radius = radius
        self.patch_encoder1 = PatchEncoder(in_channels, 128, [64, 128])
        self.patch_encoder2 = PatchEncoder(128 + 3, embed_dim, [128, 256])
        self.no_mask_embed = nn.Embedding(1, embed_dim)

    def forward(self, masks: Union[torch.Tensor, None], coords, centers1, knn_idx1, centers2, knn_idx2):
        """No mask: no_mask_embed broadcast over [B, G2, D]; otherwise the list [x1 [B*M, G1, 128], x2 [B*M, G2, D]]."""
        return engine.run_mask_encoder_hier(self, masks, coords, centers1, knn_idx1, centers2, knn_idx2)
