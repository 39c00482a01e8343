"""ORACLE (test infrastructure, NOT product code).

CPU / plain-PyTorch fp32 restatement of the Point-SAM hot path, used only by tests/,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg as the
checker and the CPU baseline.  The product path (``point-sam_b200/``) never imports this file.

Every class follows the reference module of the same name and keeps the reference's
state-dict key names so that weights can be exchanged with ``load_state_dict``:

* tokenizer             pc_sam/model/common.py:27-123, 126-187, 238-284
* PatchEncoder          pc_sam/model/common.py:477-506
* PatchEmbed / encoder  pc_sam/model/pc_encoder.py:13-41, 84-145
* prompt / mask encoder pc_sam/model/prompt_encoder.py:13-133
* mask decoder          pc_sam/model/mask_decoder.py:21-211
* two-way transformer   pc_sam/model/transformer.py:15-253
* PointCloudSAM         pc_sam/model/pc_sam.py:20-196
* FPS                   third_party/torkit3d/torkit3d/csrc/cuda/sample_farthest_points_kernel.cu:8-104
                        (restated in oracle/tokenizer_ref.c, called here through ctypes)
* EVA / EVA02 blocks    timm (un-vendored pip dependency "timm>=0.9.0", reference README.md:49):
                        timm/models/eva.py EvaAttention / EvaBlock / Eva and timm/layers/mlp.py
                        SwiGLU / Mlp, restated from the published source.  PARITY UNPINNED for this
                        part: timm is not installable offline and the reference holds no test or
                        golden vector at this boundary.

Distance semantics: the reference's ``torch.cdist`` uses the matmul expansion whose rounding noise
differs between backends.  ``exact_dist=True`` (default) uses the
direct-difference form ``compute_mode="donot_use_mm_for_euclid_dist"`` which is what the CUDA path
implements; ``exact_dist=False`` reproduces the reference call literally.
"""
from __future__ import annotations

import dataclasses
import math
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import tokenizer_ref

EXACT_DIST = True


# --------------------------------------------------------------------------------------------
# tokenizer pieces
# --------------------------------------------------------------------------------------------
def batch_index_select(x: torch.Tensor, index: torch.Tensor, dim: int) -> torch.Tensor:
    """torkit3d/nn/functional.py:34-69 (batched gather)."""
    squeeze = index.dim() == 1
    if squeeze:
        index = index.unsqueeze(1)
    views = [1] * x.dim()
    views[0] = index.size(0)
    views[dim] = index.size(1)
    shape = list(x.shape)
    shape[dim] = -1
    out = torch.gather(x, dim, index.view(views).expand(shape))
    return out.squeeze(1) if squeeze else out


def sample_farthest_points(points: torch.Tensor, num_samples: int) -> torch.Tensor:
    """FPS indices [B, G] int64 with the reference kernel's arithmetic and tie-break."""
    pts = points.detach().cpu().float().contiguous().numpy()
    return torch.from_numpy(tokenizer_ref.fps(pts, num_samples)).to(points.device)


def knn_points(query, key, k: int, sorted: bool = False):
    """pc_sam/model/common.py:27-56."""
    if EXACT_DIST:
        distance = torch.cdist(query, key, compute_mode="donot_use_mm_for_euclid_dist")
    else:
        distance = torch.cdist(query, key)
    if k == 1:
        return torch.min(distance, dim=2, keepdim=True)
    return torch.topk(distance, k, dim=2, largest=False, sorted=sorted)


def compute_interp_weights(query, key, k=3, eps=1e-8):
    """pc_sam/model/common.py:238-255."""
    dist, idx = knn_points(query, key, k)
    inv = 1.0 / torch.clamp(dist.square(), min=eps)
    return idx, inv / inv.sum(dim=2, keepdim=True)


def interpolate_features(x, index, weight):
    """pc_sam/model/common.py:258-274."""
    B, Nq, K = index.shape
    off = torch.arange(B, device=x.device).reshape(-1, 1, 1) * x.shape[1]
    g = x.flatten(0, 1)[(index + off).flatten()].reshape(B, Nq, K, x.shape[-1])
    return (g * weight.unsqueeze(-1)).sum(-2)


def repeat_interleave(x, repeats: int, dim: int):
    """pc_sam/model/common.py:277-284."""
    if repeats == 1:
        return x
    shape = list(x.shape)
    shape.insert(dim + 1, repeats)
    return x.unsqueeze(dim + 1).expand(shape).flatten(dim, dim + 1)


class KNNGrouper(nn.Module):
    """pc_sam/model/common.py:59-123."""

    def __init__(self, num_groups, group_size, radius=None, centralize_features=False):
        super().__init__()
        self.num_groups, self.group_size = num_groups, group_size
        self.radius, self.centralize_features = radius, centralize_features

    def forward(self, xyz, features, use_fps=True):
        B, N, _ = xyz.shape
        with torch.no_grad():
            if use_fps:
                fps_idx = sample_farthest_points(xyz.float(), self.num_groups)
                centers = batch_index_select(xyz, fps_idx, dim=1)
            else:
                fps_idx = torch.arange(self.num_groups, device=xyz.device).expand(B, -1)
                centers = xyz[:, : self.num_groups]
            _, knn_idx = knn_points(centers, xyz, self.group_size)
        flat = (knn_idx + torch.arange(B, device=xyz.device).reshape(-1, 1, 1) * N).reshape(-1)
        nbr_xyz = xyz.reshape(-1, 3)[flat].reshape(B, self.num_groups, self.group_size, 3)
        nbr_xyz = nbr_xyz - centers.unsqueeze(2)
        if self.radius is not None:
            nbr_xyz = nbr_xyz / self.radius
        C = features.shape[-1]
        nbr_feats = features.reshape(-1, C)[flat].reshape(B, self.num_groups, self.group_size, C)
        parts = [nbr_xyz, nbr_feats]
        if self.centralize_features:
            parts.append(nbr_feats - batch_index_select(features, fps_idx, dim=1).unsqueeze(2))
        return dict(features=torch.cat(parts, dim=-1), centers=centers, knn_idx=knn_idx, fps_idx=fps_idx)


def group_with_centers_and_knn(xyz, features, centers, knn_idx, radius=None,
                               centralize_features=False, center_idx=None):
    """pc_sam/model/common.py:126-187 (features may carry M masks per cloud)."""
    B, N, _ = xyz.shape
    _, L, K = knn_idx.shape
    flat = (knn_idx + torch.arange(B, device=xyz.device).reshape(-1, 1, 1) * N).reshape(-1)
    nbr_xyz = xyz.reshape(-1, 3)[flat].reshape(B, L, K, 3) - centers.unsqueeze(2)
    if radius is not None:
        nbr_xyz = nbr_xyz / radius
    B2 = features.shape[0]
    rep = B2 // B
    knn2 = torch.repeat_interleave(knn_idx, rep, dim=0)
    flat2 = (knn2 + torch.arange(B2, device=xyz.device).reshape(-1, 1, 1) * N).reshape(-1)
    C = features.shape[-1]
    nbr_feats = features.reshape(-1, C)[flat2].reshape(B2, L, K, C)
    parts = [torch.repeat_interleave(nbr_xyz, rep, dim=0), nbr_feats]
    if centralize_features:
        cidx = torch.repeat_interleave(center_idx, rep, dim=0)
        parts.append(nbr_feats - batch_index_select(features, cidx, dim=1).unsqueeze(2))
    return torch.cat(parts, dim=-1)


class PatchEncoder(nn.Module):
    """pc_sam/model/common.py:477-506."""

    def __init__(self, in_channels, out_channels, hidden_dims):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        h0, h1 = hidden_dims
        self.conv1 = nn.Sequential(nn.Linear(in_channels, h0), nn.LayerNorm(h0), nn.GELU(), nn.Linear(h0, h0))
        self.conv2 = nn.Sequential(nn.Linear(h0 * 2, h1), nn.LayerNorm(h1), nn.GELU(), nn.Linear(h1, out_channels))

    def forward(self, patches):
        x = self.conv1(patches)
        y = torch.max(x, dim=-2, keepdim=True).values
        x = self.conv2(torch.cat([y.expand_as(x), x], dim=-1))
        return torch.max(x, dim=-2).values


class PatchEmbed(nn.Module):
    """pc_sam/model/pc_encoder.py:13-41."""

    def __init__(self, in_channels, out_channels, num_patches, patch_size, radius=None, centralize_features=False):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.grouper = KNNGrouper(num_patches, patch_size, radius=radius, centralize_features=centralize_features)
        self.patch_encoder = PatchEncoder(in_channels, out_channels, [128, 512])

    def forward(self, coords, features):
        patches = self.grouper(coords, features)
        patches["embeddings"] = self.patch_encoder(patches["features"])
        return patches


class NNGrouper(nn.Module):
    """pc_sam/model/common.py:190-212 (Voronoi grouping: every point joins its nearest FPS centre)."""

    def __init__(self, num_groups: int):
        super().__init__()
        self.num_groups = num_groups

    def forward(self, xyz, features):
        with torch.no_grad():
            fps_idx = sample_farthest_points(xyz.float(), self.num_groups)
            centers = batch_index_select(xyz, fps_idx, dim=1)
            _, nn_idx = knn_points(xyz, centers, 1)
        nn_idx = nn_idx.squeeze(-1)
        return dict(features=group_with_centers_and_nn(xyz, features, centers, nn_idx), centers=centers, nn_idx=nn_idx)


def group_with_centers_and_nn(xyz, features, centers, nn_idx):
    """pc_sam/model/common.py:214-236."""
    nbr_xyz = xyz - batch_index_select(centers, nn_idx, dim=1)
    dist = torch.linalg.norm(nbr_xyz, dim=-1, keepdim=True, ord=2)
    nbr_xyz = nbr_xyz / torch.clamp(dist, min=1e-8)
    return torch.cat([nbr_xyz, dist, features], dim=-1)


class Block(nn.Module):
    """pc_sam/model/pc_encoder.py:147-162."""

    def __init__(self, in_channels, hidden_dim, out_channels):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(in_channels, hidden_dim), nn.GELU(), nn.LayerNorm(hidden_dim),
                                 nn.Linear(hidden_dim, out_channels))
        self.norm = nn.LayerNorm(out_channels)

    def forward(self, x):
        return x + self.mlp(self.norm(x))


class PatchEmbedNN(nn.Module):
    """pc_sam/model/pc_encoder.py:165-197."""

    def __init__(self, in_channels, hidden_dim, out_channels, num_patches):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        hidden_dim = hidden_dim or out_channels
        self.grouper = NNGrouper(num_patches)
        self.in_proj = nn.Linear(in_channels, hidden_dim)
        self.blocks1 = nn.Sequential(*[Block(hidden_dim, hidden_dim, hidden_dim) for _ in range(3)])
        self.blocks2 = nn.Sequential(*[Block(hidden_dim, hidden_dim, hidden_dim) for _ in range(3)])
        self.norm = nn.LayerNorm(hidden_dim)
        self.out_proj = nn.Linear(hidden_dim, out_channels)

    def forward(self, coords, features):
        patches = self.grouper(coords, features)
        nn_idx = patches["nn_idx"]
        x = self.blocks1(self.in_proj(patches["features"]))
        y = x.new_zeros(x.shape[0], self.grouper.num_groups, x.shape[-1])
        y.scatter_reduce_(1, nn_idx.unsqueeze(-1).expand_as(x), x, "amax", include_self=False)
        patches["embeddings"] = self.out_proj(self.norm(self.blocks2(y)))
        return patches


class PatchEmbedHier(nn.Module):
    """pc_sam/model/pc_encoder.py:200-239."""

    def __init__(self, in_channels, out_channels, num_patches, patch_size, radius=None):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.grouper1 = KNNGrouper(num_patches[0], patch_size[0], radius=radius[0] if radius else None)
        self.patch_encoder1 = PatchEncoder(in_channels, 128, [64, 128])
        self.grouper2 = KNNGrouper(num_patches[1], patch_size[1], radius=radius[1] if radius else None)
        self.patch_encoder2 = PatchEncoder(128 + 3, out_channels, [128, 256])

    def forward(self, coords, features):
        patches1 = self.grouper1(coords, features)
        x1 = self.patch_encoder1(patches1["features"])
        patches1["embeddings"] = x1
        patches2 = self.grouper2(patches1["centers"], x1, use_fps=False)
        patches2["embeddings"] = self.patch_encoder2(patches2["features"])
        return [patches1, patches2]


# --------------------------------------------------------------------------------------------
# timm EVA / EVA02 blocks (restated; rope=None, no CLS/abs-pos on the Point-SAM path)
# --------------------------------------------------------------------------------------------
class EvaAttention(nn.Module):
    def __init__(self, dim, num_heads, qkv_fused):
        super().__init__()
        self.num_heads = num_heads
        self.head_dim = dim // num_heads
        if qkv_fused:
            self.qkv = nn.Linear(dim, dim * 3, bias=False)
            self.q_bias = nn.Parameter(torch.zeros(dim))
            self.register_buffer("k_bias", torch.zeros(dim), persistent=False)
            self.v_bias = nn.Parameter(torch.zeros(dim))
            self.q_proj = self.k_proj = self.v_proj = None
        else:
            self.q_proj = nn.Linear(dim, dim, bias=True)
            self.k_proj = nn.Linear(dim, dim, bias=False)
            self.v_proj = nn.Linear(dim, dim, bias=True)
            self.qkv = None
        self.proj = nn.Linear(dim, dim)

    def forward(self, x):
        B, N, C = x.shape
        if self.qkv is not None:
            bias = torch.cat((self.q_bias, self.k_bias, self.v_bias))
            qkv = F.linear(x, self.qkv.weight, bias).reshape(B, N, 3, self.num_heads, -1).permute(2, 0, 3, 1, 4)
            q, k, v = qkv.unbind(0)
        else:
            q = self.q_proj(x).reshape(B, N, self.num_heads, -1).transpose(1, 2)
            k = self.k_proj(x).reshape(B, N, self.num_heads, -1).transpose(1, 2)
            v = self.v_proj(x).reshape(B, N, self.num_heads, -1).transpose(1, 2)
        attn = (q * self.head_dim ** -0.5) @ k.transpose(-2, -1)
        x = attn.softmax(dim=-1) @ v
        return self.proj(x.transpose(1, 2).reshape(B, N, C))


class SwiGLU(nn.Module):
    """timm.layers.mlp.SwiGLU with norm_layer (scale_mlp=True)."""

    def __init__(self, dim, hidden, eps):
        super().__init__()
        self.fc1_g = nn.Linear(dim, hidden)
        self.fc1_x = nn.Linear(dim, hidden)
        self.norm = nn.LayerNorm(hidden, eps=eps)
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(self.norm(F.silu(self.fc1_g(x)) * self.fc1_x(x)))


class Mlp(nn.Module):
    """timm.layers.mlp.Mlp (GELU)."""

    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x)))


class EvaBlock(nn.Module):
    def __init__(self, dim, num_heads, hidden, qkv_fused, swiglu, eps=1e-6):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = EvaAttention(dim, num_heads, qkv_fused)
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = SwiGLU(dim, hidden, eps) if swiglu else Mlp(dim, hidden)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


EVA_CONFIGS = {
    # name: (embed_dim, depth, heads, mlp hidden, qkv_fused, swiglu, img, patch)
    "eva02_base_patch14_448": (768, 12, 12, int(768 * 4 * 2 / 3), False, True, 448, 14),
    "eva02_large_patch14_448": (1024, 24, 16, int(1024 * 4 * 2 / 3), False, True, 448, 14),
    "eva_giant_patch14_560": (1408, 40, 16, 6144, True, False, 560, 14),
    # tiny config used only by tests (not a timm model)
    "eva02_test_tiny": (128, 2, 4, 344, False, True, 28, 14),
    "eva_test_tiny_fused": (176, 2, 2, 256, True, False, 28, 14),
}


class Eva(nn.Module):
    """Stand-in for ``timm.create_model(name, pretrained=False)`` exposing what
    pc_encoder.py:93,136-142 touches: embed_dim, pos_drop, blocks, norm, fc_norm (plus the unused
    cls_token / pos_embed / patch_embed.proj / head parameters so checkpoints strict-load)."""

    def __init__(self, name: str):
        super().__init__()
        D, depth, heads, hidden, fused, swiglu, img, patch = EVA_CONFIGS[name]
        self.embed_dim = D
        self.patch_embed = nn.Module()
        self.patch_embed.proj = nn.Conv2d(3, D, patch, patch)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, D))
        self.pos_embed = nn.Parameter(torch.zeros(1, (img // patch) ** 2 + 1, D))
        self.pos_drop = nn.Identity()
        self.blocks = nn.ModuleList([EvaBlock(D, heads, hidden, fused, swiglu) for _ in range(depth)])
        self.norm = nn.Identity()
        self.fc_norm = nn.LayerNorm(D, eps=1e-6)
        self.head = nn.Linear(D, 1000)


def create_model(model_name: str, pretrained: bool = False) -> Eva:
    assert not pretrained
    return Eva(model_name)


class PointCloudEncoder(nn.Module):
    """pc_sam/model/pc_encoder.py:84-145."""

    def __init__(self, patch_embed, transformer, embed_dim, patch_drop_rate=0.0):
        super().__init__()
        assert patch_drop_rate == 0
        self.transformer_dim, self.embed_dim = transformer.embed_dim, embed_dim
        self.patch_embed = patch_embed
        self.patch_proj = nn.Linear(patch_embed.out_channels, self.transformer_dim)
        self.pos_embed = nn.Sequential(nn.Linear(3, 128), nn.GELU(), nn.Linear(128, self.transformer_dim))
        self.transformer = transformer
        self.out_proj = nn.Linear(self.transformer_dim, embed_dim)

    def forward(self, coords, features):
        patches = self.patch_embed(coords, features)
        x = self.patch_proj(patches["embeddings"]) + self.pos_embed(patches["centers"])
        x = self.transformer.pos_drop(x)
        for blk in self.transformer.blocks:
            x = blk(x)
        x = self.transformer.fc_norm(self.transformer.norm(x))
        return self.out_proj(x), patches


# --------------------------------------------------------------------------------------------
# prompt / mask encoders
# --------------------------------------------------------------------------------------------
class PositionEmbeddingRandom(nn.Module):
    """pc_sam/model/prompt_encoder.py:13-48."""

    def __init__(self, num_pos_feats=64, scale=None):
        super().__init__()
        if scale is None or scale <= 0.0:
            scale = 1.0
        self.register_buffer("positional_encoding_gaussian_matrix", scale * torch.randn((3, num_pos_feats)))

    def forward(self, coords):
        if (coords < -1 - 1e-6).any() or (coords > 1 + 1e-6).any():
            raise ValueError("Input coordinates must be normalized to [-1, 1].")
        c = 2 * np.pi * (coords @ self.positional_encoding_gaussian_matrix)
        return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)


class PointEncoder(nn.Module):
    """pc_sam/model/prompt_encoder.py:51-77."""

    def __init__(self, embed_dim):
        super().__init__()
        self.embed_dim = embed_dim
        self.pe_layer = PositionEmbeddingRandom(embed_dim // 2)
        self.point_embeddings = nn.ModuleList([nn.Embedding(1, embed_dim) for _ in range(2)])

    def forward(self, points, labels):
        assert points.shape[:-1] == labels.shape
        e = self.pe_layer(points)
        e[labels == 0] += self.point_embeddings[0].weight
        e[labels == 1] += self.point_embeddings[1].weight
        return e


class MaskEncoder(nn.Module):
    """pc_sam/model/prompt_encoder.py:80-133."""

    def __init__(self, embed_dim, in_channels=4, radius=None, centralize_features=False):
        super().__init__()
        self.embed_dim, self.in_channels = embed_dim, in_channels
        self.radius, self.centralize_features = radius, centralize_features
        self.patch_encoder = PatchEncoder(in_channels, embed_dim, [128, 512])
        self.no_mask_embed = nn.Embedding(1, embed_dim)

    def forward(self, masks, coords, centers, knn_idx, center_idx=None):
        if masks is None:
            return self.no_mask_embed.weight.reshape(1, 1, -1).expand(centers.shape[0], centers.shape[1], -1)
        patches = group_with_centers_and_knn(coords, masks.detach().unsqueeze(-1), centers, knn_idx,
                                             radius=self.radius, center_idx=center_idx,
                                             centralize_features=self.centralize_features)
        return self.patch_encoder(patches)


# --------------------------------------------------------------------------------------------
# two-way transformer + mask decoder
# --------------------------------------------------------------------------------------------
class Attention(nn.Module):
    """pc_sam/model/transformer.py:183-236."""

    def __init__(self, embedding_dim, num_heads, downsample_rate=1):
        super().__init__()
        self.embedding_dim = embedding_dim
        self.internal_dim = embedding_dim // downsample_rate
        self.num_heads = num_heads
        assert self.internal_dim % num_heads == 0
        self.q_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.k_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.v_proj = nn.Linear(embedding_dim, self.internal_dim)
        self.out_proj = nn.Linear(self.internal_dim, embedding_dim)

    def _split(self, x):
        b, n, c = x.shape
        return x.reshape(b, n, self.num_heads, c // self.num_heads).transpose(1, 2)

    def forward(self, q, k, v):
        q, k, v = self._split(self.q_proj(q)), self._split(self.k_proj(k)), self._split(self.v_proj(v))
        attn = torch.softmax(q @ k.permute(0, 1, 3, 2) / math.sqrt(q.shape[-1]), dim=-1)
        out = (attn @ v).transpose(1, 2)
        return self.out_proj(out.reshape(out.shape[0], out.shape[1], -1))


class MLPBlock(nn.Module):
    """pc_sam/model/transformer.py:239-253."""

    def __init__(self, embedding_dim, mlp_dim, act=nn.GELU):
        super().__init__()
        self.lin1 = nn.Linear(embedding_dim, mlp_dim)
        self.lin2 = nn.Linear(mlp_dim, embedding_dim)
        self.act = act()

    def forward(self, x):
        return self.lin2(self.act(self.lin1(x)))


class TwoWayAttentionBlock(nn.Module):
    """pc_sam/model/transformer.py:103-180."""

    def __init__(self, embedding_dim, num_heads, mlp_dim=2048, activation=nn.ReLU,
                 attention_downsample_rate=2, skip_first_layer_pe=False):
        super().__init__()
        self.self_attn = Attention(embedding_dim, num_heads)
        self.norm1 = nn.LayerNorm(embedding_dim)
        self.cross_attn_token_to_image = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.norm2 = nn.LayerNorm(embedding_dim)
        self.mlp = MLPBlock(embedding_dim, mlp_dim, activation)
        self.norm3 = nn.LayerNorm(embedding_dim)
        self.norm4 = nn.LayerNorm(embedding_dim)
        self.cross_attn_image_to_token = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.skip_first_layer_pe = skip_first_layer_pe

    def forward(self, queries, keys, query_pe, key_pe):
        if self.skip_first_layer_pe:
            queries = self.self_attn(q=queries, k=queries, v=queries)
        else:
            q = queries + query_pe
            queries = queries + self.self_attn(q=q, k=q, v=queries)
        queries = self.norm1(queries)
        q, k = queries + query_pe, keys + key_pe
        queries = self.norm2(queries + self.cross_attn_token_to_image(q=q, k=k, v=keys))
        queries = self.norm3(queries + self.mlp(queries))
        q, k = queries + query_pe, keys + key_pe
        keys = self.norm4(keys + self.cross_attn_image_to_token(q=k, k=q, v=queries))
        return queries, keys


class TwoWayTransformer(nn.Module):
    """pc_sam/model/transformer.py:15-100."""

    def __init__(self, depth, embedding_dim, num_heads, mlp_dim, activation=nn.ReLU, attention_downsample_rate=2):
        super().__init__()
        self.depth, self.embedding_dim, self.num_heads, self.mlp_dim = depth, embedding_dim, num_heads, mlp_dim
        self.layers = nn.ModuleList([
            TwoWayAttentionBlock(embedding_dim, num_heads, mlp_dim, activation, attention_downsample_rate,
                                 skip_first_layer_pe=(i == 0)) for i in range(depth)])
        self.final_attn_token_to_image = Attention(embedding_dim, num_heads, attention_downsample_rate)
        self.norm_final_attn = nn.LayerNorm(embedding_dim)

    def forward(self, pc_embedding, pc_pe, point_embedding):
        queries, keys = point_embedding, pc_embedding
        for layer in self.layers:
            queries, keys = layer(queries=queries, keys=keys, query_pe=point_embedding, key_pe=pc_pe)
        q, k = queries + point_embedding, keys + pc_pe
        queries = self.norm_final_attn(queries + self.final_attn_token_to_image(q=q, k=k, v=keys))
        return queries, keys


class MLP(nn.Module):
    """pc_sam/model/mask_decoder.py:189-211."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers, sigmoid_output=False):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))
        self.sigmoid_output = sigmoid_output

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = F.relu(layer(x)) if i < self.num_layers - 1 else layer(x)
        return torch.sigmoid(x) if self.sigmoid_output else x


@dataclasses.dataclass
class AuxInputs:
    coords: torch.Tensor
    features: torch.Tensor
    centers: torch.Tensor
    interp_index: torch.Tensor = None
    interp_weight: torch.Tensor = None


class MaskDecoder(nn.Module):
    """pc_sam/model/mask_decoder.py:21-184."""

    def __init__(self, transformer_dim, transformer, num_multimask_outputs=3, iou_head_depth=3, iou_head_hidden_dim=256):
        super().__init__()
        self.transformer_dim, self.transformer = transformer_dim, transformer
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

    def forward(self, pc_embeddings, pc_pe, sparse_prompt_embeddings, dense_prompt_embeddings, aux_inputs, multimask_output):
        mask_slice = slice(1, None) if multimask_output else slice(0, 1)
        out_tokens = torch.cat([self.iou_token.weight, self.mask_tokens.weight], dim=0)
        out_tokens = out_tokens.unsqueeze(0).expand(sparse_prompt_embeddings.size(0), -1, -1)
        tokens = torch.cat((out_tokens, sparse_prompt_embeddings), dim=1)
        rep = tokens.shape[0] // pc_embeddings.shape[0]
        src = repeat_interleave(pc_embeddings, rep, 0) + dense_prompt_embeddings
        pos_src = repeat_interleave(pc_pe, rep, 0)
        hs, src = self.transformer(src, pos_src, tokens)
        iou_token_out = hs[:, 0, :]
        mask_tokens_out = hs[:, 1:1 + self.num_mask_tokens, :]
        if aux_inputs.interp_index is None or aux_inputs.interp_weight is None:
            with torch.no_grad():
                aux_inputs.interp_index, aux_inputs.interp_weight = compute_interp_weights(aux_inputs.coords, aux_inputs.centers)
        rep2 = tokens.shape[0] // aux_inputs.interp_index.shape[0]
        idx = repeat_interleave(aux_inputs.interp_index, rep2, 0)
        w = repeat_interleave(aux_inputs.interp_weight, rep2, 0)
        up = self.output_upscaling(interpolate_features(src, idx, w))
        ids = list(range(self.num_mask_tokens))[mask_slice]
        hyper_in = torch.stack([self.output_hypernetworks_mlps[i](mask_tokens_out[:, i, :]) for i in ids], dim=1)
        masks = hyper_in @ up.transpose(-1, -2)
        iou_pred = self.iou_prediction_head(iou_token_out)[:, mask_slice]
        return masks, iou_pred


class PointCloudSAM(nn.Module):
    """pc_sam/model/pc_sam.py:20-196 (predict_masks and the prompt loop; prompts are supplied)."""

    def __init__(self, pc_encoder, mask_encoder, mask_decoder, prompt_iters, enable_mask_refinement_iterations=True):
        super().__init__()
        self.pc_encoder = pc_encoder
        self.point_encoder = PointEncoder(pc_encoder.embed_dim)
        self.mask_encoder, self.mask_decoder = mask_encoder, mask_decoder
        self.prompt_iters = prompt_iters
        self.enable_mask_refinement_iterations = enable_mask_refinement_iterations

    def predict_masks(self, coords, features, prompt_coords, prompt_labels, prompt_masks=None, multimask_output=True):
        pc_embeddings, patches = self.pc_encoder(coords, features)
        centers, knn_idx = patches["centers"], patches["knn_idx"]
        aux = AuxInputs(coords=coords, features=features, centers=centers)
        pc_pe = self.point_encoder.pe_layer(centers)
        sparse = self.point_encoder(prompt_coords, prompt_labels)
        dense = self.mask_encoder(prompt_masks, coords, centers, knn_idx)
        dense = repeat_interleave(dense, sparse.shape[0] // dense.shape[0], 0)
        return self.mask_decoder(pc_embeddings, pc_pe, sparse, dense, aux_inputs=aux, multimask_output=multimask_output)

    def predict_iterative(self, coords, features, prompt_coords_seq: List[torch.Tensor], prompt_labels_seq: List[torch.Tensor]):
        """The loop body of forward (pc_sam.py:139-194) with externally supplied prompts:
        iteration t appends prompt_coords_seq[t]; multimask only at t=0; best mask fed back."""
        pc_embeddings, patches = self.pc_encoder(coords, features)
        centers, knn_idx = patches["centers"], patches["knn_idx"]
        aux = AuxInputs(coords=coords, features=features, centers=centers)
        pc_pe = self.point_encoder.pe_layer(centers)
        outs, pm = [], None
        pc = prompt_coords_seq[0][:, :0]
        pl = prompt_labels_seq[0][:, :0]
        for t in range(len(prompt_coords_seq)):
            pc = torch.cat([pc, prompt_coords_seq[t]], dim=1)
            pl = torch.cat([pl, prompt_labels_seq[t]], dim=1)
            sparse = self.point_encoder(pc, pl)
            dense = self.mask_encoder(pm, coords, centers, knn_idx, center_idx=patches.get("fps_idx"))
            dense = repeat_interleave(dense, sparse.shape[0] // dense.shape[0], 0)
            masks, iou = self.mask_decoder(pc_embeddings, pc_pe, sparse, dense, aux_inputs=aux, multimask_output=(t == 0))
            if t == 0:
                best = torch.argmax(iou, dim=1)
                pm = batch_index_select(masks, best, dim=1)
            else:
                best = 0
                pm = masks[:, 0]
            outs.append(dict(prompt_coords=pc, prompt_labels=pl, masks=masks, iou_preds=iou,
                             max_iou_pred_ind=best, prompt_masks=pm))
        return outs



# ---------------------------------------------------------------------------------------------------------
# ground-truth prompt sampling (pc_sam/model/common.py:371-474), evaluation branch of sample_prompts_adapter
# ---------------------------------------------------------------------------------------------------------
def _farthest_from_border(coords, labels, gt):
    """common.py:445-474: among points with label 1, the one whose nearest label-0 point is farthest (squared distance
    with the chamfer kernel's arithmetic, chamfer_distance_kernel.cu:62-76; first index on ties like torch.argmax)."""
    bg, fg = labels == 0, labels == 1
    if int(bg.sum()) == 0 or int(fg.sum()) == 0:
        return None, None, -1
    q = coords[fg].detach().cpu().float().numpy()[None]
    k = coords[bg].detach().cpu().float().numpy()[None]
    _, d2 = tokenizer_ref.knn(q, k, 1)
    d = torch.from_numpy(d2[0, :, 0])
    i = torch.argmax(d)
    return coords[fg][i][None], gt[fg][i][None], float(d.max())


def sample_fixed_points(points, gt_masks, pred_logits, threshold=None, from_error_region=False):
    """common.py:371-442.  points [B,N,3], gt_masks [B,M,N] bool, pred_logits [B*M,N] | None."""
    B, M, _ = gt_masks.shape
    if pred_logits is None:
        fn, fp = gt_masks, torch.zeros_like(gt_masks)
    else:
        pl = pred_logits.reshape(B, M, -1)
        pm = pl > 0 if threshold is None else pl.sigmoid() > threshold
        fn, fp = gt_masks & ~pm, ~gt_masks & pm
    pts, labs = [], []
    for b in range(B):
        for m in range(M):
            if from_error_region:
                c, l, _ = _farthest_from_border(points[b], (fn | fp)[b, m], gt_masks[b, m])
            else:
                c, l, pd = _farthest_from_border(points[b], fn[b, m], gt_masks[b, m])
                c2, l2, nd = _farthest_from_border(points[b], fp[b, m], gt_masks[b, m])
                if not pd > nd:
                    if nd == -1:
                        c, l, _ = _farthest_from_border(points[b], gt_masks[b, m], gt_masks[b, m])
                    else:
                        c, l = c2, l2
            pts.append(c)
            labs.append(l)
    return torch.stack(pts), torch.stack(labs)


def sample_prompts_eval(points, gt_masks, pred_logits, threshold=None):
    """sample_prompts_adapter(..., is_eval=True) (common.py:287-318)."""
    return sample_fixed_points(points, gt_masks, pred_logits, threshold, from_error_region=pred_logits is None)


def build_model(encoder: str = "eva02_large_patch14_448", num_patches=512, patch_size=64, embed_dim=256,
                prompt_iters=5, seed: Optional[int] = 1234) -> PointCloudSAM:
    """Mirror of configs/model/{base,default,giant}.yaml with default torch initialisation."""
    if seed is not None:
        torch.manual_seed(seed)
    pe = PatchEmbed(6, 512, num_patches, patch_size)
    enc = PointCloudEncoder(pe, create_model(encoder), embed_dim)
    me = MaskEncoder(embed_dim)
    md = MaskDecoder(embed_dim, TwoWayTransformer(2, embed_dim, 8, 2048))
    return PointCloudSAM(enc, me, md, prompt_iters).eval()
