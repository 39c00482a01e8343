"""Tensor-level wrappers over the C ABI (one Python function per exported kernel).

Everything here takes/returns CUDA torch tensors, allocates outputs with torch (device memory is
PyTorch's job) and enqueues work on torch's current stream.  No math is done in PyTorch.
"""
from __future__ import annotations

from ctypes import byref
from typing import Optional

import numpy as np
import torch

from . import native as nv
from .native import ACT_GELU, ACT_NONE, ACT_RELU, GemmOut, LinearArgs, LnArgs, Operand  # noqa: F401


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class Split:
    """split-bf16 matrix: planes [2, rows, pitch] (hi, lo), logical width `cols`."""

    __slots__ = ("t", "rows", "cols", "pitch")

    def __init__(self, rows: int, cols: int, device, pitch: Optional[int] = None, zero: bool = False):
        self.rows, self.cols = rows, cols
        self.pitch = pitch if pitch is not None else _round_up(cols, 64)
        alloc = torch.zeros if zero else torch.empty
        self.t = alloc((2, rows, self.pitch), dtype=torch.bfloat16, device=device)

    @property
    def plane(self) -> int:
        return self.rows * self.pitch

    def ptr(self, col: int = 0, row: int = 0) -> int:
        return self.t.data_ptr() + 2 * (row * self.pitch + col)

    def operand(self, rows=None, k=None, col=0, row=0, nb1=0, b1_stride=0, nb2=0, b2_stride=0) -> Operand:
        return Operand(self.ptr(col, row), self.plane, rows if rows is not None else self.rows,
                       k if k is not None else self.cols, self.pitch, nb1, nb2, b1_stride, b2_stride)

    def float(self) -> torch.Tensor:  # debugging / tests only
        return (self.t[0].float() + self.t[1].float())[:, : self.cols]


def pack_weight(w: torch.Tensor) -> Split:
    """fp32 [N,K] -> split-bf16 (done once at model load)."""
    w = w.detach().float().contiguous()
    s = Split(w.shape[0], w.shape[1], w.device)
    split_f32(w, s)
    return s


# ------------------------------------------------------------------------------------------------
def pad_clouds(*clouds):
    """Padded batch of clouds of different sizes: each argument is a sequence of B tensors [N_b, C] (the same N_b for every
    argument) and becomes one [B, N_max, C] fp32 tensor whose rows n >= N_b are zeros.  Returns the padded tensors followed
    by lengths [B] int32 on the device (the `lengths` of the varlen ops).  Nothing waits for the device: the lengths are
    copied from pinned host memory without a synchronisation."""
    first = clouds[0]
    if not len(first):
        raise ValueError("pad_clouds: no clouds")
    sizes = [int(t.shape[0]) for t in first]
    for seq in clouds:
        if len(seq) != len(first) or any(t.dim() != 2 or int(t.shape[0]) != n for t, n in zip(seq, sizes)):
            raise ValueError(f"pad_clouds: every sequence must hold {len(first)} tensors [N_b, C] with N_b = {sizes}")
    dev = first[0].device
    out = [torch.nn.utils.rnn.pad_sequence([t.float() for t in seq], batch_first=True).contiguous() for seq in clouds]
    host = torch.tensor(sizes, dtype=torch.int32)
    lengths = (host.pin_memory() if dev.type == "cuda" else host).to(dev, non_blocking=True)
    return (*out, lengths)


def fps(xyz: torch.Tensor, num_samples: int, lengths: Optional[torch.Tensor] = None):
    """Farthest-point sampling of num_samples centres per cloud of xyz [B, N, 3] -> (idx [B, G] int64, centers [B, G, 3]).
    lengths [B] int32 (device): cloud b is its first lengths[b] points (psam_fps_varlen_f32); slots past lengths[b] repeat
    sample 0."""
    B, N, _ = xyz.shape
    idx = torch.empty((B, num_samples), dtype=torch.int64, device=xyz.device)
    centers = torch.empty((B, num_samples, 3), dtype=torch.float32, device=xyz.device)
    nbytes = nv.lib().psam_fps_workspace_bytes(B, N, num_samples)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xyz.device) if nbytes else None
    if lengths is None:
        nv.check(nv.lib().psam_fps_f32(nv.ptr(xyz), B, N, num_samples, nv.ptr(idx), nv.ptr(centers), nv.ptr(ws), nv.stream()), "fps")
    else:
        lengths = _lengths(lengths, B, "fps")
        nv.check(nv.lib().psam_fps_varlen_f32(nv.ptr(xyz), nv.ptr(lengths), B, N, num_samples, nv.ptr(idx), nv.ptr(centers),
                                              nv.ptr(ws), nv.stream()), "fps")
    return idx, centers


def knn(query: torch.Tensor, key: torch.Tensor, k: int, want_d2: bool = False, lengths: Optional[torch.Tensor] = None):
    """k nearest keys of every query: query [B, Q, 3], key [B, N, 3] -> (idx [B, Q, k] int64, d2 [B, Q, k] or None).
    lengths [B] int32 (device): the keys of cloud b are its first lengths[b] rows (psam_knn_varlen_f32)."""
    B, Q, _ = query.shape
    N = key.shape[1]
    idx = torch.empty((B, Q, k), dtype=torch.int64, device=query.device)
    d2 = torch.empty((B, Q, k), dtype=torch.float32, device=query.device) if want_d2 else None
    if lengths is None:
        nv.check(nv.lib().psam_knn_f32(nv.ptr(query), nv.ptr(key), B, Q, N, k, nv.ptr(idx), nv.ptr(d2), nv.stream()), "knn")
    else:
        lengths = _lengths(lengths, B, "knn")
        nv.check(nv.lib().psam_knn_varlen_f32(nv.ptr(query), nv.ptr(key), nv.ptr(lengths), B, Q, N, k, nv.ptr(idx), nv.ptr(d2),
                                              nv.stream()), "knn")
    return idx, d2


def _lengths(lengths: torch.Tensor, B: int, what: str) -> torch.Tensor:
    if lengths.dtype != torch.int32 or lengths.numel() != B:
        raise ValueError(f"{what}: lengths must be {B} int32 values, got {lengths.numel()} of {lengths.dtype}")
    return lengths.contiguous()


def group_gather(xyz, feats, centers, knn_idx, radius=None, center_idx=None):
    """center_idx [B,G] int64: centralize_features=True (C more channels feats[idx] - feats[center])."""
    B, N, _ = xyz.shape
    B2, _, C = feats.shape
    _, G, K = knn_idx.shape
    out = torch.empty((B2, G, K, 3 + C + (C if center_idx is not None else 0)), dtype=torch.float32, device=xyz.device)
    nv.check(nv.lib().psam_group_gather_f32(nv.ptr(xyz), nv.ptr(feats), nv.ptr(centers), nv.ptr(knn_idx), nv.ptr(center_idx), B, B2 // B,
                                            N, G, K, C, float(radius) if radius else 0.0, nv.ptr(out), nv.stream()), "group_gather")
    return out


def nn_index(query, key):
    """Nearest key of every query point, one cloud at a time (first index on ties): idx [B,Nq] int64."""
    B, Nq, _ = query.shape
    Nk = key.shape[1]
    idx = torch.empty((B, Nq), dtype=torch.int64, device=query.device)
    dist = torch.empty((B, Nq), dtype=torch.float32, device=query.device)
    for b in range(B):
        nv.check(nv.lib().psam_nn_distance_f32(nv.ptr(query[b]), nv.ptr(key[b]), Nq, Nk, nv.ptr(dist[b]), nv.ptr(idx[b]), nv.stream()),
                 "nn_distance")
    return idx


def voronoi_features(xyz, centers, nn_idx, feats, want_split: bool = False):
    """[unit direction to the nearest centre, distance, features] per point: fp32 [B2,N,4+C] (+ split copy, pitch 64)."""
    B, N, _ = xyz.shape
    B2, _, C = feats.shape
    out = torch.empty((B2, N, 4 + C), dtype=torch.float32, device=xyz.device)
    sp = Split(B2 * N, 4 + C, xyz.device) if want_split else None
    nv.check(nv.lib().psam_voronoi_features_f32(nv.ptr(xyz), nv.ptr(centers), nv.ptr(nn_idx), nv.ptr(feats), B, B2 // B, N,
                                                centers.shape[1], C, nv.ptr(out), sp.ptr() if sp is not None else None,
                                                sp.plane if sp is not None else 0, sp.pitch if sp is not None else 0, nv.stream()),
             "voronoi_features")
    return (out, sp) if want_split else out


def scatter_amax(x, nn_idx, G: int):
    """x [B,N,D], nn_idx [B,N] -> [B,G,D] maximum per Voronoi cell (empty cells 0)."""
    B, N, D = x.shape
    y = torch.empty((B, G, D), dtype=torch.float32, device=x.device)
    nv.check(nv.lib().psam_scatter_amax_f32(nv.ptr(x), nv.ptr(nn_idx), B, N, G, D, nv.ptr(y), nv.stream()), "scatter_amax")
    return y


def knn3_interp(xyz, centers):
    B, N, _ = xyz.shape
    G = centers.shape[1]
    idx = torch.empty((B, N, 3), dtype=torch.int64, device=xyz.device)
    w = torch.empty((B, N, 3), dtype=torch.float32, device=xyz.device)
    nv.check(nv.lib().psam_knn3_interp_f32(nv.ptr(xyz), nv.ptr(centers), B, N, G, nv.ptr(idx), nv.ptr(w), nv.stream()), "knn3_interp")
    return idx, w


def nn_distance(query: torch.Tensor, key: torch.Tensor):
    """Squared distance from each query [n1,3] to its nearest key [n2,3]."""
    q, k = query.float().contiguous(), key.float().contiguous()
    d = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
    nv.check(nv.lib().psam_nn_distance_f32(nv.ptr(q), nv.ptr(k), q.shape[0], k.shape[0], nv.ptr(d), None, nv.stream()), "nn_distance")
    return d


def border_prompt(coords: torch.Tensor, gt_masks: torch.Tensor, pred_logits: Optional[torch.Tensor] = None,
                  pred_masks: Optional[torch.Tensor] = None, from_error_region: bool = False,
                  status: Optional[torch.Tensor] = None, lengths: Optional[torch.Tensor] = None):
    """Batched farthest-from-border prompt sampling (psam_border_prompt_f32).  coords [B,N,3], gt_masks [B,M,N] bool,
    prediction as logits [B*M,N] or bool masks [B*M,N] or neither.  Returns (xyz [B*M,1,3], labels [B*M,1] bool, status).
    lengths [B] int32 (device): padded clouds, cloud b is its first lengths[b] rows (psam_border_prompt_varlen_f32); each
    (cloud, mask) gets what the single-cloud sampler returns on that cloud alone."""
    B, M, N = gt_masks.shape
    if lengths is not None:
        lengths = _lengths(lengths, B, "border_prompt")
    c = coords.float().contiguous()
    g = gt_masks.contiguous().view(torch.uint8) if gt_masks.dtype == torch.bool else gt_masks.to(torch.uint8).contiguous()
    lg = pred_logits.float().contiguous() if pred_logits is not None else None
    pm = None
    if pred_masks is not None:
        pm = pred_masks.contiguous().view(torch.uint8) if pred_masks.dtype == torch.bool else pred_masks.to(torch.uint8).contiguous()
    dev = c.device
    xyz = torch.empty((B * M, 1, 3), dtype=torch.float32, device=dev)
    lab = torch.empty((B * M, 1), dtype=torch.uint8, device=dev)
    if status is None:
        status = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.empty(nv.lib().psam_border_prompt_workspace_bytes(B, M, N), dtype=torch.uint8, device=dev)
    if lengths is None:
        nv.check(nv.lib().psam_border_prompt_f32(nv.ptr(c), nv.ptr(g), nv.ptr(lg), nv.ptr(pm), B, M, N, int(from_error_region),
                                                 nv.ptr(xyz), nv.ptr(lab), nv.ptr(status), nv.ptr(ws), nv.stream()), "border_prompt")
    else:
        nv.check(nv.lib().psam_border_prompt_varlen_f32(nv.ptr(c), nv.ptr(lengths), nv.ptr(g), nv.ptr(lg), nv.ptr(pm), B, M, N,
                                                        int(from_error_region), nv.ptr(xyz), nv.ptr(lab), nv.ptr(status), nv.ptr(ws),
                                                        nv.stream()), "border_prompt")
    return xyz, lab.view(torch.bool), status


GEMM_TILE_HINT = 0  # 0 = latency-optimal tiles, 1 = SM-time-optimal tiles (set by PipelinedPredictor)
GEMM_TILE_BN = 0    # 32..256: explicit tile width (experiments / tests)
# psam_gemm_out.variant (experiment switches, see include/psam_b200.h); PSAM_GEMM_VARIANT seeds it once at import
GV_2CTA, GV_BK32, GV_SCALAR_EPI, GV_DUAL, GV_NO_DUAL, GV_PERSIST, GV_NO_PERSIST, GV_TWO_ISSUERS = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40, 0x80
GEMM_VARIANT = int(__import__("os").environ.get("PSAM_GEMM_VARIANT", "0"), 0)


def gemm_raw(a: Operand, w: Operand, out: GemmOut, passes: int = 3, split_k: int = 1):
    if out.tile_hint == 0:
        out.tile_hint = GEMM_TILE_BN if GEMM_TILE_BN else GEMM_TILE_HINT
    if out.variant == 0:
        out.variant = GEMM_VARIANT
    nv.check(nv.lib().psam_gemm_bf16x3(byref(a), byref(w), byref(out), passes, split_k, nv.stream()), "gemm_bf16x3")


def gemm(a: Split, w: Split, *, bias=None, out_f32: Optional[torch.Tensor] = None, out_split: Optional[Split] = None,
         resid: Optional[torch.Tensor] = None, act: int = ACT_NONE, alpha: float = 1.0, accumulate: bool = False,
         split_k: int = 1, passes: int = 3, rows: Optional[int] = None, swiglu: bool = False,
         gmax: Optional[torch.Tensor] = None, group_rows: int = 0, rowdot=None, stats_out: Optional[torch.Tensor] = None,
         ln_fold=None):
    """out = act(alpha * a @ w^T + bias (+ resid)); a [M,K], w [N,K] split-bf16."""
    M = rows if rows is not None else a.rows
    o = GemmOut()
    o.out_f32 = nv.ptr(out_f32)
    o.ldo = out_f32.stride(-2) if out_f32 is not None else 0
    o.out_hi = out_split.ptr() if out_split is not None else None
    o.out_plane = out_split.plane if out_split is not None else 0
    o.ldo_s = out_split.pitch if out_split is not None else 0
    o.bias = nv.ptr(bias)
    o.resid = nv.ptr(resid)
    o.alpha = alpha
    o.act = act
    o.accumulate = int(accumulate)
    o.swiglu = int(swiglu)
    if gmax is not None:
        o.gmax, o.ld_gmax, o.group_rows = nv.ptr(gmax), gmax.shape[-1], group_rows
    if rowdot is not None:  # (w [Z,C,N], out [Z,C,rows] zero-filled)
        rw, ro = rowdot
        o.rd_w, o.rd_out, o.rd_rows, o.rd_c = nv.ptr(rw), nv.ptr(ro), ro.shape[-1], ro.shape[-2]
    o.stats_out = nv.ptr(stats_out)
    if ln_fold is not None:  # (stats [M,2], c [N], H, eps): LayerNorm over the K axis folded into this GEMM
        st, c, hh, eps = ln_fold
        o.ln_stats, o.ln_c, o.ln_h, o.ln_eps = nv.ptr(st), nv.ptr(c), int(hh), float(eps)
    gemm_raw(a.operand(rows=M), w.operand(), o, passes, split_k)


def gemm_rowln(a: Split, w: Split, gamma, beta, eps: float, out: Split, *, gbias: Optional[torch.Tensor] = None, group_rows: int = 0,
               act: int = ACT_NONE, passes: int = 3):
    """out = act(LayerNorm(a @ w^T + gbias[row // group_rows])) as split-bf16; K <= 128, N in {256, 512} (psam_gemm_rowln_bf16x3)."""
    ao, wo = a.operand(), w.operand()
    nv.check(nv.lib().psam_gemm_rowln_bf16x3(byref(ao), byref(wo), nv.ptr(gbias), gbias.shape[-1] if gbias is not None else 0, group_rows,
                                             nv.ptr(gamma), nv.ptr(beta), float(eps), act, out.ptr(), out.plane, out.pitch, passes,
                                             nv.stream()), "gemm_rowln_bf16x3")


def gemm_rowln_supported(K: int, N: int) -> bool:
    return K <= 128 and N in (256, 512)


def linear_f32(x, w, b=None, *, x2=None, r=None, act=ACT_NONE, out=None, M=None, K=None, ldx=None, Z=1, x_z=0, x2_z=0,
               w_z=0, b_z=0, r_z=0, y_z=0, ldy=None, x_off=0):
    """fp32 SIMT linear (see psam_linear_f32). x [.., K] flattened to rows unless M/ldx given."""
    N = w.shape[-2]
    Kd = K if K is not None else w.shape[-1]
    if M is None:
        M = x.numel() // x.shape[-1]
    if out is None:
        out = torch.empty((Z * M, N) if Z > 1 else (M, N), dtype=torch.float32, device=x.device)
    a = LinearArgs()
    a.x = nv.ptr(x) + 4 * x_off
    a.ldx = ldx if ldx is not None else x.shape[-1]
    a.x_z = x_z
    a.x2 = nv.ptr(x2)
    a.x2_z = x2_z
    a.w = nv.ptr(w)
    a.ldw = w.shape[-1]
    a.w_z = w_z
    a.b = nv.ptr(b)
    a.b_z = b_z
    a.r = nv.ptr(r)
    a.r_z = r_z
    a.y = nv.ptr(out)
    a.ldy = ldy if ldy is not None else N
    a.y_z = y_z
    a.M, a.N, a.K, a.Z, a.act = M, N, Kd, Z, act
    nv.check(nv.lib().psam_linear_f32(byref(a), nv.stream()), "linear_f32")
    return out


def layernorm(x, gamma, beta, eps, *, rows=None, D=None, r=None, gbias=None, group_rows=0, act=ACT_NONE,
              out_f32: Optional[torch.Tensor] = None, out_split: Optional[Split] = None, ldx=None, padded: bool = False,
              post_add: Optional[torch.Tensor] = None, out_split2: Optional[Split] = None):
    D = D if D is not None else x.shape[-1]
    rows = rows if rows is not None else x.numel() // x.shape[-1]
    a = LnArgs()
    a.x, a.ldx = nv.ptr(x), (ldx if ldx is not None else x.shape[-1])
    a.r, a.ldr = nv.ptr(r), (r.shape[-1] if r is not None else 0)
    a.gbias, a.ld_gbias, a.group_rows = nv.ptr(gbias), (gbias.shape[-1] if gbias is not None else 0), group_rows
    a.gamma, a.beta, a.eps = nv.ptr(gamma), nv.ptr(beta), eps
    a.rows, a.D, a.act = rows, D, act
    a.y, a.ldy = nv.ptr(out_f32), (out_f32.shape[-1] if out_f32 is not None else 0)
    if out_split is not None:
        a.y_hi, a.y_plane, a.ldy_s, a.pitch = out_split.ptr(), out_split.plane, out_split.pitch, out_split.pitch
    a.padded = int(padded)
    if out_split2 is not None:  # second split output = split(y + post_add)
        a.post_add, a.ld_post = nv.ptr(post_add), post_add.shape[-1]
        a.y2_hi, a.y2_plane, a.ldy2_s = out_split2.ptr(), out_split2.plane, out_split2.pitch
    a.policy = GEMM_TILE_HINT  # same switch as the GEMM tile policy: 1 while capturing the pipelined predictor's graphs
    nv.check(nv.lib().psam_layernorm_f32(byref(a), nv.stream()), "layernorm")


def swiglu_ln(gx: torch.Tensor, H: int, x_off: int, gamma, beta, eps, out: Split):
    rows = gx.shape[0]
    nv.check(nv.lib().psam_swiglu_ln(nv.ptr(gx), gx.shape[1], x_off, rows, H, nv.ptr(gamma), nv.ptr(beta), eps,
                                     out.ptr(), out.plane, out.pitch, out.pitch, nv.stream()), "swiglu_ln")


def small_in_linear(x, W, b, gamma, beta, eps, use_ln: bool, act: int, out: Split):
    rows, Cin = x.numel() // x.shape[-1], x.shape[-1]
    nv.check(nv.lib().psam_small_in_linear(nv.ptr(x), rows, Cin, nv.ptr(W), nv.ptr(b), nv.ptr(gamma), nv.ptr(beta), eps,
                                           int(use_ln), act, W.shape[0], out.ptr(), out.plane, out.pitch, nv.stream()),
             "small_in_linear")


def group_max(x: torch.Tensor, groups: int, K: int, out_f32=None, out_split: Optional[Split] = None):
    D = x.shape[-1]
    nv.check(nv.lib().psam_group_max(nv.ptr(x), D, groups, K, D, nv.ptr(out_f32), D,
                                     out_split.ptr() if out_split is not None else None,
                                     out_split.plane if out_split is not None else 0,
                                     out_split.pitch if out_split is not None else 0, nv.stream()), "group_max")


def softmax_split(s: torch.Tensor, L: int, scale: float, out: Split):
    rows = s.numel() // s.shape[-1]
    nv.check(nv.lib().psam_softmax_split(nv.ptr(s), s.shape[-1], rows, L, scale, out.ptr(), out.plane, out.pitch, nv.stream()),
             "softmax_split")


def posenc(coords, gauss, labels=None, emb0=None, emb1=None, bad_flag=None):
    rows = coords.numel() // 3
    F = gauss.shape[1]
    out = torch.empty(coords.shape[:-1] + (2 * F,), dtype=torch.float32, device=coords.device)
    nv.check(nv.lib().psam_posenc_f32(nv.ptr(coords), rows, nv.ptr(gauss), F, nv.ptr(labels), nv.ptr(emb0), nv.ptr(emb1),
                                      nv.ptr(out), nv.ptr(bad_flag), nv.stream()), "posenc")
    return out


def attention_f32(q, k, v, Z, Lq, Lk, H, dh, q_off=0, k_off=0, v_off=0):
    """q / k / v may be column windows of wider row-major tensors: *_off = first column, the row stride is the tensor's width."""
    o = torch.empty((Z * Lq, H * dh), dtype=torch.float32, device=q.device)
    nv.check(nv.lib().psam_attention_f32(nv.ptr(q) + 4 * q_off, nv.ptr(k) + 4 * k_off, nv.ptr(v) + 4 * v_off, nv.ptr(o), Z, Lq, Lk, H,
                                         dh, q.shape[-1], k.shape[-1], v.shape[-1], H * dh, nv.stream()), "attention_f32")
    return o


def add_bcast(a, b, chunk=None, rep=1):
    out = torch.empty_like(a)
    n = a.numel()
    nv.check(nv.lib().psam_add_bcast_f32(nv.ptr(a), nv.ptr(b), n, chunk if chunk else n, rep, b.numel(), nv.ptr(out), nv.stream()),
             "add_bcast")
    return out


def split_f32(x: torch.Tensor, out: Split, add: Optional[torch.Tensor] = None):
    """out = split-bf16(x (+ add))."""
    rows = x.numel() // x.shape[-1]
    if add is None:
        nv.check(nv.lib().psam_split_f32(nv.ptr(x), x.shape[-1], rows, x.shape[-1], out.ptr(), out.plane, out.pitch, out.pitch,
                                         nv.stream()), "split_f32")
    else:
        nv.check(nv.lib().psam_split_add_f32(nv.ptr(x), nv.ptr(add), x.shape[-1], rows, x.shape[-1], out.ptr(), out.plane, out.pitch,
                                             out.pitch, nv.stream()), "split_add_f32")



# ------------------------------------------------------------------------------------------------
# automatic mask generation: candidate extraction and mask NMS
# ------------------------------------------------------------------------------------------------
NMS_MAX_CANDIDATES = 16384


def mask_words(N: int) -> int:
    """32-bit words of one bit-packed mask of N points."""
    return (N + 31) // 32


def mask_candidates(logits: torch.Tensor, iou_preds: torch.Tensor, *, mask_threshold: float = 0.0,
                    stability_offset: float = 1.0, pred_iou_thresh: float = 0.0, stability_thresh: float = 0.0,
                    min_area: int = 0, out=None, base: int = 0):
    """Candidate extraction (psam_mask_candidates_f32): logits [Z,C,N], iou_preds [Z,C] fill slots base .. base + Z*C of
    out = (bits [K,W] int32 bit patterns, area [K] int32, stability [K] fp32, score [K] fp32; -inf = filtered out).
    Without `out` the four tensors are allocated for K = Z*C slots."""
    Z, C, N = logits.shape
    lg = logits.float().contiguous()
    io = iou_preds.float().contiguous()
    if out is None:
        if base != 0:
            raise ValueError("mask_candidates: base needs a caller-owned `out`")
        K, dev = Z * C, logits.device
        out = (torch.empty((K, mask_words(N)), dtype=torch.int32, device=dev), torch.empty(K, dtype=torch.int32, device=dev),
               torch.empty(K, dtype=torch.float32, device=dev), torch.empty(K, dtype=torch.float32, device=dev))
    bits, area, stab, score = out
    if base < 0 or base + Z * C > bits.shape[0]:
        raise ValueError(f"mask_candidates: slots {base}..{base + Z * C} do not fit {bits.shape[0]} candidates")
    nv.check(nv.lib().psam_mask_candidates_f32(nv.ptr(lg), nv.ptr(io), Z, C, N, float(mask_threshold), float(stability_offset),
                                               float(pred_iou_thresh), float(stability_thresh), int(min_area), int(base),
                                               bits.shape[1], nv.ptr(bits), nv.ptr(area), nv.ptr(stab), nv.ptr(score),
                                               nv.stream()), "mask_candidates")
    return out


def mask_nms(bits: torch.Tensor, area: torch.Tensor, score: torch.Tensor, nms_thresh: float):
    """Greedy mask-IoU NMS (psam_mask_nms) over the K candidates of mask_candidates.  Returns (keep [max(K,1)] int32, the
    kept candidate indices in score order, and keep_count [1] int32); both stay on the device."""
    K, W = bits.shape
    if K > NMS_MAX_CANDIDATES:
        raise ValueError(f"mask_nms: {K} candidates, at most {NMS_MAX_CANDIDATES}")
    dev = bits.device
    keep = torch.empty(max(K, 1), dtype=torch.int32, device=dev)
    keep_count = torch.empty(1, dtype=torch.int32, device=dev)
    ws = torch.empty(nv.lib().psam_mask_nms_workspace_bytes(K, W), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_mask_nms(nv.ptr(bits) if K else None, nv.ptr(area) if K else None, nv.ptr(score) if K else None, K, W,
                                    float(nms_thresh), nv.ptr(keep), nv.ptr(keep_count), nv.ptr(ws), nv.stream()), "mask_nms")
    return keep, keep_count


def mask_regions(bits: torch.Tensor, keep: torch.Tensor, keep_count: torch.Tensor, nbr: torch.Tensor, min_area: int):
    """Small hole / island removal (psam_mask_regions) on the kept masks keep[:keep_count] of mask_candidates' bits, over
    the kNN graph nbr [N, k1] or [1, N, k1] int64 (knn(xyz, xyz, k1)).  Returns (bits_out [K,W] int32, area_out [K] int32,
    score_out [K] fp32), indexed by kept rank with K = len(keep): 1.0 = unchanged, 0.0 = changed, -inf past the kept count.
    The outputs feed mask_nms directly; nothing waits for the device."""
    K, W = keep.shape[0], bits.shape[1]
    N, k1 = nbr.shape[-2], nbr.shape[-1]
    if K > NMS_MAX_CANDIDATES:
        raise ValueError(f"mask_regions: {K} kept masks, at most {NMS_MAX_CANDIDATES}")
    nbr = nbr.reshape(N, k1).contiguous()
    dev = bits.device
    bits_out = torch.empty((K, W), dtype=torch.int32, device=dev)
    area_out = torch.empty(K, dtype=torch.int32, device=dev)
    score_out = torch.empty(K, dtype=torch.float32, device=dev)
    ws = torch.empty(nv.lib().psam_mask_regions_workspace_bytes(K, N), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_mask_regions(nv.ptr(bits), K, W, N, nv.ptr(keep), nv.ptr(keep_count), nv.ptr(nbr), k1, int(min_area),
                                        nv.ptr(bits_out), nv.ptr(area_out), nv.ptr(score_out), nv.ptr(ws), nv.stream()),
             "mask_regions")
    return bits_out, area_out, score_out


def mask_candidates_batched(logits: torch.Tensor, iou_preds: torch.Tensor, B: int, *, out, base: int = 0,
                            mask_threshold: float = 0.0, stability_offset: float = 1.0, pred_iou_thresh: float = 0.0,
                            stability_thresh: float = 0.0, min_area: int = 0, lengths: Optional[torch.Tensor] = None,
                            num_prompts: int = 0):
    """mask_candidates for B clouds in one launch (psam_mask_candidates_batched_f32): logits [B*Zc,C,N], iou_preds [B*Zc,C],
    rows b*Zc .. b*Zc+Zc-1 of cloud b.  Row b*Zc + j, output c fills slot base + j*C + c of cloud b in
    out = (bits [B,K,W] int32, area [B,K] int32, stability [B,K] fp32, score [B,K] fp32).
    lengths [B] int32 (device), padded clouds (psam_mask_candidates_varlen_f32): only cloud b's first lengths[b] points are
    counted and packed, and the slots of its prompts past min(num_prompts, lengths[b]) score -inf."""
    Z, C, N = logits.shape
    bits, area, stab, score = out
    if B < 1 or Z % B or bits.shape[0] != B:
        raise ValueError(f"mask_candidates_batched: {Z} rows and {bits.shape[0]} candidate blocks for {B} clouds")
    Zc, K = Z // B, bits.shape[1]
    if base < 0 or base + Zc * C > K:
        raise ValueError(f"mask_candidates_batched: slots {base}..{base + Zc * C} do not fit {K} candidates per cloud")
    lg = logits.float().contiguous()
    io = iou_preds.float().contiguous()
    if lengths is None:
        nv.check(nv.lib().psam_mask_candidates_batched_f32(nv.ptr(lg), nv.ptr(io), B, Zc, C, N, float(mask_threshold),
                                                           float(stability_offset), float(pred_iou_thresh), float(stability_thresh),
                                                           int(min_area), int(base), K, bits.shape[2], nv.ptr(bits), nv.ptr(area),
                                                           nv.ptr(stab), nv.ptr(score), nv.stream()), "mask_candidates_batched")
        return out
    lengths = _lengths(lengths, B, "mask_candidates_batched")
    nv.check(nv.lib().psam_mask_candidates_varlen_f32(nv.ptr(lg), nv.ptr(io), nv.ptr(lengths), B, Zc, C, N, int(num_prompts),
                                                      float(mask_threshold), float(stability_offset), float(pred_iou_thresh),
                                                      float(stability_thresh), int(min_area), int(base), K, bits.shape[2],
                                                      nv.ptr(bits), nv.ptr(area), nv.ptr(stab), nv.ptr(score), nv.stream()),
             "mask_candidates_batched")
    return out


def mask_nms_batched(bits: torch.Tensor, area: torch.Tensor, score: torch.Tensor, nms_thresh: float):
    """mask_nms on each of B clouds in the same three launches (psam_mask_nms_batched): bits [B,K,W], area / score [B,K].
    Returns (keep [B, max(K,1)] int32: each cloud's kept slots 0..K-1 in score order, keep_count [B] int32), on the device."""
    B, K, W = bits.shape
    if K > NMS_MAX_CANDIDATES:
        raise ValueError(f"mask_nms_batched: {K} candidates per cloud, at most {NMS_MAX_CANDIDATES}")
    dev = bits.device
    keep = torch.empty((B, max(K, 1)), dtype=torch.int32, device=dev)
    keep_count = torch.empty(B, dtype=torch.int32, device=dev)
    ws = torch.empty(nv.lib().psam_mask_nms_batched_workspace_bytes(B, K, W), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_mask_nms_batched(nv.ptr(bits) if K else None, nv.ptr(area) if K else None, nv.ptr(score) if K else None,
                                            B, K, W, float(nms_thresh), nv.ptr(keep), nv.ptr(keep_count), nv.ptr(ws), nv.stream()),
             "mask_nms_batched")
    return keep, keep_count


def mask_regions_batched(bits: torch.Tensor, keep: torch.Tensor, keep_count: torch.Tensor, nbr: torch.Tensor, min_area: int,
                         lengths: Optional[torch.Tensor] = None):
    """mask_regions on each of B clouds in one launch (psam_mask_regions_batched): candidate masks bits [B,K',W], kept slots
    keep [B,K] with counts keep_count [B], kNN graphs nbr [B,N,k1].  Returns (bits_out [B,K,W], area_out [B,K],
    score_out [B,K]) by kept rank; nothing waits for the device.  lengths [B] int32 (device), padded clouds
    (psam_mask_regions_varlen): cloud b's working sets hold only its first lengths[b] points."""
    B, Kc, W = bits.shape
    K = keep.shape[1]
    N, k1 = nbr.shape[-2], nbr.shape[-1]
    if keep.shape[0] != B or keep_count.numel() != B or nbr.shape[0] != B:
        raise ValueError(f"mask_regions_batched: keep {tuple(keep.shape)}, keep_count {tuple(keep_count.shape)} and nbr "
                         f"{tuple(nbr.shape)} do not match {B} clouds")
    if K > NMS_MAX_CANDIDATES:
        raise ValueError(f"mask_regions_batched: {K} kept masks per cloud, at most {NMS_MAX_CANDIDATES}")
    keep, nbr = keep.contiguous(), nbr.contiguous()
    dev = bits.device
    bits_out = torch.empty((B, K, W), dtype=torch.int32, device=dev)
    area_out = torch.empty((B, K), dtype=torch.int32, device=dev)
    score_out = torch.empty((B, K), dtype=torch.float32, device=dev)
    ws = torch.empty(nv.lib().psam_mask_regions_batched_workspace_bytes(B, K, N), dtype=torch.uint8, device=dev)
    if lengths is None:
        nv.check(nv.lib().psam_mask_regions_batched(nv.ptr(bits), Kc, B, K, W, N, nv.ptr(keep), nv.ptr(keep_count), nv.ptr(nbr), k1,
                                                    int(min_area), nv.ptr(bits_out), nv.ptr(area_out), nv.ptr(score_out), nv.ptr(ws),
                                                    nv.stream()), "mask_regions_batched")
    else:
        lengths = _lengths(lengths, B, "mask_regions_batched")
        nv.check(nv.lib().psam_mask_regions_varlen(nv.ptr(bits), Kc, nv.ptr(lengths), B, K, W, N, nv.ptr(keep), nv.ptr(keep_count),
                                                   nv.ptr(nbr), k1, int(min_area), nv.ptr(bits_out), nv.ptr(area_out),
                                                   nv.ptr(score_out), nv.ptr(ws), nv.stream()), "mask_regions_batched")
    return bits_out, area_out, score_out


# ------------------------------------------------------------------------------------------------
# crop layers of automatic mask generation
# ------------------------------------------------------------------------------------------------
CROP_MAX_LAYERS = 3


def crop_total(n_layers: int) -> int:
    """Crops of layers 0 .. n_layers: sum of 8^i."""
    return sum(8 ** i for i in range(n_layers + 1))


def crop_layout(xyz: torch.Tensor, n_layers: int, overlap_ratio: float):
    """Crop boxes and point counts of every layer (psam_crop_layout_f32).  xyz [N, 3] or [1, N, 3].  Returns (boxes [T, 6]
    fp32, counts [T] int32: -1 marks a box equal to an earlier one of its layer); both stay on the device."""
    x = xyz.reshape(-1, 3).float().contiguous()
    T = crop_total(n_layers)
    boxes = torch.empty((T, 6), dtype=torch.float32, device=x.device)
    counts = torch.empty(T, dtype=torch.int32, device=x.device)
    nv.check(nv.lib().psam_crop_layout_f32(nv.ptr(x), x.shape[0], int(n_layers), float(overlap_ratio), nv.ptr(boxes), nv.ptr(counts),
                                           nv.stream()), "crop_layout")
    return boxes, counts


def crop_gather(xyz: torch.Tensor, rgb: torch.Tensor, boxes: torch.Tensor, crop: int, count: int, edge_margin: float):
    """The crop cloud of crop `crop` with `count` points (its entry of crop_layout's counts), psam_crop_gather_f32.  Returns
    (idx [count] int32 global indices in ascending order, xyz [1, count, 3] renormalised, rgb [1, count, 3], edge
    [mask_words(count)] int32: the points near an interior face of the crop)."""
    x, c = xyz.reshape(-1, 3).float().contiguous(), rgb.reshape(-1, 3).float().contiguous()
    N, dev = x.shape[0], x.device
    idx = torch.empty(count, dtype=torch.int32, device=dev)
    xo = torch.empty((1, count, 3), dtype=torch.float32, device=dev)
    co = torch.empty((1, count, 3), dtype=torch.float32, device=dev)
    edge = torch.empty(mask_words(count), dtype=torch.int32, device=dev)
    ws = torch.empty(nv.lib().psam_crop_gather_workspace_bytes(N), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_crop_gather_f32(nv.ptr(x), nv.ptr(c), N, nv.ptr(boxes), int(crop), boxes.shape[0], float(edge_margin),
                                           int(count), nv.ptr(idx), nv.ptr(xo), nv.ptr(co), nv.ptr(edge), nv.ptr(ws), nv.stream()),
             "crop_gather")
    return idx, xo, co, edge


def crop_edge_filter(bits: torch.Tensor, score: torch.Tensor, edge: torch.Tensor):
    """score[k] = -inf in place for every candidate whose mask bits[k] touches the crop's edge bitset (psam_crop_edge_filter)."""
    K, W = bits.shape
    if edge.numel() != W or score.numel() != K:
        raise ValueError(f"crop_edge_filter: edge has {edge.numel()} words and score {score.numel()} entries for bits {tuple(bits.shape)}")
    nv.check(nv.lib().psam_crop_edge_filter(nv.ptr(bits) if K else None, K, W, nv.ptr(edge) if K else None,
                                            nv.ptr(score) if K else None, nv.stream()), "crop_edge_filter")


def crop_uncrop(cand, keep: torch.Tensor, keep_count: torch.Tensor, idx: torch.Tensor, prompt_index: torch.Tensor, slots: int,
                crop: int, layer_score: float, offsets: torch.Tensor, k: int, out, overflow: torch.Tensor, N: int):
    """Append the kept masks keep[:keep_count] of one crop to the global set (psam_crop_uncrop) of a cloud of N points.
    cand = (bits [K, W], area, stability, score) of mask_candidates on the crop's idx.numel() points; prompt_index [P] int64
    (crop-local FPS indices);
    offsets [>= k + 2] int32 device running offsets: reads offsets[k], writes offsets[k + 1]; out = (gbits [cap, Wg] int32,
    area, iou, stability, prompt int64, slot, crop int32, score fp32), each of length cap.  Sets overflow[0] = 1 when the
    set outgrows cap."""
    bits, area, stab, score = cand
    gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore = out
    cap, Wg = gbits.shape
    nv.check(nv.lib().psam_crop_uncrop(nv.ptr(bits), nv.ptr(area), nv.ptr(score), nv.ptr(stab), keep.shape[0], bits.shape[1], nv.ptr(keep),
                                       nv.ptr(keep_count), nv.ptr(idx), idx.shape[0], nv.ptr(prompt_index.reshape(-1)), int(slots), int(crop),
                                       float(layer_score), int(N), Wg, cap, nv.ptr(offsets[k:]), nv.ptr(offsets[k + 1:]), nv.ptr(gbits),
                                       nv.ptr(garea), nv.ptr(giou), nv.ptr(gstab), nv.ptr(gprompt), nv.ptr(gslot), nv.ptr(gcrop),
                                       nv.ptr(gscore), nv.ptr(overflow), nv.stream()), "crop_uncrop")


def _host_to_device(a: np.ndarray, dev) -> torch.Tensor:
    """A small host table on the device without a host synchronisation (pinned memory, asynchronous copy)."""
    host = torch.from_numpy(np.ascontiguousarray(a))
    return (host.pin_memory() if dev.type == "cuda" else host).to(dev, non_blocking=True)


def crop_layout_batched(xyz: torch.Tensor, n_layers: int, overlap_ratio: float, lengths: Optional[torch.Tensor] = None):
    """crop_layout on each cloud of xyz [B, N_max, 3] in one pair of launches (psam_crop_layout_batched_f32).  lengths [B]
    int32 (device): cloud b is its first lengths[b] rows.  Returns (boxes [B, T, 6], counts [B, T]) on the device."""
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise ValueError(f"crop_layout_batched: xyz must be [B, N, 3], got {tuple(xyz.shape)}")
    x = xyz.float().contiguous()
    B, N, dev = x.shape[0], x.shape[1], x.device
    T = crop_total(n_layers)
    if lengths is not None:
        lengths = _lengths(lengths, B, "crop_layout_batched")
    boxes = torch.empty((B, T, 6), dtype=torch.float32, device=dev)
    counts = torch.empty((B, T), dtype=torch.int32, device=dev)
    nv.check(nv.lib().psam_crop_layout_batched_f32(nv.ptr(x), nv.ptr(lengths), B, N, int(n_layers), float(overlap_ratio), nv.ptr(boxes),
                                                   nv.ptr(counts), nv.stream()), "crop_layout_batched")
    return boxes, counts


def crop_gather_batched(xyz: torch.Tensor, rgb: torch.Tensor, boxes: torch.Tensor, pairs, edge_margin: float,
                        lengths: Optional[torch.Tensor] = None):
    """The crop clouds of P (cloud, crop, count) pairs (host ints; count = the crop's entry of crop_layout_batched's counts)
    as one padded batch (psam_crop_gather_batched_f32): xyz / rgb [B, N_max, 3] with lengths [B] as for the layout, boxes
    [B, T, 6].  Returns (idx [P, n_max] int32, xyz [P, n_max, 3] renormalised, rgb [P, n_max, 3], edge [P, mask_words(n_max)]
    int32, counts [P] int32 on the device: the `lengths` of the padded batch), n_max = the largest count; row p equals
    crop_gather of its pair, and its rows past the count are 0.  Nothing waits for the device."""
    x, c = xyz.float().contiguous(), rgb.float().contiguous()
    if x.dim() != 3 or x.shape[2] != 3 or c.shape != x.shape:
        raise ValueError(f"crop_gather_batched: xyz {tuple(x.shape)} and rgb {tuple(c.shape)} must both be [B, N, 3]")
    B, N, dev = x.shape[0], x.shape[1], x.device
    if boxes.dim() != 3 or boxes.shape[0] != B or boxes.shape[2] != 6:
        raise ValueError(f"crop_gather_batched: boxes must be [{B}, T, 6], got {tuple(boxes.shape)}")
    table = np.asarray(pairs, dtype=np.int32).reshape(-1, 3)
    P = table.shape[0]
    if P < 1 or table[:, 2].min() < 1:
        raise ValueError("crop_gather_batched: need at least one pair, each with a count >= 1")
    n_max = int(table[:, 2].max())
    if lengths is not None:
        lengths = _lengths(lengths, B, "crop_gather_batched")
    table = _host_to_device(table.T, dev)
    idx = torch.empty((P, n_max), dtype=torch.int32, device=dev)
    xo = torch.empty((P, n_max, 3), dtype=torch.float32, device=dev)
    co = torch.empty((P, n_max, 3), dtype=torch.float32, device=dev)
    edge = torch.empty((P, mask_words(n_max)), dtype=torch.int32, device=dev)
    ws = torch.empty(max(1, nv.lib().psam_crop_gather_batched_workspace_bytes(P, N)), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_crop_gather_batched_f32(nv.ptr(x), nv.ptr(c), nv.ptr(lengths), B, N, nv.ptr(boxes.contiguous()), boxes.shape[1],
                                                   nv.ptr(table), P, n_max, float(edge_margin), nv.ptr(idx), nv.ptr(xo), nv.ptr(co),
                                                   nv.ptr(edge), nv.ptr(ws), nv.stream()), "crop_gather_batched")
    return idx, xo, co, edge, table[2]


def crop_edge_filter_batched(bits: torch.Tensor, score: torch.Tensor, edge: torch.Tensor):
    """crop_edge_filter on each crop of bits [T, K, W], score [T, K] and edge [T, W] in one launch
    (psam_crop_edge_filter_batched)."""
    T, K, W = bits.shape
    if tuple(edge.shape) != (T, W) or tuple(score.shape) != (T, K):
        raise ValueError(f"crop_edge_filter_batched: edge {tuple(edge.shape)} and score {tuple(score.shape)} for bits {tuple(bits.shape)}")
    nv.check(nv.lib().psam_crop_edge_filter_batched(nv.ptr(bits) if K else None, T, K, W, nv.ptr(edge) if K else None,
                                                    nv.ptr(score) if K else None, nv.stream()), "crop_edge_filter_batched")


# psam_crop_run of include/psam_b200.h
CROP_RUN = np.dtype([("bits", "<u8"), ("area", "<u8"), ("score", "<u8"), ("stability", "<u8"), ("keep", "<u8"), ("keep_count", "<u8"),
                     ("idx", "<u8"), ("prompt_index", "<u8"), ("K", "<i4"), ("W", "<i4"), ("n", "<i4"), ("slots", "<i4"), ("crop", "<i4"),
                     ("cloud", "<i4"), ("first", "<i4"), ("last", "<i4"), ("layer_score", "<f4"), ("capacity", "<i4")])


def crop_uncrop_batched(runs, out, N: int):
    """The kept masks of every crop run of B clouds lifted to their clouds in one launch (psam_crop_uncrop_batched).
    runs: per run a dict with cand = (bits [K', W], area, stability, score) of its candidates, keep [K] int32 and keep_count
    [1] (its NMS), idx (int32, the crop's point indices in its cloud: n = idx.numel()), prompt_index (int64, crop-local), slots,
    crop, layer, cloud and capacity (its cloud's); the runs of a cloud consecutive and in the cloud's crop order, every cloud
    0 .. B-1 with at least one.  out = (gbits [B, cap, Wg] int32, area, iou, stability, prompt int64, slot, crop int32,
    score fp32, each [B, cap]); N = the clouds' N_max.  Returns (lifted [B], overflow [B]) int32 on the device: each cloud's
    kept count over all its runs and 1 where it exceeds the cloud's capacity.  The slices in `runs` must stay alive until the
    launch has run (the caller holds them)."""
    gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore = out
    B, cap, Wg = gbits.shape
    dev = gbits.device
    if nv.lib().psam_crop_run_bytes() != CROP_RUN.itemsize:
        raise RuntimeError(f"crop_uncrop_batched: psam_crop_run is {nv.lib().psam_crop_run_bytes()} bytes, the binding lays out "
                           f"{CROP_RUN.itemsize}")
    table = np.zeros(len(runs), dtype=CROP_RUN)
    first, K_max = 0, 1
    for r, run in enumerate(runs):
        bits, area, stab, score = run["cand"]
        if bits.dim() != 2 or not bits.is_contiguous() or run["idx"].dim() != 1:
            raise ValueError("crop_uncrop_batched: each run's bits must be a contiguous [K, W] slice and its idx one row")
        if r and runs[r - 1]["cloud"] != run["cloud"]:
            first = r
        last = r + 1 == len(runs) or runs[r + 1]["cloud"] != run["cloud"]
        if not 0 <= run["cloud"] < B or not 1 <= run["capacity"] <= cap or (r and run["cloud"] < runs[r - 1]["cloud"]):
            raise ValueError(f"crop_uncrop_batched: run {r} has cloud {run['cloud']} and capacity {run['capacity']} for {B} clouds of "
                             f"{cap} rows (runs grouped by cloud in ascending order)")
        keep = run["keep"]
        K_max = max(K_max, keep.numel())
        table[r] = (nv.ptr(bits), nv.ptr(area), nv.ptr(score), nv.ptr(stab), nv.ptr(keep), nv.ptr(run["keep_count"]), nv.ptr(run["idx"]),
                    nv.ptr(run["prompt_index"]), keep.numel(), bits.shape[1], run["idx"].numel(), int(run["slots"]), int(run["crop"]),
                    int(run["cloud"]), first, int(last), float(run["layer"]), int(run["capacity"]))
    if sorted({int(r["cloud"]) for r in runs}) != list(range(B)):
        raise ValueError(f"crop_uncrop_batched: every one of the {B} clouds needs at least one run")
    dtable = _host_to_device(table.view(np.uint8), dev)
    lifted = torch.empty(B, dtype=torch.int32, device=dev)
    overflow = torch.empty(B, dtype=torch.int32, device=dev)
    nv.check(nv.lib().psam_crop_uncrop_batched(nv.ptr(dtable), len(runs), K_max, B, int(N), Wg, cap, nv.ptr(gbits), nv.ptr(garea),
                                               nv.ptr(giou), nv.ptr(gstab), nv.ptr(gprompt), nv.ptr(gslot), nv.ptr(gcrop), nv.ptr(gscore),
                                               nv.ptr(lifted), nv.ptr(overflow), nv.stream()), "crop_uncrop_batched")
    return lifted, overflow


# ------------------------------------------------------------------------------------------------
# meshes and dense clouds
# ------------------------------------------------------------------------------------------------
def mesh_sample(vertices: torch.Tensor, faces: torch.Tensor, S: int, seed: int = 0, vertex_colors=None, uv=None, texture=None):
    """S area-weighted samples of a triangle mesh (psam_mesh_sample_f32): vertices [V, 3] fp32, faces [F, 3] int32, optional
    vertex_colors [V, 3] fp32, or uv [V, 2] fp32 with texture [H, W, C] uint8 (C = 3 or 4).  Returns (xyz [S, 3], rgb [S, 3],
    face [S] int32, stats [3] int64 = (total weight, bad faces, faces with an index outside [0, V))), all on the device;
    nothing waits for it."""
    v = vertices.reshape(-1, 3).float().contiguous()
    f = faces.reshape(-1, 3).to(torch.int32).contiguous()
    V, F, dev = v.shape[0], f.shape[0], v.device
    vc = vertex_colors.reshape(V, 3).float().contiguous() if vertex_colors is not None else None
    tuv = uv.reshape(V, 2).float().contiguous() if uv is not None else None
    tex = texture.contiguous() if texture is not None else None
    if tex is not None and (tex.dim() != 3 or tex.dtype != torch.uint8):
        raise ValueError(f"mesh_sample: texture must be uint8 [H, W, C], got {tex.dtype} {tuple(tex.shape)}")
    H, W, C = tuple(tex.shape) if tex is not None else (0, 0, 0)
    xyz = torch.empty((S, 3), dtype=torch.float32, device=dev)
    rgb = torch.empty((S, 3), dtype=torch.float32, device=dev)
    face = torch.empty(S, dtype=torch.int32, device=dev)
    stats = torch.empty(3, dtype=torch.int64, device=dev)
    ws = torch.empty(nv.lib().psam_mesh_sample_workspace_bytes(F), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_mesh_sample_f32(nv.ptr(v), V, nv.ptr(f), F, int(S), int(seed) & (2 ** 64 - 1), nv.ptr(vc), nv.ptr(tuv),
                                           nv.ptr(tex), H, W, C, nv.ptr(xyz), nv.ptr(rgb), nv.ptr(face), nv.ptr(stats), nv.ptr(ws),
                                           nv.stream()), "mesh_sample")
    return xyz, rgb, face, stats


def mesh_face_centers(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """((a + b) + c) / 3 of every face (psam_mesh_face_centers_f32): [F, 3] fp32, NaN for a face with a bad index."""
    v = vertices.reshape(-1, 3).float().contiguous()
    f = faces.reshape(-1, 3).to(torch.int32).contiguous()
    centers = torch.empty((f.shape[0], 3), dtype=torch.float32, device=v.device)
    nv.check(nv.lib().psam_mesh_face_centers_f32(nv.ptr(v), v.shape[0], nv.ptr(f), f.shape[0], nv.ptr(centers), nv.stream()),
             "mesh_face_centers")
    return centers


def mask_lift(bits: torch.Tensor, nearest: torch.Tensor, S: int):
    """Masks over S points carried to M points through their nearest point (psam_mask_lift): bits [K, W >= mask_words(S)]
    int32, nearest [M] int64 (entries outside [0, S) read as 0).  Returns (bits [K, mask_words(M)] int32, area [K] int32)."""
    K, Ws = bits.shape
    near = nearest.reshape(-1).to(torch.int64).contiguous()
    M, dev = near.shape[0], bits.device
    Wm = mask_words(M)
    out = torch.empty((K, Wm), dtype=torch.int32, device=dev)
    area = torch.empty(K, dtype=torch.int32, device=dev)
    b = bits.contiguous()
    nv.check(nv.lib().psam_mask_lift(nv.ptr(b) if K else None, K, Ws, int(S), nv.ptr(near), M, Wm, nv.ptr(out) if K else None,
                                     nv.ptr(area) if K else None, nv.stream()), "mask_lift")
    return out, area


def mask_label_map(bits: torch.Tensor, priority: torch.Tensor, N: int) -> torch.Tensor:
    """One label per point (psam_mask_label_map): the row of bits [K, W >= mask_words(N)] containing the point with the
    smallest priority [K] (int32), ties to the lower row, -1 for a point in no row.  Returns labels [N] int32."""
    K, W = bits.shape
    pr = priority.reshape(-1).to(torch.int32).contiguous()
    if pr.shape[0] != K:
        raise ValueError(f"mask_label_map: {pr.shape[0]} priorities for {K} masks")
    labels = torch.empty(int(N), dtype=torch.int32, device=bits.device)
    b = bits.contiguous()
    nv.check(nv.lib().psam_mask_label_map(nv.ptr(b) if K else None, K, W, nv.ptr(pr) if K else None, int(N), nv.ptr(labels),
                                          nv.stream()), "mask_label_map")
    return labels


# ------------------------------------------------------------------------------------------------
# dense scans
# ------------------------------------------------------------------------------------------------
def nearest_grid(query: torch.Tensor, key: torch.Tensor):
    """Nearest key of every query point on a uniform grid (psam_nn_grid_f32): query [n1, 3], key [n2, 3] (any leading shape,
    fp32).  Returns (dist [n1] fp32, idx [n1] int64), bit for bit those of psam_nn_distance_f32: exact squared distance, ties
    to the lower key index, (3.4e38, -1) for a query with no finite distance.  Nothing waits for the device."""
    q = query.reshape(-1, 3).float().contiguous()
    k = key.reshape(-1, 3).float().contiguous()
    n1, n2, dev = q.shape[0], k.shape[0], q.device
    dist = torch.empty(n1, dtype=torch.float32, device=dev)
    idx = torch.empty(n1, dtype=torch.int64, device=dev)
    ws = torch.empty(nv.lib().psam_nn_grid_workspace_bytes(n2), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_nn_grid_f32(nv.ptr(q), n1, nv.ptr(k), n2, nv.ptr(dist), nv.ptr(idx), nv.ptr(ws), nv.stream()), "nn_grid")
    return dist, idx


def voxel_subsample(xyz: torch.Tensor, S: int, seed: int = 0):
    """At most S points of xyz [P, 3] (normalised fp32), one per occupied voxel of the coarsest level with at least S voxels
    (psam_voxel_subsample_f32).  Returns (idx [S] int64: the kept indices ascending, then -1; stats [4] int64 = (valid
    points, level, occupied voxels, kept)), both on the device; nothing waits for it."""
    x = xyz.reshape(-1, 3).float().contiguous()
    P, dev = x.shape[0], x.device
    idx = torch.empty(int(S), dtype=torch.int64, device=dev)
    stats = torch.empty(4, dtype=torch.int64, device=dev)
    ws = torch.empty(nv.lib().psam_voxel_subsample_workspace_bytes(P), dtype=torch.uint8, device=dev)
    nv.check(nv.lib().psam_voxel_subsample_f32(nv.ptr(x), P, int(S), int(seed) & (2 ** 64 - 1), nv.ptr(idx), nv.ptr(stats), nv.ptr(ws),
                                               nv.stream()), "voxel_subsample")
    return idx, stats
