"""Fine-tuning of ``mask_decoder`` on a frozen encoder (the reference's train.py with only the prompt decoder learning).

Split of the work, by where the FLOPs and the memory are:
  * the token / patch-level trunk (token and src preparation, the two-way transformer, hyper-network MLPs, IoU head,
    output_upscaling[0] on the G patch rows) is differentiable torch code over the live ``mask_decoder`` parameters;
  * the per-point mask head (3-NN interpolation, output_upscaling[1..4], the hyper-network product) is ``MaskHead``: its
    forward is the engine's inference code (``engine.upscale_ln_gelu`` + ``engine.mask_product``), and its backward is
    CUDA (csrc/train.cu + the split-bf16 GEMM).  It saves f0, hyper and the decoder weights only - never a tensor of
    Z * N * D elements - and recomputes the per-point activations in backward, one chunk of rows at a time;
  * the mask loss (``mask_loss``, pc_sam.model.loss.Criterion) is two CUDA kernels: per-row statistics, then dlogits.

The fused row-dot of the forward accumulates the C mask logits of a point with float atomics, so the logits of two runs may
differ in the last bit; everything downstream of given logits (loss, dlogits, every head gradient) is bitwise reproducible.
"""
from __future__ import annotations

import math
import types

import torch
import torch.nn.functional as F

from . import engine
from . import native as nv
from . import ops
from .ops import Split

# rows (points x prompts) of one backward chunk: the transient per-point buffers are about 5 * rows * D * 4 bytes
# (1.3 GB at D = 256)
BACKWARD_ROWS = 262144
# K rows of each partial product of the weight gradient dW3 = dp^T u1 (fixed partial buffers, summed in a fixed order)
DW_SPLIT_K = 4096
LN_ROWS_PER_BLOCK = 256
# decoder widths of psam_interp_ln_gelu_backward, and the most patches psam_interp_inverse sorts in one CTA
TRAIN_WIDTHS = (128, 256, 512)
MAX_TRAIN_GROUPS = 8192


def check_head_shape(D: int, G: int):
    """Refuses a decoder width or patch count the head backward has no kernel for (NotImplementedError), so that training
    stops before any device work rather than in loss.backward()."""
    if D not in TRAIN_WIDTHS:
        raise NotImplementedError(f"fine-tuning supports decoder widths {', '.join(map(str, TRAIN_WIDTHS))} (the LayerNorm "
                                  f"backward of the mask head), got {D}")
    if G > MAX_TRAIN_GROUPS:
        raise NotImplementedError(f"fine-tuning supports at most {MAX_TRAIN_GROUPS} patches per cloud (the inverse of the "
                                  f"interpolation index), got {G}")


# ------------------------------------------------------------------------------------------------
# interpolation geometry (3-NN index, weights and its inverse), cached per encoded cloud on AuxInputs
# ------------------------------------------------------------------------------------------------
def interp_inverse(idx: torch.Tensor, G: int):
    """idx [B,N,3] int64 -> (offsets [B, G+1] int32, entries [B, 3N] int32): per cloud and patch, the entries n * 3 + k that
    interpolate from it, ascending (psam_interp_inverse)."""
    B, N, _ = idx.shape
    offsets = torch.empty((B, G + 1), dtype=torch.int32, device=idx.device)
    entries = torch.empty((B, 3 * N), dtype=torch.int32, device=idx.device)
    nv.check(nv.lib().psam_interp_inverse(nv.ptr(idx.contiguous()), B, N, G, nv.ptr(offsets), nv.ptr(entries), nv.stream()),
             "interp_inverse")
    return offsets, entries


def head_geometry(aux, G: int, rep: int, eps: float):
    """The per-cloud interpolation data of the head, computed once per encoded cloud: the inverse index is cached on
    ``aux`` next to interp_index (and rebuilt if interp_index is replaced)."""
    if aux.interp_index is None or aux.interp_weight is None:
        aux.interp_index, aux.interp_weight = ops.knn3_interp(aux.coords.float().contiguous(), aux.centers.float().contiguous())
    inv = aux.interp_inverse
    if inv is None or inv[0] is not aux.interp_index:
        inv = (aux.interp_index,) + interp_inverse(aux.interp_index, G)
        aux.interp_inverse = inv
    return types.SimpleNamespace(idx=aux.interp_index, w=aux.interp_weight.contiguous(), offsets=inv[1], entries=inv[2],
                                 B=aux.interp_index.shape[0], N=aux.interp_index.shape[1], G=G, rep=rep, eps=float(eps))


def _f32(t):
    return t.detach().float().contiguous()


def _sum_partials(part: torch.Tensor, nb: int, S: int, n: int, out: torch.Tensor):
    nv.check(nv.lib().psam_sum_partials(nv.ptr(part), nb, S, n, nv.ptr(out), nv.stream()), "sum_partials")
    return out


class MaskHead(torch.autograd.Function):
    """masks [Z,C,N] = hyper . GELU(W3 GELU(LN(interp(f0))) + b3): output_upscaling[1..4] and the hyper-network product
    (mask_decoder.py:146-176) with output_upscaling[0] already applied to the patch rows (f0 [Z*G, D])."""

    @staticmethod
    def forward(ctx, f0, hyper, gamma, beta, w3, b3, geo):
        Z, C, D = hyper.shape
        f0c, hc = _f32(f0), _f32(hyper)
        g, b, bb = _f32(gamma), _f32(beta), _f32(b3)
        u1 = engine.upscale_ln_gelu(f0c, Z, geo.rep, geo.G, D, geo.idx, geo.w, geo.N, (g, b, geo.eps))
        masks = engine.mask_product(u1, ops.pack_weight(w3), bb, hc, Z, C, geo.N)
        ctx.save_for_backward(f0c, hc, g, b, _f32(w3), bb)
        ctx.geo = geo
        return masks

    @staticmethod
    def backward(ctx, dm):
        f0, hyper, gamma, beta, w3, b3 = ctx.saved_tensors
        geo = ctx.geo
        n_f0, n_hyper, n_gamma, n_beta, n_w3, n_b3 = ctx.needs_input_grad[:6]
        grads = head_backward(f0, hyper, gamma, beta, w3, b3, geo, dm.float().contiguous(),
                              need_f0=n_f0, need_ln=n_gamma or n_beta, need_w3=n_w3)
        df0, dhyper, dgamma, dbeta, dw3, db3 = grads
        return (df0 if n_f0 else None, dhyper if n_hyper else None, dgamma if n_gamma else None, dbeta if n_beta else None,
                dw3 if n_w3 else None, db3 if n_b3 else None, None)


def head_backward(f0, hyper, gamma, beta, w3, b3, geo, dm, need_f0=True, need_ln=True, need_w3=True):
    """Gradients of MaskHead for the upstream gradient dm [Z,C,N]: (df0 [Z*G,D], dhyper [Z,C,D], dgamma, dbeta, dW3, db3);
    df0 / (dgamma, dbeta) / dW3 are None when not needed.  Rows are processed in chunks of one cloud's prompts at a time
    (at most BACKWARD_ROWS rows), recomputing u1 = GELU(LN(interp f0)) and p = u1 W3^T + b3 per chunk."""
    Z, C, D = hyper.shape
    N, G, rep = geo.N, geo.G, geo.rep
    dev = hyper.device
    need_du = need_f0 or need_ln
    w3s = ops.pack_weight(w3)
    w3t = ops.pack_weight(w3.t()) if need_du else None  # du1 = dp W3: the GEMM's W operand is W3^T
    K = nv.lib().psam_head_dp_chunks(N)
    part_h = torch.empty((Z, K, C, D), dtype=torch.float32, device=dev)
    part_b = torch.empty((Z, K, D), dtype=torch.float32, device=dev)
    zc = max(1, min(rep, BACKWARD_ROWS // N))
    chunks = [(b, z0, min((b + 1) * rep, z0 + zc)) for b in range(Z // rep) for z0 in range(b * rep, (b + 1) * rep, zc)]
    df0 = torch.empty((Z * G, D), dtype=torch.float32, device=dev) if need_f0 else None
    part_w, part_ln = [], []
    up1 = (gamma, beta, geo.eps)
    for b, z0, z1 in chunks:
        nz = z1 - z0
        R = nz * N
        idx_b, w_b = geo.idx[b:b + 1], geo.w[b:b + 1]
        f0_c = f0[z0 * G:z1 * G]
        u1 = engine.upscale_ln_gelu(f0_c, nz, nz, G, D, idx_b, w_b, N, up1)
        p = torch.empty((R, D), dtype=torch.float32, device=dev)
        ops.gemm(u1, w3s, bias=b3, out_f32=p, passes=engine.PASSES)
        dps = Split(R, D, dev)
        nv.check(nv.lib().psam_head_dp(nv.ptr(p), nv.ptr(dm[z0:z1]), nv.ptr(hyper[z0:z1]), nz, C, N, D, dps.ptr(), dps.plane,
                                       dps.pitch, nv.ptr(part_h[z0:z1]), nv.ptr(part_b[z0:z1]), nv.stream()), "head_dp")
        if need_w3:
            part_w.append(_dw_partials(dps, u1, R))
        if need_du:
            du = p  # p is dead after head_dp: du1 = dp W3 overwrites it, and the LayerNorm backward turns it into dv in place
            ops.gemm(dps, w3t, out_f32=du, passes=engine.PASSES)
            nblk = (R + LN_ROWS_PER_BLOCK - 1) // LN_ROWS_PER_BLOCK
            pl = torch.empty((nblk, 2, D), dtype=torch.float32, device=dev)
            nv.check(nv.lib().psam_interp_ln_gelu_backward(nv.ptr(f0_c), nz, nz, G, D, nv.ptr(idx_b), nv.ptr(w_b), N, nv.ptr(gamma),
                                                           nv.ptr(beta), geo.eps, nv.ptr(du), nv.ptr(pl), LN_ROWS_PER_BLOCK,
                                                           nv.stream()), "interp_ln_gelu_backward")
            part_ln.append(pl)
            if need_f0:
                nv.check(nv.lib().psam_interp_backward(nv.ptr(du), nz, nz, G, D, nv.ptr(geo.offsets[b]), nv.ptr(geo.entries[b]),
                                                       nv.ptr(w_b), N, nv.ptr(df0[z0 * G:z1 * G]), nv.stream()), "interp_backward")
        del u1, p, dps
    dhyper = _sum_partials(part_h, Z, K, C * D, torch.empty((Z, C, D), dtype=torch.float32, device=dev))
    db3 = _sum_partials(part_b, 1, Z * K, D, torch.empty(D, dtype=torch.float32, device=dev))
    dw3 = dgamma = dbeta = None
    if need_w3:
        pw = torch.cat(part_w) if len(part_w) > 1 else part_w[0]
        dw3 = _sum_partials(pw, 1, pw.shape[0], D * D, torch.empty((D, D), dtype=torch.float32, device=dev))
    if need_ln:
        pl = torch.cat(part_ln) if len(part_ln) > 1 else part_ln[0]
        gb = _sum_partials(pl, 1, pl.shape[0], 2 * D, torch.empty((2, D), dtype=torch.float32, device=dev))
        dgamma, dbeta = gb[0], gb[1]
    return df0, dhyper, dgamma, dbeta, dw3, db3


def _dw_partials(dy: Split, x: Split, R: int) -> torch.Tensor:
    """A weight gradient dW = dy^T x over R rows (dy [R, n], x [R, k]) as S partial products [S, n, k] of DW_SPLIT_K rows
    each: both operands are transposed to [n | k, R] (psam_transpose_split) and the K axis is cut into S batches of the
    split-bf16 GEMM (operand batch dimension with a column stride), zero-padded to S * Kc columns."""
    n, k, dev = dy.cols, x.cols, dy.t.device
    S = max(1, -(-R // DW_SPLIT_K))
    Kc = ops._round_up(-(-R // S), 64)
    Kp = S * Kc
    outs = torch.empty((S, n, k), dtype=torch.float32, device=dev)
    ts = []
    for src in (dy, x):
        t = Split(src.cols, Kp, dev, pitch=Kp, zero=Kp != R)
        nv.check(nv.lib().psam_transpose_split(src.ptr(), src.plane, src.pitch, 0, 0, t.ptr(), t.plane, t.pitch, 0, 0, R, src.cols,
                                               1, 1, nv.stream()), "transpose_split")
        ts.append(t)
    a = ts[0].operand(rows=n, k=Kc, nb1=S, b1_stride=Kc)
    w = ts[1].operand(rows=k, k=Kc, nb1=S, b1_stride=Kc)
    o = ops.GemmOut()
    o.out_f32, o.ldo, o.out_b1 = nv.ptr(outs), k, n * k
    o.alpha = 1.0
    ops.gemm_raw(a, w, o, engine.PASSES, 1)
    return outs


def _weight_grad(dy: Split, x: Split, R: int) -> torch.Tensor:
    """dW = dy^T x [n, k] over R rows, the partials finished in a fixed order."""
    pw = _dw_partials(dy, x, R)
    return _sum_partials(pw, 1, pw.shape[0], dy.cols * x.cols, torch.empty((dy.cols, x.cols), dtype=torch.float32, device=pw.device))


def _col_sum(t: torch.Tensor) -> torch.Tensor:
    """Column sums of t [R, n] fp32 (a bias gradient), sequential over the rows."""
    return _sum_partials(t, 1, t.shape[0], t.shape[1], torch.empty(t.shape[1], dtype=torch.float32, device=t.device))


# ------------------------------------------------------------------------------------------------
# mask loss (pc_sam/model/loss.py:58-77) and its hard IoU (:80-98)
# ------------------------------------------------------------------------------------------------
DICE_EPS = 1e-3
DICE_WEIGHT = 2.0


class MaskLoss(torch.autograd.Function):
    """loss [Z,C] = mean_n focal + 2 dice of logits [Z,C,N] against gt [Z,N] bool; also returns (non-differentiable)
    stats [Z,C,4] = (sum focal, sum p t, sum p^2, sum t) and counts [Z,C,2] int32 = (|pred & gt|, |pred | gt|)."""

    @staticmethod
    def forward(ctx, logits, gt):
        Z, C, N = logits.shape
        x = logits.detach().float().contiguous()
        g = gt.contiguous().view(torch.uint8)
        stats = torch.empty((Z, C, 4), dtype=torch.float32, device=x.device)
        counts = torch.empty((Z, C, 2), dtype=torch.int32, device=x.device)
        nv.check(nv.lib().psam_mask_loss_stats(nv.ptr(x), nv.ptr(g), Z, C, N, nv.ptr(stats), nv.ptr(counts), nv.stream()),
                 "mask_loss_stats")
        dice = 1.0 - (2.0 * stats[..., 1] + DICE_EPS) / (stats[..., 2] + stats[..., 3] + DICE_EPS)
        loss = stats[..., 0] / N + DICE_WEIGHT * dice
        ctx.save_for_backward(x, g, stats)
        ctx.mark_non_differentiable(stats, counts)
        return loss, stats, counts

    @staticmethod
    def backward(ctx, dloss, _dstats, _dcounts):
        x, g, stats = ctx.saved_tensors
        Z, C, N = x.shape
        dl = torch.empty_like(x)
        nv.check(nv.lib().psam_mask_loss_grad(nv.ptr(x), nv.ptr(g), Z, C, N, nv.ptr(stats), nv.ptr(dloss.float().contiguous()),
                                              nv.ptr(dl), nv.stream()), "mask_loss_grad")
        return dl, None


def mask_loss(logits: torch.Tensor, gt: torch.Tensor):
    """(loss [Z,C], stats [Z,C,4], counts [Z,C,2]) of logits [Z,C,N] against gt [Z,N] bool (MaskLoss)."""
    if logits.dim() != 3 or gt.dim() != 2 or gt.shape != (logits.shape[0], logits.shape[2]):
        raise ValueError(f"mask_loss: logits must be [Z,C,N] and gt [Z,N], got {tuple(logits.shape)} and {tuple(gt.shape)}")
    if gt.dtype != torch.bool:
        raise TypeError(f"mask_loss: gt must be bool, got {gt.dtype}")
    return MaskLoss.apply(logits, gt)


# ------------------------------------------------------------------------------------------------
# the token / patch-level trunk in torch autograd (transformer.py, mask_decoder.py:126-145)
# ------------------------------------------------------------------------------------------------
def _linear(m, x):
    return F.linear(x, m.weight, m.bias)


def _ln(m, x):
    return F.layer_norm(x, (x.shape[-1],), m.weight, m.bias, m.eps)


def _attention(a, q, k, v):
    """SAM's Attention (transformer.py:183-236) with downsample: heads over internal_dim."""
    q, k, v = _linear(a.q_proj, q), _linear(a.k_proj, k), _linear(a.v_proj, v)
    Z, Lq, Di = q.shape
    H = a.num_heads
    split = lambda t: t.reshape(Z, t.shape[1], H, Di // H).transpose(1, 2)
    q, k, v = split(q), split(k), split(v)
    attn = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(Di // H), dim=-1)
    out = (attn @ v).transpose(1, 2).reshape(Z, Lq, Di)
    return _linear(a.out_proj, out)


def two_way_transformer(tr, src, pos_src, tokens):
    """TwoWayTransformer.forward (transformer.py:55-100): returns (queries [Z,T,D], keys [Z,G,D])."""
    queries, keys = tokens, src
    for l in tr.layers:
        if l.skip_first_layer_pe:
            queries = _attention(l.self_attn, queries, queries, queries)
        else:
            q = queries + tokens
            queries = queries + _attention(l.self_attn, q, q, queries)
        queries = _ln(l.norm1, queries)
        q, k = queries + tokens, keys + pos_src
        queries = _ln(l.norm2, queries + _attention(l.cross_attn_token_to_image, q, k, keys))
        queries = _ln(l.norm3, queries + _linear(l.mlp.lin2, l.mlp.act(_linear(l.mlp.lin1, queries))))
        q, k = queries + tokens, keys + pos_src
        keys = _ln(l.norm4, keys + _attention(l.cross_attn_image_to_token, k, q, queries))
    q, k = queries + tokens, keys + pos_src
    queries = _ln(tr.norm_final_attn, queries + _attention(tr.final_attn_token_to_image, q, k, keys))
    return queries, keys


def _mlp(m, x):
    for i, layer in enumerate(m.layers):
        x = F.relu(_linear(layer, x)) if i < m.num_layers - 1 else _linear(layer, x)
    return torch.sigmoid(x) if m.sigmoid_output else x


def decoder_trunk(md, pc_embeddings, pc_pe, sparse, dense, multimask_output: bool):
    """mask_decoder.py:126-145 and the token-side heads: returns (f0 [Z*G, D] = output_upscaling[0](keys), hyper [Z,C,D],
    iou_pred [Z,C]) as differentiable functions of md's parameters."""
    Z = sparse.shape[0]
    B, G, D = pc_embeddings.shape
    rep = Z // B
    mask_slice = slice(1, None) if multimask_output else slice(0, 1)
    out_tokens = torch.cat([md.iou_token.weight, md.mask_tokens.weight], dim=0)
    tokens = torch.cat((out_tokens.unsqueeze(0).expand(Z, -1, -1), sparse.float()), dim=1)
    src = torch.repeat_interleave(pc_embeddings.float(), rep, dim=0)
    if dense.shape[0] != Z:
        dense = torch.repeat_interleave(dense, Z // dense.shape[0], dim=0)
    src = src + dense.float()
    pos_src = torch.repeat_interleave(pc_pe.float(), rep, dim=0)
    hs, keys = two_way_transformer(md.transformer, src, pos_src, tokens)
    f0 = _linear(md.output_upscaling[0], keys).reshape(Z * G, D)
    ids = list(range(md.num_mask_tokens))[mask_slice]
    hyper = torch.stack([_mlp(md.output_hypernetworks_mlps[i], hs[:, 1 + i, :]) for i in ids], dim=1)
    iou_pred = _mlp(md.iou_prediction_head, hs[:, 0, :])[:, mask_slice]
    return f0, hyper, iou_pred


def run_mask_decoder_train(md, pc_embeddings, pc_pe, sparse, dense, aux, multimask_output: bool):
    """MaskDecoder.forward with autograd into md's parameters: the torch trunk, then MaskHead.  Returns (masks [Z,C,N],
    iou_preds [Z,C]), both with grad_fn when any decoder parameter requires grad."""
    if hasattr(md, "output_upscaling2"):
        raise NotImplementedError("fine-tuning covers MaskDecoder; the backward of MaskDecoderHier is not implemented")
    Z = sparse.shape[0]
    B, G, _ = pc_embeddings.shape
    check_head_shape(md.transformer_dim, G)
    f0, hyper, iou_pred = decoder_trunk(md, pc_embeddings, pc_pe, sparse, dense, multimask_output)
    up = md.output_upscaling
    geo = head_geometry(aux, G, Z // B, up[1].eps)
    masks = MaskHead.apply(f0, hyper, up[1].weight, up[1].bias, up[3].weight, up[3].bias, geo)
    return masks, iou_pred


# ------------------------------------------------------------------------------------------------
# the point-cloud encoder: EvaBlock backward recomputed from each block's input (pc_encoder.py:118-145)
# ------------------------------------------------------------------------------------------------
# most attention score rows (clouds x heads x L) one chunk of the block backward holds: six transient [rows, L] buffers of
# 4 bytes per element, about 0.8 GB at the limit
ATTENTION_SCORE_ELEMS = 1 << 25
ENCODER_TRAINABLE = ("transformer.blocks.", "transformer.norm.", "transformer.fc_norm.", "out_proj.", "patch_proj.", "pos_embed.")


def check_block_shape(blk, D: int):
    """Refuses a trainable EvaBlock whose shapes the backward has no kernel for (NotImplementedError, before any device
    work): its split-bf16 operands start at column offsets h * dh, D and 2 D, which the GEMM needs 16-byte aligned."""
    H = blk.attn.num_heads
    if D % H or D % 8 or (D // H) % 8:
        raise NotImplementedError(f"encoder fine-tuning supports blocks whose width and head dim are multiples of 8, got width {D} "
                                  f"with {H} heads")


class _SplitRows(Split):
    """Rows [r0, r0 + n) of a split-bf16 matrix, sharing its storage (the lo plane stays one full plane after the hi)."""
    __slots__ = ("_plane",)

    def __init__(self, s: Split, r0: int, n: int):
        self.t, self.rows, self.cols, self.pitch, self._plane = s.t[:, r0:r0 + n], n, s.cols, s.pitch, s.plane

    @property
    def plane(self) -> int:
        return self._plane


def _transposes(pb, blk):
    """W^T operands of the block's dX products, packed on the first backward and kept with the block's pack."""
    if pb.transposed is None:
        D = pb.D
        mlp = blk.mlp
        wqkv, _ = engine.qkv_weights(blk.attn, D)
        if pb.swiglu:
            w1 = engine.swiglu_fc1(mlp, pb.hp)[0]
            w2 = engine.swiglu_fc2(mlp, pb.hp)
        else:
            w1, w2 = mlp.fc1.weight.detach().float(), mlp.fc2.weight.detach().float()
        pack_t = lambda w: ops.pack_weight(w.t())
        pb.transposed = types.SimpleNamespace(wqkv=pack_t(wqkv), wproj=pack_t(blk.attn.proj.weight.detach().float()), w1=pack_t(w1),
                                              w2=pack_t(w2))
    return pb.transposed


def _ln_backward(x, dy, gamma, eps, dres=None, out_split=None):
    """(dx [M, D], part [blocks, 2, D]) of a LayerNorm over the rows of x (psam_layernorm_backward)."""
    M, D = x.shape
    dx = torch.empty_like(x)
    nblk = (M + LN_ROWS_PER_BLOCK - 1) // LN_ROWS_PER_BLOCK
    part = torch.empty((nblk, 2, D), dtype=torch.float32, device=x.device)
    nv.check(nv.lib().psam_layernorm_backward(nv.ptr(x), D, M, D, nv.ptr(dy), dy.shape[1], nv.ptr(gamma), float(eps), nv.ptr(dres), D,
                                              nv.ptr(dx), D, out_split.ptr() if out_split is not None else None,
                                              out_split.plane if out_split is not None else 0,
                                              out_split.pitch if out_split is not None else 0, nv.ptr(part), LN_ROWS_PER_BLOCK,
                                              nv.stream()), "layernorm_backward")
    return dx, part


def _ln_params(part):
    nblk, _, D = part.shape
    gb = _sum_partials(part, 1, nblk, 2 * D, torch.empty((2, D), dtype=torch.float32, device=part.device))
    return gb[0], gb[1]


def _attention_backward(qkv: Split, datt: Split, dqkv: torch.Tensor, B: int, L: int, H: int, dh: int, D: int):
    """dqkv [B*L, 3D] fp32 (dQ | dK | dV) from datt = dL/d(attention output), per (cloud, head) through the GEMM's batch
    dimensions: S = Q K^T recomputed, dP = dO V^T, dS = scale P (dP - rowsum(dP P)), dQ = dS K, dK = dS^T Q, dV = P^T dO.
    Clouds are processed in chunks of at most ATTENTION_SCORE_ELEMS score elements."""
    dev = dqkv.device
    Lp = ops._round_up(L, 64)
    scale = dh ** -0.5
    cpc = max(1, ATTENTION_SCORE_ELEMS // (H * L * Lp))
    for c0 in range(0, B, cpc):
        nb = min(cpc, B - c0)
        q, dO = _SplitRows(qkv, c0 * L, nb * L), _SplitRows(datt, c0 * L, nb * L)
        rows = nb * H * L

        def heads_t(src, col):  # [nb, H, dh, Lp]: the per-head column block of src transposed
            t = Split(nb * H * dh, L, dev, pitch=Lp, zero=Lp != L)
            nv.check(nv.lib().psam_transpose_split(src.ptr(col), src.plane, src.pitch, dh, L * src.pitch, t.ptr(), t.plane, t.pitch,
                                                   dh * Lp, H * dh * Lp, L, dh, H, nb, nv.stream()), "transpose_split")
            return t.operand(rows=dh, k=L, nb1=H, b1_stride=dh * Lp, nb2=nb, b2_stride=H * dh * Lp)

        def heads(src, col):  # per-head [L, dh] blocks of src
            return src.operand(rows=L, k=dh, col=col, nb1=H, b1_stride=dh, nb2=nb, b2_stride=L * src.pitch)

        def square(t: Split):  # per-head [L, L] blocks
            return t.operand(rows=L, k=L, nb1=H, b1_stride=L * Lp, nb2=nb, b2_stride=H * L * Lp)

        def scores(a, w):
            out = torch.empty((rows, L), dtype=torch.float32, device=dev)
            o = ops.GemmOut()
            o.out_f32, o.ldo, o.out_b1, o.out_b2 = nv.ptr(out), L, L * L, H * L * L
            o.alpha = 1.0
            ops.gemm_raw(a, w, o, engine.PASSES, 1)
            return out

        def into_dqkv(a, w, col):
            o = ops.GemmOut()
            o.out_f32, o.ldo, o.out_b1, o.out_b2 = nv.ptr(dqkv) + 4 * (c0 * L * 3 * D + col), 3 * D, dh, L * 3 * D
            o.alpha = 1.0
            ops.gemm_raw(a, w, o, engine.PASSES, 1)

        s = scores(heads(q, 0), heads(q, D))
        dp = scores(heads(dO, 0), heads(q, 2 * D))
        ds = Split(rows, L, dev, pitch=Lp, zero=Lp != L)
        nv.check(nv.lib().psam_softmax_backward(nv.ptr(s), L, nv.ptr(dp), L, rows, L, scale, ds.ptr(), ds.plane, ds.pitch, nv.stream()),
                 "softmax_backward")
        del dp
        p = Split(rows, L, dev, pitch=Lp, zero=Lp != L)
        ops.softmax_split(s, L, scale, p)
        del s

        def square_t(src: Split):
            t = Split(rows, L, dev, pitch=Lp, zero=Lp != L)
            nv.check(nv.lib().psam_transpose_split(src.ptr(), src.plane, src.pitch, L * Lp, H * L * Lp, t.ptr(), t.plane, t.pitch,
                                                   L * Lp, H * L * Lp, L, L, H, nb, nv.stream()), "transpose_split")
            return t

        into_dqkv(square(ds), heads_t(q, D), 0)                    # dQ = dS K
        into_dqkv(square(square_t(ds)), heads_t(q, 0), D)          # dK = dS^T Q
        del ds
        into_dqkv(square(square_t(p)), heads_t(dO, 0), 2 * D)      # dV = P^T dO
        del p


def block_backward(blk, pb, x: torch.Tensor, dy: torch.Tensor, B: int, L: int, need_x: bool = True):
    """Gradients of one EvaBlock (pre-LN attention + SwiGLU / GELU MLP, rope=None) at its input x [B*L, D] fp32 for the
    upstream gradient dy [B*L, D]: (dx or None, {parameter name: gradient}).  The forward is recomputed from x (unfused
    LayerNorms), keeping what one block needs; dx = None when need_x is false and norm1 is frozen."""
    D, H, dh = pb.D, pb.H, pb.dh
    M = B * L
    dev = x.device
    tr = _transposes(pb, blk)
    # ---- forward, recomputed
    xn = Split(M, D, dev)
    ops.layernorm(x, pb.g1, pb.b1, pb.eps1, out_split=xn)
    qkv = Split(M, 3 * D, dev)
    ops.gemm(xn, pb.wqkv, bias=pb.bqkv, out_split=qkv, passes=engine.PASSES)
    att = Split(M, D, dev)
    engine.attention(qkv, att, B, L, H, dh, D)
    x1 = x.clone()
    ops.gemm(att, pb.wproj, bias=pb.bproj, out_f32=x1, resid=x1, passes=engine.PASSES)
    xn2 = Split(M, D, dev)
    ops.layernorm(x1, pb.g2, pb.b2, pb.eps2, out_split=xn2)
    n1 = 2 * pb.hp if pb.swiglu else pb.hid
    a = torch.empty((M, n1), dtype=torch.float32, device=dev)
    ops.gemm(xn2, pb.w1, bias=pb.bb1, out_f32=a, passes=engine.PASSES)
    # ---- MLP
    g = {}
    dys = Split(M, D, dev)
    ops.split_f32(dy, dys)
    das = Split(M, n1, dev)
    mlp = blk.mlp
    if pb.swiglu:
        Hd, Hp = pb.hid, pb.hp
        dhn = torch.empty((M, Hp), dtype=torch.float32, device=dev)
        ops.gemm(dys, tr.w2, out_f32=dhn, passes=engine.PASSES)
        hn = Split(M, Hp, dev, pitch=Hp)
        da = torch.empty_like(a)
        nblk = (M + LN_ROWS_PER_BLOCK - 1) // LN_ROWS_PER_BLOCK
        part = torch.empty((nblk, 2, Hd), dtype=torch.float32, device=dev)
        nv.check(nv.lib().psam_swiglu_ln_backward(nv.ptr(a), n1, M, Hd, Hp, nv.ptr(dhn), Hp, nv.ptr(pb.gn), nv.ptr(pb.bn), float(pb.epsn),
                                                  nv.ptr(da), n1, das.ptr(), das.plane, das.pitch, hn.ptr(), hn.plane, hn.pitch, nv.ptr(part),
                                                  LN_ROWS_PER_BLOCK, nv.stream()), "swiglu_ln_backward")
        del dhn
        g["mlp.norm.weight"], g["mlp.norm.bias"] = _ln_params(part)
        g["mlp.fc2.weight"] = _weight_grad(dys, hn, M)[:, :Hd]
        del hn
        db1 = _col_sum(da)
        dw1 = _weight_grad(das, xn2, M)
        g["mlp.fc1_g.weight"], g["mlp.fc1_x.weight"] = dw1[0:2 * Hd:2], dw1[1:2 * Hd:2]
        g["mlp.fc1_g.bias"], g["mlp.fc1_x.bias"] = db1[0:2 * Hd:2], db1[1:2 * Hd:2]
    else:
        dh_ = torch.empty((M, n1), dtype=torch.float32, device=dev)
        ops.gemm(dys, tr.w2, out_f32=dh_, passes=engine.PASSES)
        h = Split(M, n1, dev)
        da = a  # the GELU backward reads a[i] before it writes da[i]
        nv.check(nv.lib().psam_gelu_backward(nv.ptr(a), n1, M, n1, nv.ptr(dh_), n1, nv.ptr(da), n1, das.ptr(), das.plane, das.pitch,
                                             h.ptr(), h.plane, h.pitch, nv.stream()), "gelu_backward")
        del dh_
        g["mlp.fc2.weight"] = _weight_grad(dys, h, M)
        del h
        g["mlp.fc1.bias"] = _col_sum(da)
        g["mlp.fc1.weight"] = _weight_grad(das, xn2, M)
    g["mlp.fc2.bias"] = _col_sum(dy)
    del da, a
    dxn2 = torch.empty((M, D), dtype=torch.float32, device=dev)
    ops.gemm(das, tr.w1, out_f32=dxn2, passes=engine.PASSES)
    del das
    dx1s = Split(M, D, dev)
    dx1, part2 = _ln_backward(x1, dxn2, pb.g2, pb.eps2, dres=dy, out_split=dx1s)
    del dxn2, x1
    g["norm2.weight"], g["norm2.bias"] = _ln_params(part2)
    # ---- attention
    g["attn.proj.weight"] = _weight_grad(dx1s, att, M)
    g["attn.proj.bias"] = _col_sum(dx1)
    datt = Split(M, D, dev)
    ops.gemm(dx1s, tr.wproj, out_split=datt, passes=engine.PASSES)
    del dx1s, att
    dqkv = torch.empty((M, 3 * D), dtype=torch.float32, device=dev)
    _attention_backward(qkv, datt, dqkv, B, L, H, dh, D)
    del qkv, datt
    dqkvs = Split(M, 3 * D, dev)
    ops.split_f32(dqkv, dqkvs)
    dwqkv, dbqkv = _weight_grad(dqkvs, xn, M), _col_sum(dqkv)
    del dqkv
    at = blk.attn
    if getattr(at, "qkv", None) is not None:
        g["attn.qkv.weight"], g["attn.q_bias"], g["attn.v_bias"] = dwqkv, dbqkv[:D], dbqkv[2 * D:]
    else:
        for i, n in enumerate(("q_proj", "k_proj", "v_proj")):
            g[f"attn.{n}.weight"], g[f"attn.{n}.bias"] = dwqkv[i * D:(i + 1) * D], dbqkv[i * D:(i + 1) * D]
    dx = None
    if need_x or blk.norm1.weight.requires_grad or blk.norm1.bias.requires_grad:
        dxn = torch.empty((M, D), dtype=torch.float32, device=dev)
        ops.gemm(dqkvs, tr.wqkv, out_f32=dxn, passes=engine.PASSES)
        dx, part1 = _ln_backward(x, dxn, pb.g1, pb.eps1, dres=dx1)
        g["norm1.weight"], g["norm1.bias"] = _ln_params(part1)
    return (dx if need_x else None), g


class EvaBlockFn(torch.autograd.Function):
    """One EvaBlock as an autograd node: the forward is the engine's inference block (un-folded LayerNorms) on a copy of
    x [B*L, D]; the inputs after the block's pack are its live parameters (named_parameters order), so their gradients land
    on the module.  Saves x only; the backward (block_backward) recomputes the rest."""

    @staticmethod
    def forward(ctx, x, blk, pb, B, L, *params):
        y = x.detach().clone()
        engine._run_block(pb, y, B, L, pb.D)
        ctx.save_for_backward(x)
        ctx.blk, ctx.pb, ctx.B, ctx.L = blk, pb, B, L
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, g = block_backward(ctx.blk, ctx.pb, x.detach(), dy.float().contiguous(), ctx.B, ctx.L, need_x=need[0])
        names = [n for n, _ in ctx.blk.named_parameters()]
        return (dx, None, None, None, None) + tuple(g[n].contiguous() if need[5 + i] else None for i, n in enumerate(names))


def encoder_trains(enc) -> bool:
    return any(p.requires_grad for p in enc.parameters())


def run_pc_encoder_train(enc, coords, features):
    """PointCloudEncoder.forward with autograd into the trainable parameters of the transformer blocks, the tail LayerNorms,
    out_proj, patch_proj and pos_embed: returns (pc_embeddings [B, L, E] with grad_fn, patches).  The tokenizer and the
    blocks below the lowest trainable one run through the engine without gradient; every block from there on is an
    EvaBlockFn; patch_proj / pos_embed (when trainable), the tail and out_proj are torch autograd on the per-token rows."""
    if hasattr(enc.patch_embed, "grouper1"):
        raise NotImplementedError("encoder fine-tuning covers the kNN tokenizer (PatchEmbed); PatchEmbedHier is not implemented")
    pk = engine._cached(enc, engine._PackedEncoder)
    tail = engine.validate_transformer(enc.transformer)
    blocks = list(enc.transformer.blocks)
    D = enc.transformer_dim
    with torch.no_grad():
        patches = engine.run_knn_grouper(enc.patch_embed.grouper, coords, features)
        emb, embs = engine.run_patch_encoder(enc.patch_embed.patch_encoder, patches["features"], want_split=True)
        patches["embeddings"] = emb
    B, L, _ = emb.shape
    M, dev = B * L, emb.device
    centers = patches["centers"]
    trains = lambda m: any(p.requires_grad for p in m.parameters())
    if trains(enc.patch_proj) or trains(enc.pos_embed):
        pe = enc.pos_embed
        x = _linear(enc.patch_proj, emb) + _linear(pe[2], F.gelu(_linear(pe[0], centers)))
        x = x.reshape(M, D)
        lo = 0
    else:
        with torch.no_grad():
            x = torch.empty((M, D), dtype=torch.float32, device=dev)
            ops.gemm(embs, pk.wpp, bias=pk.bpp, out_f32=x, passes=engine.PASSES)
            pos = Split(M, pk.wpos0.shape[0], dev)
            ops.small_in_linear(centers, pk.wpos0, pk.bpos0, None, None, 0.0, False, ops.ACT_GELU, pos)
            ops.gemm(pos, pk.wpos2, bias=pk.bpos2, out_f32=x, resid=x, passes=engine.PASSES)
        lo = next((i for i, b in enumerate(blocks) if trains(b)), len(blocks))
    with torch.no_grad():
        for pb in pk.blocks[:lo]:
            engine._run_block(pb, x, B, L, D)
    for blk, pb in zip(blocks[lo:], pk.blocks[lo:]):
        x = EvaBlockFn.apply(x, blk, pb, B, L, *blk.parameters())
    for m in tail:
        x = _ln(m, x)
    out = _linear(enc.out_proj, x).reshape(B, L, -1)
    return out, patches
