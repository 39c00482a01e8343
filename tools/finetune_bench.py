"""Fine-tuning step benchmark: PointCloudSAM (ViT-L encoder by default) in training mode, Criterion, backward and an AdamW
step, on one fixed synthetic batch.

--train-blocks K (several values allowed): K = 0 trains mask_decoder only, with two arms alternated step by step in the same
process:
  cuda  - the shipped path: the per-point head (psam_b200.train.MaskHead) and the mask loss (psam_b200.train.mask_loss) in CUDA;
  torch - the same step with the head and the loss as plain torch autograd (restated below), everything else unchanged.
K > 0 also trains the last K encoder blocks, fc_norm and out_proj (the README's example), with the arms
  cuda  - the shipped path: each trainable block is psam_b200.train.EvaBlockFn (CUDA backward, recomputed from its input);
  torch - the blocks as fp32 torch autograd (TorchBlock below); head and loss in CUDA in both arms.
Reported per arm: steps/s, the split of a step from CUDA events (encoder forward, encoder backward from the gradient's arrival
at the encoder output to the end of backward, weight repacking, trunk, head, loss, optimizer) and the peak allocated memory.
The card and its power limit are printed with the numbers.

    python tools/finetune_bench.py --points 10000 32768 --train-blocks 0 2 8 24 --steps 5 --warmup 2
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "point-sam_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


# ------------------------------------------------------------------------------------------------
# the torch arm: the head and the loss as plain autograd
# ------------------------------------------------------------------------------------------------
class TorchHead:
    @staticmethod
    def apply(f0, hyper, gamma, beta, w3, b3, geo):
        Z, C, D = hyper.shape
        idx = geo.idx.repeat_interleave(geo.rep, 0)  # [Z, N, 3]
        w = geo.w.repeat_interleave(geo.rep, 0)
        f = f0.view(Z, geo.G, D)
        g = torch.gather(f, 1, idx.reshape(Z, -1, 1).expand(-1, -1, D)).view(Z, geo.N, 3, D)
        v = (g * w.unsqueeze(-1)).sum(-2)
        u1 = F.gelu(F.layer_norm(v, (D,), gamma, beta, geo.eps))
        u2 = F.gelu(F.linear(u1, w3, b3))
        return hyper @ u2.transpose(-1, -2)


def torch_mask_loss(logits, gt):
    t = gt.unsqueeze(1).expand_as(logits).float()
    p = logits.sigmoid()
    ce = F.binary_cross_entropy_with_logits(logits, t, reduction="none")
    p_t = p * t + (1 - p) * (1 - t)
    focal = ce * (1 - p_t) ** 2
    pt, pp, ts = (p * t).sum(-1), p.square().sum(-1), t.sum(-1)
    loss = focal.mean(-1) + 2 * (1 - (2 * pt + 1e-3) / (pp + ts + 1e-3))
    pred = logits.detach() > 0
    counts = torch.stack([(pred & gt.unsqueeze(1)).sum(-1), (pred | gt.unsqueeze(1)).sum(-1)], -1).int()
    stats = torch.stack([focal.sum(-1), pt, pp, ts], -1).detach()
    return loss, stats, counts


class TorchBlock:
    """timm EvaBlock (pre-LN attention, SwiGLU with inner LayerNorm or GELU Mlp) in fp32 torch autograd."""

    @staticmethod
    def apply(x, blk, pb, B, L, *params):
        D = x.shape[1]
        at, m = blk.attn, blk.mlp
        H = at.num_heads
        xn = F.layer_norm(x, (D,), blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
        if at.qkv is not None:
            qkv = F.linear(xn, at.qkv.weight, torch.cat([at.q_bias, at.k_bias, at.v_bias]))
        else:
            qkv = torch.cat([F.linear(xn, l.weight, l.bias) for l in (at.q_proj, at.k_proj, at.v_proj)], -1)
        q, k, v = qkv.view(B, L, 3, H, D // H).permute(2, 0, 3, 1, 4)
        a = torch.softmax((q * (D // H) ** -0.5) @ k.transpose(-1, -2), -1) @ v
        x = x + F.linear(a.transpose(1, 2).reshape(B * L, D), at.proj.weight, at.proj.bias)
        h = F.layer_norm(x, (D,), blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
        if hasattr(m, "fc1_g"):
            h = F.silu(F.linear(h, m.fc1_g.weight, m.fc1_g.bias)) * F.linear(h, m.fc1_x.weight, m.fc1_x.bias)
            h = F.layer_norm(h, (h.shape[1],), m.norm.weight, m.norm.bias, m.norm.eps)
        else:
            h = F.gelu(F.linear(h, m.fc1.weight, m.fc1.bias))
        return x + F.linear(h, m.fc2.weight, m.fc2.bias)


# ------------------------------------------------------------------------------------------------
# event timing of the phases
# ------------------------------------------------------------------------------------------------
class Phases:
    def __init__(self):
        self.marks = {}

    @contextlib.contextmanager
    def time(self, name):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        try:
            yield
        finally:
            b.record()
            self.marks.setdefault(name, []).append((a, b))

    def wrap(self, obj, attr, name):
        fn = getattr(obj, attr)
        ph = self

        def timed(*a, **k):
            with ph.time(name):
                return fn(*a, **k)

        setattr(obj, attr, timed)
        return fn

    def totals(self):
        torch.cuda.synchronize()
        out = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.marks.items()}
        self.marks = {}
        return out


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        power = q.stdout.strip()
    except Exception as e:  # the query is informational
        power = f"unknown ({type(e).__name__})"
    return name, power


def batch(B, M, N, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    rgb = torch.rand(B, N, 3, generator=g)
    gt = torch.zeros(B, M, N, dtype=torch.bool)
    for b in range(B):
        for m in range(M):
            c = xyz[b, torch.randint(0, N, (1,), generator=g)]
            gt[b, m] = (xyz[b] - c).norm(dim=-1) < 0.3 + 0.5 * torch.rand(1, generator=g)
    return xyz.to(dev), rgb.to(dev), gt.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoder", default="eva02_large_patch14_448")
    ap.add_argument("--points", type=int, nargs="+", default=[10000, 32768])
    ap.add_argument("--clouds", type=int, default=2)
    ap.add_argument("--masks", type=int, default=8)
    ap.add_argument("--prompt-iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--train-blocks", type=int, nargs="+", default=[0])
    args = ap.parse_args()

    from pc_sam.model import build_point_sam
    from pc_sam.model import loss as loss_mod
    from pc_sam.model import pc_sam as pc_sam_mod
    from psam_b200 import engine, train

    dev = torch.device("cuda:0")
    name, power = card()
    print(json.dumps(dict(card=name, power_limit=power, encoder=args.encoder, clouds=args.clouds, masks=args.masks,
                          prompt_iters=args.prompt_iters)), flush=True)
    torch.manual_seed(0)
    model = build_point_sam(args.encoder, prompt_iters=args.prompt_iters).to(dev)
    model.train()
    crit = loss_mod.Criterion()

    ph = Phases()
    ph.wrap(pc_sam_mod.PointCloudSAM, "_encode", "encoder")
    enc_train = train.run_pc_encoder_train

    def timed_enc_train(*a):
        with ph.time("encoder"):
            out, patches = enc_train(*a)
        start = torch.cuda.Event(enable_timing=True)

        def arrived(g):
            start.record()
            ph.bwd_start = start
        out.register_hook(arrived)
        return out, patches

    train.run_pc_encoder_train = timed_enc_train
    depth = [0]
    cached = engine._cached

    def timed_cached(*a, **k):  # weight packing, outermost call only (the encoder pack holds the per-block packs)
        depth[0] += 1
        try:
            if depth[0] > 1:
                return cached(*a, **k)
            with ph.time("repack"):
                return cached(*a, **k)
        finally:
            depth[0] -= 1

    engine._cached = timed_cached
    transposes = ph.wrap(train, "_transposes", "repack_transposed")  # noqa: F841
    ph.wrap(train, "decoder_trunk", "trunk_fwd")
    cuda_head = train.MaskHead
    cuda_loss = train.mask_loss
    hb = ph.wrap(train, "head_backward", "head_bwd")  # noqa: F841  (the CUDA arm's head backward)

    class TimedHead:
        impl = cuda_head

        @staticmethod
        def apply(*a):
            with ph.time("head_fwd"):
                return TimedHead.impl.apply(*a)

    def timed_loss(impl):
        def f(logits, gt):
            with ph.time("loss_fwd"):
                return impl(logits, gt)
        return f

    train.MaskHead = TimedHead
    cuda_block = train.EvaBlockFn
    for N, K in [(n, k) for k in args.train_blocks for n in args.points]:
        model.requires_grad_(False)
        model.mask_decoder.requires_grad_(True)
        if K:
            tr = model.pc_encoder.transformer
            tr.blocks[-K:].requires_grad_(True)
            tr.fc_norm.requires_grad_(True)
            model.pc_encoder.out_proj.requires_grad_(True)
        opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=3e-4, weight_decay=0.1)
        xyz, rgb, gt = batch(args.clouds, args.masks, N, dev)
        if K:
            arms = {"cuda": (cuda_head, cuda_loss, cuda_block), "torch": (cuda_head, cuda_loss, TorchBlock)}
        else:
            arms = {"cuda": (cuda_head, cuda_loss, cuda_block), "torch": (TorchHead, torch_mask_loss, cuda_block)}
        res = {k: dict(times=[], phases=[], peak=0) for k in arms}
        for step in range(args.warmup + args.steps):
            for arm, (head, lossf, block) in arms.items():
                TimedHead.impl = head
                train.mask_loss = timed_loss(lossf)
                train.EvaBlockFn = block
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                ph.totals()
                ph.bwd_start = None
                t0 = time.perf_counter()
                outputs = model(xyz, rgb, gt)
                loss, aux = crit(outputs, gt.flatten(0, 1))
                with ph.time("backward"):
                    loss.backward()
                if ph.bwd_start is not None:
                    end = torch.cuda.Event(enable_timing=True)
                    end.record()
                    ph.marks.setdefault("encoder_bwd", []).append((ph.bwd_start, end))
                with ph.time("optimizer"):
                    opt.step()
                    opt.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                tot = ph.totals()
                if step >= args.warmup:
                    res[arm]["times"].append(dt)
                    res[arm]["phases"].append(tot)
                    res[arm]["peak"] = max(res[arm]["peak"], torch.cuda.max_memory_allocated())
                del outputs, loss, aux
        for arm, r in res.items():
            keys = sorted({k for p in r["phases"] for k in p})
            mean = {k: round(sum(p.get(k, 0.0) for p in r["phases"]) / len(r["phases"]), 3) for k in keys}
            # the CUDA arm times its head backward directly; trunk and loss backward are the rest of loss.backward()
            mean["trunk_and_loss_bwd"] = round(mean.get("backward", 0.0) - mean.get("head_bwd", 0.0), 3)
            ts = sorted(r["times"])
            print(json.dumps(dict(arm=arm, N=N, train_blocks=K, steps_per_s=round(1.0 / ts[len(ts) // 2], 3), step_ms_median=round(1e3 * ts[len(ts) // 2], 2),
                                  phases_ms=mean, peak_allocated_gb=round(r["peak"] / 2 ** 30, 2), card=name, power_limit=power)),
                  flush=True)
    train.MaskHead, train.mask_loss, train.EvaBlockFn = cuda_head, cuda_loss, cuda_block
    train.run_pc_encoder_train, engine._cached = enc_train, cached


if __name__ == "__main__":
    main()
