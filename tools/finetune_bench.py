"""Fine-tuning step benchmark: PointCloudSAM (ViT-L encoder by default) in training mode with only mask_decoder learning,
Criterion, backward and an AdamW step, on one fixed synthetic batch.

Two arms, alternated step by step in the same process:
  cuda  - the shipped path: the per-point head (psam_b200.train.MaskHead) and the mask loss (psam_b200.train.mask_loss) in CUDA;
  torch - the same step with the head and the loss as plain torch autograd (restated below), everything else unchanged.
Reported per arm: steps/s, the split of a step between encoder, trunk forward / backward, head forward / backward, loss
(forward + backward) and optimizer from CUDA events, and the peak allocated memory.  The card and its power limit are printed
with the numbers.

    python tools/finetune_bench.py --points 10000 32768 --steps 5 --warmup 2
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
    args = ap.parse_args()

    from pc_sam.model import build_point_sam
    from pc_sam.model import loss as loss_mod
    from pc_sam.model import pc_sam as pc_sam_mod
    from psam_b200 import train

    dev = torch.device("cuda:0")
    name, power = card()
    print(json.dumps(dict(card=name, power_limit=power, encoder=args.encoder, clouds=args.clouds, masks=args.masks,
                          prompt_iters=args.prompt_iters)), flush=True)
    torch.manual_seed(0)
    model = build_point_sam(args.encoder, prompt_iters=args.prompt_iters).to(dev)
    model.requires_grad_(False)
    model.mask_decoder.requires_grad_(True)
    model.train()
    crit = loss_mod.Criterion()
    opt = torch.optim.AdamW(model.mask_decoder.parameters(), lr=3e-4, weight_decay=0.1)

    ph = Phases()
    ph.wrap(pc_sam_mod.PointCloudSAM, "_encode", "encoder")
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
    for N in args.points:
        xyz, rgb, gt = batch(args.clouds, args.masks, N, dev)
        arms = {"cuda": (cuda_head, cuda_loss), "torch": (TorchHead, torch_mask_loss)}
        res = {k: dict(times=[], phases=[], peak=0) for k in arms}
        for step in range(args.warmup + args.steps):
            for arm, (head, lossf) in arms.items():
                TimedHead.impl = head
                train.mask_loss = timed_loss(lossf)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                ph.totals()
                t0 = time.perf_counter()
                outputs = model(xyz, rgb, gt)
                loss, aux = crit(outputs, gt.flatten(0, 1))
                with ph.time("backward"):
                    loss.backward()
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
            print(json.dumps(dict(arm=arm, N=N, steps_per_s=round(1.0 / ts[len(ts) // 2], 3), step_ms_median=round(1e3 * ts[len(ts) // 2], 2),
                                  phases_ms=mean, peak_allocated_gb=round(r["peak"] / 2 ** 30, 2), card=name, power_limit=power)),
                  flush=True)
    train.MaskHead, train.mask_loss = cuda_head, cuda_loss


if __name__ == "__main__":
    main()
