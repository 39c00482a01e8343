"""The evaluation loop (forward(is_eval=True): encode, then 5 rounds of ground-truth prompt sampling, prompt / mask
encoding, decode and best-mask feedback) on crops of different sizes, three arms on the same seeded crops, alternated in
the same run:
  (1) per-crop   forward_varlen on one crop at a time and one host copy of its IoU row (evaluate(batch_size=1))
  (2) varlen     forward_varlen on batches of up to --batch crops (plan_eval_batches: sorted by size, one group shape)
  (3) graph      the varlen graph predictor (make_iterative_predictor_varlen) captured once for --batch crops of at most
                 --max-points points, replayed for every batch of (2)

Model: eva02_large_patch14_448 with random weights from a seed (no checkpoint offline), 2048 groups of 256 points (what
the evaluation driver sets for crops of 2048 points or more), 5 prompt iterations.  Crops: synth "kitti" clouds with
N drawn log-uniform in [--min-points, --max-points] and synth.make_region_masks ground truth (one mask per crop).

Prints one JSON line: device name and power limit (read in the same run), crops/s per arm (median and range over --steps
after --warmup, CUDA events around each pass over all crops), the padding fraction 1 - sum N_b / sum (B * N_max) of (2)
and of (3), and for (2) and (3) how many crops' IoU rows equal those of (1) exactly - next to how many rows of (1) equal
its own rows of the first step (the encoder's float atomics let a logit within ~1e-5 of 0 change sign between runs).
--profile: instead, one pass of (1) and of (2) with CUDA events around every encode, decode and prompt-sampling call,
and the summed CUDA kernel time of the sampler's kernels under torch.profiler (a separate run: tracing slows the host).
usage: python tools/eval_varlen_bench.py [--crops 32] [--batch 8] [--min-points 2048] [--max-points 30000] [--steps 3]"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "point-sam_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from evaluation.eval_kitti import group_shape_for, plan_eval_batches  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402
from pc_sam.model.loss import compute_iou  # noqa: E402
from psam_b200 import synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--crops", type=int, default=32)
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--min-points", type=int, default=2048)
ap.add_argument("--max-points", type=int, default=30000)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--profile", action="store_true")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("eval_varlen_bench: needs a CUDA device")
if a.min_points < 2048:
    sys.exit("eval_varlen_bench: --min-points must be >= 2048 (one group shape, 2048 x 256, for every crop)")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


torch.manual_seed(1234)
model = build_point_sam("eva02_large_patch14_448", 2048, 256, prompt_iters=5).to(dev).eval()
rng = np.random.default_rng(a.seed)
sizes = [int(n) for n in np.exp(rng.uniform(np.log(a.min_points), np.log(a.max_points), a.crops))]
assert len({group_shape_for(n) for n in sizes}) == 1
crops = []
for i, n in enumerate(sizes):
    x, f = synth.make_batch(1, n, a.seed + i, "kitti")
    crops.append((x[0].to(dev), f[0].to(dev), synth.make_region_masks(x, 1)[0].to(dev)))
plan = plan_eval_batches(sizes, [0] * len(sizes), a.batch, 1 << 30)
pred = model.make_iterative_predictor_varlen(a.batch, 1, max(sizes))
pred.warmup(*zip(*[crops[i] for i in plan[0]]))


def rows_of(outs, idx):
    """IoU rows [len(idx), iterations] of forward_varlen's per-crop outputs, one host copy."""
    r = torch.stack([torch.stack([compute_iou(o["prompt_masks"], crops[i][2]) for o in out]) for out, i in zip(outs, idx)])
    return r.cpu().numpy().mean(axis=-1)


def per_crop():
    return np.concatenate([rows_of(model.forward_varlen(*[[t] for t in crops[i]]), [i]) for i in range(len(crops))])


def batched(run):
    rows = np.zeros((len(crops), model.prompt_iters), np.float32)
    for idx in plan:
        rows[idx] = rows_of(run(*zip(*[crops[i] for i in idx])), idx)
    return rows


arms = {"per_crop": per_crop, "varlen": lambda: batched(model.forward_varlen), "graph": lambda: batched(pred)}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, out


def profile():
    """Stage split: CUDA events around every encode, decode and sampling call (no synchronisation inside the pass)."""
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile

    stages = {"encode": [], "decode": [], "sample": []}
    originals = {"encode": model._encode, "decode": model._decode_unchecked, "sample": model._sample_prompts}

    def wrap(name):
        def fn(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = originals[name](*args, **kw)
            e1.record()
            stages[name].append((e0, e1))
            return out
        return fn

    res = {}
    for arm in ("per_crop", "varlen"):
        for k in stages:
            stages[k].clear()
        model._encode, model._decode_unchecked, model._sample_prompts = wrap("encode"), wrap("decode"), wrap("sample")
        try:
            t, _ = timed(arms[arm])
        finally:
            del model._encode, model._decode_unchecked, model._sample_prompts
        split = {k: round(sum(e0.elapsed_time(e1) for e0, e1 in v), 2) for k, v in stages.items()}
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            arms[arm]()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if e.device_time_total > 0]
        total = sum(e.device_time_total for e in kern) / 1e3
        sampler = sum(e.device_time_total for e in kern if "border_" in e.key) / 1e3
        res[arm] = dict(pass_ms=round(t * 1e3, 2), stage_ms=split, kernel_ms=round(total, 2), sampler_kernel_ms=round(sampler, 2))
    return res


with torch.no_grad():
    if a.profile:
        for fn in arms.values():
            fn()
        print(json.dumps(dict(device=gpu_info(), sizes=sizes, batches=[len(b) for b in plan], profile=profile())))
        sys.exit(0)
    for _ in range(a.warmup):
        for fn in arms.values():
            fn()
    times = {k: [] for k in arms}
    rows, first_rows = {}, None
    for _ in range(a.steps):
        for k, fn in arms.items():  # alternated: every step runs every arm once
            t, rows[k] = timed(fn)
            times[k].append(t)
        first_rows = rows["per_crop"] if first_rows is None else first_rows


def rate(ts):
    r = [a.crops / t for t in ts]
    return dict(median=round(float(np.median(r)), 2), min=round(min(r), 2), max=round(max(r), 2))


res = {k: rate(v) for k, v in times.items()}
pad = 1 - sum(sizes) / sum(len(b) * max(sizes[i] for i in b) for b in plan)
pad_graph = 1 - sum(sizes) / (len(plan) * a.batch * max(sizes))
print(json.dumps(dict(
    device=gpu_info(), crops=a.crops, sizes=sorted(sizes), batch=a.batch, batches=[len(b) for b in plan], steps=a.steps,
    warmup=a.warmup, crops_per_s=res, varlen_over_per_crop=round(res["varlen"]["median"] / res["per_crop"]["median"], 3),
    graph_over_per_crop=round(res["graph"]["median"] / res["per_crop"]["median"], 3),
    padding_fraction=round(pad, 3), graph_padding_fraction=round(pad_graph, 3),
    equal_rows=dict(varlen=int(sum(np.array_equal(u, v) for u, v in zip(rows["varlen"], rows["per_crop"]))),
                    graph=int(sum(np.array_equal(u, v) for u, v in zip(rows["graph"], rows["per_crop"]))),
                    # the per-crop arm against itself: its first and last pass (the encoder's float atomics)
                    per_crop_rerun=int(sum(np.array_equal(u, v) for u, v in zip(first_rows, rows["per_crop"])))),
    mean_iou_per_crop_loop=[round(float(v), 4) for v in rows["per_crop"].mean(axis=0)])))
