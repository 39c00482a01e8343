"""Automatic mask generation with crop layers on a set of clouds: two arms on the same seeded clouds, alternated in the same
run.
  (a) loop    generate_packed(..., crop_n_layers=1) on each cloud
  (b) batch   one generate_packed_batch_crops(..., crop_n_layers=1) on the list

Two workloads (--workload object / scene / both):
  object  8 clouds of 10000-30000 points (synth.make_batch), 256 prompts, points_per_batch 64
  scene   --scene-clouds "kitti" clouds of about 131072 points, 1024 prompts, points_per_batch 32

Model: eva02_large_patch14_448, 512 x 64 groups, random weights from a seed (no checkpoint offline), so the IoU and
stability filters are off, as in amg_bench.py.

Prints one JSON line: device name and power limit (read in the same run) and per workload: the sizes, per arm clouds/s
(median and range over --steps after --warmup, CUDA events around each call), the encode / decode / rest split of each
arm (CUDA events around every encoder and decoder call, summed; rest = post-processing, layout, gather and host work), the
padding fraction of (b)'s crop batches, and whether the two arms kept the same (prompt point, mask slot, crop box) triples
for each cloud.
usage: python tools/amg_crops_batch_bench.py [--workload both] [--steps 3] [--warmup 1] [--scene-clouds 2]"""
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

from pc_sam.automatic_mask_generator import PointCloudMaskGenerator  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402
from psam_b200 import synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", choices=["object", "scene", "both"], default="both")
ap.add_argument("--scene-clouds", type=int, default=2)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("amg_crops_batch_bench: needs a CUDA device")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


torch.manual_seed(1234)
model = build_point_sam("eva02_large_patch14_448", 512, 64).to(dev).eval()

# CUDA events around every encoder and decoder call (instance attributes shadow the methods; the generator calls them
# through self.model)
spans = {"encode": [], "decode": []}


def _wrap(name, key):
    fn = getattr(model, name)

    def run(*args, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*args, **kw)
        e1.record()
        spans[key].append((e0, e1))
        return out

    setattr(model, name, run)


_wrap("_encode", "encode")
_wrap("_decode_unchecked", "decode")


def workload(kind):
    rng = np.random.default_rng(a.seed)
    if kind == "object":
        sizes = sorted(int(n) for n in rng.integers(10000, 30001, 8))
        clouds = [synth.make_batch(1, n, a.seed + b) for b, n in enumerate(sizes)]
        prompts, ppb = 256, 64
    else:
        sizes = [131072 - 997 * b for b in range(a.scene_clouds)]
        clouds = [synth.make_batch(1, n, 3 + b, "kitti") for b, n in enumerate(sizes)]
        prompts, ppb = 1024, 32
    xyz = [x[0].to(dev) for x, _ in clouds]
    rgb = [r[0].to(dev) for _, r in clouds]
    gen = PointCloudMaskGenerator(model, points_per_cloud=prompts, points_per_batch=ppb, pred_iou_thresh=0.0,
                                  stability_score_thresh=0.0, stability_score_offset=0.05, mask_nms_thresh=0.7)
    last = {}

    def batch():
        st = gen._enqueue_batch_crops(xyz, rgb, crop_n_layers=1)
        last["st"] = st
        return gen._finish_batch_crops(st)

    arms = {"loop": lambda: [gen.generate_packed(x, r, crop_n_layers=1) for x, r in zip(xyz, rgb)], "batch": batch}

    def timed(fn):
        for v in spans.values():
            v.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        total = e0.elapsed_time(e1) / 1e3
        split = {k: sum(s.elapsed_time(e) for s, e in v) / 1e3 for k, v in spans.items()}
        split["rest"] = total - split["encode"] - split["decode"]
        return total, split, out

    with torch.no_grad():
        for _ in range(a.warmup):
            for fn in arms.values():
                fn()
        times, splits, outs = {k: [] for k in arms}, {k: [] for k in arms}, {}
        for _ in range(a.steps):
            for k, fn in arms.items():  # alternated: every step runs every arm once
                t, s, outs[k] = timed(fn)
                times[k].append(t)
                splits[k].append(s)

    def triples(o):
        return list(zip(o["point_index"].tolist(), o["mask_slot"].tolist(), map(tuple, o["crop_box"].tolist())))

    same = [triples(x) == triples(y) for x, y in zip(outs["loop"], outs["batch"])]
    real = sum(c for _, pairs, _ in last["st"]["crop_batches"] for _, _, c in pairs)
    padded = sum(len(pairs) * n for _, pairs, n in last["st"]["crop_batches"])

    def rate(ts):
        r = [len(sizes) / t for t in ts]
        return dict(median=round(float(np.median(r)), 3), min=round(min(r), 3), max=round(max(r), 3))

    res = {k: rate(v) for k, v in times.items()}
    split = {k: {p: round(float(np.median([s[p] for s in v])), 4) for p in ("encode", "decode", "rest")} for k, v in splits.items()}
    return dict(sizes=sizes, prompts=prompts, points_per_batch=ppb, crop_n_layers=1, clouds_per_s=res,
                batch_over_loop=round(res["batch"]["median"] / res["loop"]["median"], 3), seconds_split_median=split,
                crop_batches=[(lay, len(pairs), n) for lay, pairs, n in last["st"]["crop_batches"]],
                crop_padding_fraction=round(1 - real / padded, 3) if padded else 0.0,
                kept=[int(o["area"].shape[0]) for o in outs["batch"]], same_triples_per_cloud=same)


kinds = ["object", "scene"] if a.workload == "both" else [a.workload]
print(json.dumps(dict(device=gpu_info(), steps=a.steps, warmup=a.warmup, **{k: workload(k) for k in kinds})))
