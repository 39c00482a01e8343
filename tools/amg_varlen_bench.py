"""Automatic mask generation on clouds of different sizes: three arms on the same seeded mix of clouds, alternated in the
same run.
  (a) loop      generate_packed on each cloud
  (b) varlen    one generate_packed_batch on the list (a padded batch: clouds padded to the largest, lengths on the device)
  (c) cut       one generate_packed_batch on the [B, N_min, 3] batch of every cloud cut to the smallest N (the best uniform
                batch available without padding; it segments fewer points, so it is a reference, not a competitor)

Model: eva02_large_patch14_448, 512 x 64 groups, random weights from a seed (no checkpoint offline), so the IoU and
stability filters are off, as in amg_bench.py.  Clouds: synth.make_batch per cloud with N drawn from [--n-lo, --n-hi].

Prints one JSON line: device name and power limit (read in the same run), the sizes, per arm clouds/s (median and range over
--steps after --warmup, CUDA events around each call) and the ratio (b)/(a), and whether (a) and (b) kept the same masks for
every cloud (the same (prompt point, mask slot) pairs, and the fraction of equal mask bits).
usage: python tools/amg_varlen_bench.py [--clouds 8] [--n-lo 6000] [--n-hi 14000] [--prompts 256] [--steps 5] [--warmup 1]"""
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
ap.add_argument("--clouds", type=int, default=8)
ap.add_argument("--n-lo", type=int, default=6000)
ap.add_argument("--n-hi", type=int, default=14000)
ap.add_argument("--prompts", type=int, default=256)
ap.add_argument("--points-per-batch", type=int, default=64)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("amg_varlen_bench: needs a CUDA device")
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
rng = np.random.default_rng(a.seed)
sizes = sorted(int(n) for n in rng.integers(a.n_lo, a.n_hi + 1, a.clouds))
clouds = [synth.make_batch(1, n, a.seed + b) for b, n in enumerate(sizes)]
xyz = [x[0].to(dev) for x, _ in clouds]
rgb = [r[0].to(dev) for _, r in clouds]
n_min = sizes[0]
xyz_cut = torch.stack([x[:n_min] for x in xyz])
rgb_cut = torch.stack([r[:n_min] for r in rgb])
gen = PointCloudMaskGenerator(model, points_per_cloud=a.prompts, points_per_batch=a.points_per_batch, pred_iou_thresh=0.0,
                              stability_score_thresh=0.0, stability_score_offset=0.05, mask_nms_thresh=0.7)
arms = {
    "loop": lambda: [gen.generate_packed(x, r) for x, r in zip(xyz, rgb)],
    "varlen": lambda: gen.generate_packed_batch(xyz, rgb),
    "cut": lambda: gen.generate_packed_batch(xyz_cut, rgb_cut),
}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, out


with torch.no_grad():
    for _ in range(a.warmup):
        for fn in arms.values():
            fn()
    times = {k: [] for k in arms}
    outs = {}
    for _ in range(a.steps):
        for k, fn in arms.items():  # alternated: every step runs every arm once
            t, outs[k] = timed(fn)
            times[k].append(t)

same_pairs, bit_agree = [], []
for one, bat in zip(outs["loop"], outs["varlen"]):
    pa = list(zip(one["point_index"].tolist(), one["mask_slot"].tolist()))
    pb = list(zip(bat["point_index"].tolist(), bat["mask_slot"].tolist()))
    same_pairs.append(pa == pb)
    if pa == pb and len(pa):
        bit_agree.append(float((one["bits"] == bat["bits"]).float().mean()))


def rate(ts):
    r = [a.clouds / t for t in ts]
    return dict(median=round(float(np.median(r)), 2), min=round(min(r), 2), max=round(max(r), 2))


res = {k: rate(v) for k, v in times.items()}
print(json.dumps(dict(
    device=gpu_info(), sizes=sizes, prompts=a.prompts, points_per_batch=a.points_per_batch, steps=a.steps, warmup=a.warmup,
    clouds_per_s=res, varlen_over_loop=round(res["varlen"]["median"] / res["loop"]["median"], 3),
    padding_fraction=round(1 - sum(sizes) / (len(sizes) * sizes[-1]), 3),
    kept=[int(o["area"].shape[0]) for o in outs["varlen"]], same_masks_per_cloud=same_pairs,
    mask_word_agreement=[round(x, 6) for x in bit_agree])))
