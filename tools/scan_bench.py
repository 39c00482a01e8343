"""Dense-scan segmentation on synthetic LiDAR-like scans (psam_b200.synth.make_scan) of 10^6, 10^7 and 5 x 10^7 points:
S = 32768 voxel samples, the c2 model (eva02_large_patch14_448, 512 x 64 groups, random weights), segment everything with
1024 prompts (points_per_batch 64, IoU / stability filters off).

Prints one JSON line: device name and power limit (read in the same run), and per scan the ms of each stage by CUDA events
(median of --steps after --warmup): normalisation + voxel subsample (set_scan without the encode and the nearest search),
generate_packed on the samples, the grid nearest search of every scan point, lifting + labels; then, at 10^6 and 10^7
points, the brute-force nearest search (psam_nn_distance_f32) alternated with the grid search call by call in the same run;
then the kernel times of each stage from a separate torch.profiler run.
usage: python tools/scan_bench.py [--steps 5] [--warmup 1] [--points 1000000,10000000,50000000]"""
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
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from pc_sam.automatic_mask_generator import PointCloudMaskGenerator  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402
from pc_sam.scan import ScanSegmenter  # noqa: E402
from psam_b200 import native as nv  # noqa: E402
from psam_b200 import ops, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--points", default="1000000,10000000,50000000")
ap.add_argument("--samples", type=int, default=32768)
ap.add_argument("--prompts", type=int, default=1024)
ap.add_argument("--brute-max", type=int, default=10000000, help="largest scan on which the brute-force search is timed")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("scan_bench: needs a CUDA device")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


def one(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def timed(fn, steps=None):
    """ms of fn by CUDA events: median and range over a.steps calls after a.warmup."""
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    ms = [one(fn) for _ in range(steps or a.steps)]
    return {"ms": float(np.median(ms)), "range": [min(ms), max(ms)]}


def alternated(fa, fb, steps):
    """The two functions called in turn, each timed by CUDA events: (median ms of a, median ms of b)."""
    fa(), fb()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(steps):
        ta.append(one(fa))
        tb.append(one(fb))
    return float(np.median(ta)), float(np.median(tb))


def kernel_ms(fn, reps=3):
    """Device time per call of every kernel fn launches (torch.profiler, fn alone)."""
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for evt in prof.events():
        if evt.device_type == torch.autograd.DeviceType.CUDA and "Memset" not in evt.name and "Memcpy" not in evt.name:
            name = evt.name.replace("(anonymous namespace)::", "").split("(")[0].split("::")[-1].split()[-1]
            per[name] = per.get(name, 0.0) + (getattr(evt, "device_time", None) or evt.cuda_time) / 1e3 / reps
    return dict(sorted(per.items(), key=lambda kv: -kv[1])[:10])


def brute(query, key):
    d = torch.empty(query.shape[0], dtype=torch.float32, device=dev)
    i = torch.empty(query.shape[0], dtype=torch.int64, device=dev)
    nv.check(nv.lib().psam_nn_distance_f32(nv.ptr(query), nv.ptr(key), query.shape[0], key.shape[0], nv.ptr(d), nv.ptr(i), nv.stream()),
             "nn_distance")
    return d, i


torch.manual_seed(1234)
model = build_point_sam("eva02_large_patch14_448", 512, 64).to(dev).eval()
gen = PointCloudMaskGenerator(model, points_per_cloud=a.prompts, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0)
line = {"workload": f"c2 512x64, eva02_large_patch14_448 (random weights), S={a.samples}, points_per_cloud={a.prompts}, "
                    "points_per_batch=64, IoU / stability filters off, synth.make_scan",
        "device": gpu_info(), "scans": []}
for P in (int(x) for x in a.points.split(",")):
    xyz_np, rgb_np = synth.make_scan(P, 0)
    xyz, rgb = torch.from_numpy(xyz_np).to(dev), torch.from_numpy(rgb_np).to(dev)
    del xyz_np, rgb_np
    seg = ScanSegmenter(model, num_points=a.samples, seed=0)
    seg.set_scan(xyz, rgb)
    out = gen.generate_packed(seg.xyz, seg.rgb)
    K = int(out["area"].shape[0])
    pts, samples = seg.points, seg.xyz[0]

    def normalise_and_subsample():
        x64 = xyz.double()
        valid = torch.isfinite(xyz).all(dim=1)
        shift = torch.where(valid[:, None], x64, 0.0).sum(0) / valid.sum()
        scale = torch.where(valid, (x64 - shift).norm(dim=1), 0.0).max()
        xn = torch.where(valid[:, None], (x64 - shift) / scale, float("nan")).float()
        ops.voxel_subsample(xn, a.samples, 0)

    stages = {
        "normalise_and_subsample": normalise_and_subsample,
        "generate_packed": lambda: gen.generate_packed(seg.xyz, seg.rgb),
        "nearest_grid": lambda: ops.nearest_grid(pts, samples),
        "lift_and_labels": lambda: seg.lift_packed(out),
    }
    times = {k: timed(fn) for k, fn in stages.items()}
    total = sum(t["ms"] for t in times.values())
    rec = {"points": P, "valid": int(seg.stats[0]), "level": int(seg.stats[1]), "samples": int(seg.xyz.shape[1]), "kept_masks": K,
           "stage_ms": times, "total_ms": total, "share": {k: t["ms"] / total for k, t in times.items()}}
    if P <= a.brute_max:
        g_ms, b_ms = alternated(lambda: ops.nearest_grid(pts, samples), lambda: brute(pts, samples), max(3, a.steps))
        same = torch.equal(ops.nearest_grid(pts, samples)[1], brute(pts, samples)[1])
        rec["nearest"] = {"grid_ms": g_ms, "brute_ms": b_ms, "speedup": b_ms / g_ms, "identical": bool(same)}
    rec["kernel_ms"] = {k: kernel_ms(fn) for k, fn in stages.items() if k != "generate_packed"}
    line["scans"].append(rec)
    del seg, out, xyz, rgb, pts, samples
    torch.cuda.empty_cache()
print(json.dumps(line))
