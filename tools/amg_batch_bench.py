"""Automatic mask generation on a batch of clouds: PointCloudMaskGenerator.generate_packed_batch on B clouds against B
sequential generate_packed calls on the same clouds, the two arms alternated in the same run.

Workloads (c2 model: eva02_large_patch14_448, 512 x 64 groups; points_per_batch = 64):
  dataset  N = 10000 (Point-SAM's training configs sample 10000 points per object), B = 8, points_per_cloud 1024 and 256
  large    N = 32768, B = 4, points_per_cloud 1024 (expected to be decode-bound)

Prints one JSON line: device name and power limit (read in the same run), and per workload clouds/s of each arm (median and
range over --steps after --warmup), their ratio, kept masks per cloud, the encode / decode / post-processing split of one
call of each arm by CUDA events (post-processing = everything else: FPS, candidates, NMS, small regions, the final read), and
the time and launch count of each post-processing kernel in one batched call against the B per-cloud calls (torch.profiler,
separate run, with min_mask_region_area = --profile-region-area so that the small-region kernels are included).
The weights are random (no checkpoint is available offline), so the IoU and stability filters are off, as in amg_bench.py.
usage: python tools/amg_batch_bench.py [--steps 5] [--warmup 1] [--profile-region-area 64] [--only dataset|large]"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "point-sam_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pc_sam.automatic_mask_generator import PointCloudMaskGenerator  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402
from psam_b200 import synth  # noqa: E402

POST_KERNELS = ("mask_candidates_kernel", "nms_order_kernel", "nms_pairs_kernel", "nms_scan_kernel", "knn_kernel",
                "mask_regions_kernel")
WORKLOADS = [("dataset", 10000, 8, 1024), ("dataset", 10000, 8, 256), ("large", 32768, 4, 1024)]

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--profile-region-area", type=int, default=64)
ap.add_argument("--only", choices=["dataset", "large"])
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("amg_batch_bench: needs a CUDA device")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


torch.manual_seed(1234)
model = build_point_sam("eva02_large_patch14_448", 512, 64).to(dev).eval()


def batched(gen, xyz, rgb, area=0):
    return gen.generate_packed_batch(xyz, rgb, min_mask_region_area=area)


def sequential(gen, xyz, rgb, area=0):
    return [gen.generate_packed(xyz[b], rgb[b], min_mask_region_area=area) for b in range(xyz.shape[0])]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def split(fn):
    """encode / decode / post-processing ms of one call, by CUDA events around the model's encode and decode calls."""
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    spans = {"encode": [], "decode": []}
    enc_fn, dec_fn = model._encode, model._decode_unchecked

    def wrap(name, f):
        def g(*args):
            e0, e1 = ev(), ev()
            e0.record()
            out = f(*args)
            e1.record()
            spans[name].append((e0, e1))
            return out
        return g

    model._encode, model._decode_unchecked = wrap("encode", enc_fn), wrap("decode", dec_fn)
    try:
        t0, t1 = ev(), ev()
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
    finally:
        del model._encode, model._decode_unchecked
    t = {k: sum(x.elapsed_time(y) for x, y in v) for k, v in spans.items()}
    t["total"] = t0.elapsed_time(t1)
    t["post"] = t["total"] - t["encode"] - t["decode"]
    return t


def kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for evt in prof.events():
        if evt.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for tag in POST_KERNELS:
            if tag in evt.name:
                d = kern.setdefault(tag, [0.0, 0])
                d[0] += (getattr(evt, "device_time", None) or evt.cuda_time) / 1e3  # us -> ms
                d[1] += 1
    return kern


results = []
for name, N, B, P in WORKLOADS:
    if a.only and name != a.only:
        continue
    gen = PointCloudMaskGenerator(model, points_per_cloud=P, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    xyz, rgb = (t.to(dev) for t in synth.make_batch(B, N, 11))
    for _ in range(a.warmup):
        batched(gen, xyz, rgb)
        sequential(gen, xyz, rgb)
    tb, ts = [], []
    for _ in range(a.steps):  # alternated, so both arms see the same clocks and neighbours
        dt, out_b = timed(lambda: batched(gen, xyz, rgb))
        tb.append(B / dt)
        dt, out_s = timed(lambda: sequential(gen, xyz, rgb))
        ts.append(B / dt)
    sp = {"batched": split(lambda: batched(gen, xyz, rgb)), "sequential": split(lambda: sequential(gen, xyz, rgb))}
    A = a.profile_region_area
    kb, ks = kernels(lambda: batched(gen, xyz, rgb, A)), kernels(lambda: sequential(gen, xyz, rgb, A))
    kern = {k: {"batched_ms": kb.get(k, [0.0, 0])[0], "batched_launches": kb.get(k, [0.0, 0])[1],
                "per_cloud_calls_ms": ks.get(k, [0.0, 0])[0], "per_cloud_calls_launches": ks.get(k, [0.0, 0])[1]}
            for k in POST_KERNELS}
    results.append({
        "workload": name, "points": N, "clouds": B, "points_per_cloud": P, "points_per_batch": 64,
        "batched_clouds_per_s": float(np.median(tb)), "batched_clouds_per_s_range": [min(tb), max(tb)],
        "sequential_clouds_per_s": float(np.median(ts)), "sequential_clouds_per_s_range": [min(ts), max(ts)],
        "speedup": float(np.median(tb) / np.median(ts)),
        "kept_per_cloud_batched": [int(o["area"].shape[0]) for o in out_b],
        "kept_per_cloud_sequential": [int(o["area"].shape[0]) for o in out_s],
        "split_ms_per_call": sp, "post_kernels_ms_per_call": kern, "profile_min_mask_region_area": A,
    })
    del gen
    torch.cuda.empty_cache()

print(json.dumps({"tool": "amg_batch_bench", "device": gpu_info(), "steps": a.steps, "warmup": a.warmup,
                  "model": "c2 (eva02_large_patch14_448, 512 x 64), random weights, IoU / stability filters off",
                  "workloads": results}))
