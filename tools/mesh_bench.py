"""Mesh segmentation on synthetic meshes (four spheres and four boxes, psam_b200.synth.make_mesh) of about 200k and 2M faces:
S = 32768 surface samples, the c2 model (eva02_large_patch14_448, 512 x 64 groups, random weights), segment everything with
1024 prompts (points_per_batch 64, IoU / stability filters off).

Prints one JSON line: device name and power limit (read in the same run), and per mesh the ms of each stage by CUDA events
(median of --steps after --warmup, all in the same run): surface sampling (including its one statistics read), face centres,
nearest samples of the vertices and of the faces (the exact grid search psam_nn_grid_f32), lifting to vertices and faces plus the label
maps, and generate_packed on the sampled cloud; then the kernel times of each stage from a separate torch.profiler run.
usage: python tools/mesh_bench.py [--steps 5] [--warmup 1] [--faces 200000,2000000]"""
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
from pc_sam.mesh import MeshSegmenter, nearest_samples, sample_surface  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402
from psam_b200 import ops, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--faces", default="200000,2000000")
ap.add_argument("--points", type=int, default=32768)
ap.add_argument("--prompts", type=int, default=1024)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("mesh_bench: needs a CUDA device")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


def timed(fn):
    """ms of fn by CUDA events: median and range over a.steps calls after a.warmup."""
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {"ms": float(np.median(ms)), "range": [min(ms), max(ms)]}


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
    return dict(sorted(per.items(), key=lambda kv: -kv[1])[:8])


torch.manual_seed(1234)
model = build_point_sam("eva02_large_patch14_448", 512, 64).to(dev).eval()
gen = PointCloudMaskGenerator(model, points_per_cloud=a.prompts, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0)
S = a.points
line = {"workload": f"c2 512x64, eva02_large_patch14_448 (random weights), S={S}, points_per_cloud={a.prompts}, "
                    "points_per_batch=64, IoU / stability filters off",
        "device": gpu_info(), "meshes": []}
for target in (int(x) for x in a.faces.split(",")):
    v, f, col = synth.make_mesh(target, 0)
    seg = MeshSegmenter(model, num_points=S, seed=0)
    seg.set_mesh(v, f, vertex_colors=col)
    vn, fd, cd = seg.vertices, seg.faces, torch.from_numpy(col).to(dev)
    xyz = seg.xyz[0]
    out = gen.generate_packed(seg.xyz, seg.rgb)
    K = int(out["area"].shape[0])

    def lift_and_label():
        seg.lift_packed(out)

    stages = {
        "sample_surface": lambda: sample_surface(vn, fd, S, seed=0, vertex_colors=cd),
        "face_centers": lambda: ops.mesh_face_centers(vn, fd),
        "nearest_vertices": lambda: nearest_samples(xyz, vn),
        "nearest_faces": lambda: nearest_samples(xyz, seg.face_centers),
        "lift_and_labels": lift_and_label,
        "generate_packed": lambda: gen.generate_packed(seg.xyz, seg.rgb),
    }
    times = {k: timed(fn) for k, fn in stages.items()}
    total = sum(t["ms"] for t in times.values())
    kernels = {k: kernel_ms(fn) for k, fn in stages.items() if k != "generate_packed"}
    line["meshes"].append({
        "faces": int(len(f)), "vertices": int(len(v)), "kept_masks": K,
        "stage_ms": times, "total_ms": total,
        "share": {k: t["ms"] / total for k, t in times.items()},
        "kernel_ms": kernels,
    })
print(json.dumps(line))
