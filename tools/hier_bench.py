"""Throughput of the hierarchical model (configs/model/hier.yaml: PointCloudSAMHier, tokenizer 2048 x 32 then 512 x 32, ViT-L)
served like bench.py's headline workload: independent single-cloud requests, N = 32768, 1 point prompt, `--depth` clouds in
flight (PipelinedPredictor), inputs in HBM; plus the single-cloud latency of one CUDA-graph predictor.  `--with-c2` times the
base model of bench.py's c2 workload (512 x 64 groups) the same way in the same process, for a same-session ratio.
usage: python tools/hier_bench.py [--steps 20] [--warmup 3] [--depth 8] [--with-c2] [--dump-outputs DIR]"""
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

from pc_sam.model import build_point_sam, build_point_sam_hier  # noqa: E402
from psam_b200 import synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--depth", type=int, default=8)
ap.add_argument("--points", type=int, default=32768)
ap.add_argument("--with-c2", action="store_true")
ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="mask logits / IoU of the last request (float32 .npy)")
a = ap.parse_args()
dev = torch.device("cuda:0")
N, cps = a.points, 2 * a.depth  # requests per step: two rounds of the lanes
clouds = [synth.make_batch(1, N, 17 * i, "ball") for i in range(4)]
inputs = [tuple(t.to(dev) for t in (*c, *synth.make_prompts(c[0], 1, i))) for i, c in enumerate(clouds)]


def timed(fn, steps, sync):
    """ms for `steps` calls of fn; the predictors run on their own streams, so the clock stops after `sync` has waited for them."""
    sync()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
    sync()
    return (time.perf_counter() - t0) * 1e3


def run(model):
    pp = model.make_pipelined_predictor(1, N, 1, depth=a.depth)
    pp.warmup(*inputs[0])

    def step(i):
        for c in range(cps):
            pp.submit(*inputs[(i * cps + c) % len(inputs)])

    timed(step, a.warmup, pp.synchronize)
    ms = timed(step, a.steps, pp.synchronize)
    m, iou = pp.result(pp.count - 1)
    # single-cloud latency: one graph predictor, each request waited for before the next is submitted
    gp = model.make_predictor(1, N, 1)
    gp.warmup(*inputs[0])

    def one(i):
        gp(*inputs[i % len(inputs)])
        gp.check()

    timed(one, 3, gp.stream.synchronize)
    n1 = max(3, min(24, a.steps))
    ms1 = timed(one, n1, gp.stream.synchronize) / n1
    return {"clouds_per_s": a.steps * cps / (ms / 1e3), "single_cloud_ms": ms1, "launches_per_cloud": pp.launches_per_step,
            "clouds_in_flight": a.depth}, (m.cpu().numpy(), iou.cpu().numpy())


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


torch.manual_seed(1234)
line = {"workload": f"hier: independent requests of 1 cloud, N={N}, PatchEmbedHier 2048x32 -> 512x32, eva02_large_patch14_448, "
                    "1 point prompt, multimask", "device": gpu_info()}
with torch.no_grad():
    line["hier"], (masks, iou) = run(build_point_sam_hier().to(dev).eval())
    if a.with_c2:
        torch.manual_seed(1234)
        line["c2"] = run(build_point_sam("eva02_large_patch14_448", 512, 64).to(dev).eval())[0]
        line["hier_over_c2"] = line["hier"]["clouds_per_s"] / line["c2"]["clouds_per_s"]
if a.dump_outputs:
    os.makedirs(a.dump_outputs, exist_ok=True)
    np.save(os.path.join(a.dump_outputs, "masks.npy"), masks)
    np.save(os.path.join(a.dump_outputs, "iou.npy"), iou)
    line["dumped_outputs"] = {"dir": a.dump_outputs, "masks": list(masks.shape), "iou": list(iou.shape)}
print(json.dumps(line))
