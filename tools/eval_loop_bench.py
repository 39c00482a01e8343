"""Evaluation-loop timing (config c3 shape: 4 clouds per GPU, N=32768, ViT-L, 3 prompt iterations with
GT-driven prompts; mask encoder active on iterations 2-3): forward(is_eval=True) eager (host checks per iteration)
vs the same loop replayed as one CUDA graph (PointCloudSAM.make_iterative_predictor).
usage: python tools/eval_loop_bench.py [--clouds 4] [--masks 1] [--iters 3] [--points 32768] [--steps 20]"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "point-sam_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from psam_b200 import synth  # noqa: E402
from pc_sam.model import build_point_sam  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--clouds", type=int, default=4)
ap.add_argument("--masks", type=int, default=1)
ap.add_argument("--iters", type=int, default=3)
ap.add_argument("--points", type=int, default=32768)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--encoder", default="eva02_large_patch14_448")
ap.add_argument("--groups", type=int, default=512)
ap.add_argument("--group-size", type=int, default=64)
ap.add_argument("--kind", default="ball")
a = ap.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(1234)
model = build_point_sam(a.encoder, a.groups, a.group_size).to(dev).eval()
model.prompt_iters = a.iters
B, M, N = a.clouds, a.masks, a.points
data = []
for s in range(2):
    xyz, feats = synth.make_batch(B, N, 300 + s, a.kind)
    gt = torch.stack([torch.stack([(xyz[b] - xyz[b, 997 * (m + 1)]).norm(dim=-1) < 0.45 + 0.05 * m for m in range(M)]) for b in range(B)])
    data.append(tuple(t.to(dev) for t in (xyz, feats, gt)))


def timeit(fn, steps):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


with torch.no_grad():
    ms_eager = timeit(lambda i: model(*data[i % 2], is_eval=True), a.steps)
pred = model.make_iterative_predictor(B, M, N)
pred.warmup(*data[0])
ms_graph = timeit(lambda i: pred(*data[i % 2], check=True), a.steps)
with torch.cuda.stream(pred.stream):
    ms_graph_nocheck = timeit(lambda i: pred(*data[i % 2], check=False), a.steps)
out = pred(*data[0])
from pc_sam.model.loss import compute_iou  # noqa: E402

ious = [float(compute_iou(o["prompt_masks"], data[0][2].flatten(0, 1)).mean()) for o in out]
print(json.dumps({"workload": f"{B} clouds x {M} mask(s), N={N}, G={a.groups}, K={a.group_size}, {a.encoder}, {a.iters} prompt iterations (forward(is_eval=True))",
                  "eager_ms_per_step": ms_eager, "graph_ms_per_step": ms_graph, "graph_ms_per_step_no_host_check": ms_graph_nocheck,
                  "clouds_per_s_eager": B / ms_eager * 1e3, "clouds_per_s_graph": B / ms_graph * 1e3,
                  "launches_per_step": pred.launches_per_step, "iou_vs_gt_random_weights": ious}))
