"""Automatic mask generation ("segment everything") on one cloud: N = 32768 points, the c2 model (eva02_large_patch14_448,
512 x 64 groups; --hier: PointCloudSAMHier, 2048 x 32 then 512 x 32), points_per_cloud = 1024, points_per_batch = 64.

Prints one JSON line: device name and power limit (read in the same run), ms per cloud of PointCloudMaskGenerator.generate_packed
(median of --steps after --warmup), its split into encode / decode / post-processing by CUDA events, candidates and kept masks,
the time of each new kernel (torch.profiler, separate run), mask_candidates' achieved bytes/s as a share of the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s), and a same-process PyTorch-composed arm of the post-processing (thresholds and sums,
intersections as an fp32 matmul of 0/1 masks, greedy NMS as a host loop) timed on the same logits, whose keep list must equal
the kernels'.

The weights are randomly initialised (no checkpoint is available offline), so SAM's default thresholds would reject every
candidate; by default the IoU and stability filters are off (every non-empty mask reaches NMS, its largest input).
--sam-thresholds uses SAM's defaults instead.

--min-region-area A (> 0) adds a "regions" object for SAM's small-region post-processing (min_mask_region_area = A): ms
per cloud of generate_packed with the stage, against the same without it measured alternately in the same run, the kernel
time of each op of the stage (kNN graph, mask_regions, second NMS; torch.profiler over 10 launches of the op alone on the
generator's own inputs, separate run), and the changed and kept counts.  With the default 0 the output is unchanged.

--crop-n-layers L (> 0) adds a "crops" object for SAM's crop layers (crop_n_layers = L, crop_n_points_downscale_factor =
--crop-downscale): ms per cloud with crops against the same generator without them, alternately in the same run, the
crops that ran with their point and prompt counts, and the kernel time of each new op over all crops of one cloud
(torch.profiler, each op alone on the generator's own inputs), with their share of the cloud's time.  The kNN graph of
min_mask_region_area is profiled at this N for reference.  --kind kitti uses the flattened scene-like synthetic cloud.
usage: python tools/amg_bench.py [--hier] [--steps 10] [--warmup 2] [--sam-thresholds] [--min-region-area 0]
                                 [--crop-n-layers 0] [--crop-downscale 1] [--kind ball] [--points 32768]"""
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
from pc_sam.model import build_point_sam, build_point_sam_hier  # noqa: E402
from psam_b200 import ops, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet

ap = argparse.ArgumentParser()
ap.add_argument("--hier", action="store_true")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--points", type=int, default=32768)
ap.add_argument("--prompts", type=int, default=1024)
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--sam-thresholds", action="store_true")
ap.add_argument("--min-region-area", type=int, default=0)
ap.add_argument("--crop-n-layers", type=int, default=0)
ap.add_argument("--crop-downscale", type=int, default=1)
ap.add_argument("--kind", default="ball", choices=["ball", "kitti"])
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("amg_bench: needs a CUDA device")
dev = torch.device("cuda:0")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(dev)


torch.manual_seed(1234)
model = (build_point_sam_hier() if a.hier else build_point_sam("eva02_large_patch14_448", 512, 64)).to(dev).eval()
kw = {} if a.sam_thresholds else dict(pred_iou_thresh=0.0, stability_score_thresh=0.0)
gen = PointCloudMaskGenerator(model, points_per_cloud=a.prompts, points_per_batch=a.batch, **kw)
xyz, rgb = (t.to(dev) for t in synth.make_batch(1, a.points, 5, a.kind))
N, P, Bp = a.points, a.prompts, a.batch
rules = dict(mask_threshold=gen.mask_threshold, stability_offset=gen.stability_score_offset, pred_iou_thresh=gen.pred_iou_thresh,
             stability_thresh=gen.stability_score_thresh, min_area=gen.min_mask_area)

# ---- end to end: generate_packed, host clock around a call that ends in its own synchronisation ----------------------
for _ in range(a.warmup):
    out = gen.generate_packed(xyz, rgb)
torch.cuda.synchronize()
ms = []
for _ in range(a.steps):
    t0 = time.perf_counter()
    out = gen.generate_packed(xyz, rgb)
    ms.append((time.perf_counter() - t0) * 1e3)
kept = int(out["area"].shape[0])


# ---- split by CUDA events: the generator's steps, each bracketed ------------------------------------------------------
def split_run():
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    spans = {"encode": [], "decode": [], "post": []}
    logits, ious = [], []
    with torch.no_grad():
        e0, e1 = ev(), ev()
        e0.record()
        enc = model._encode(xyz, rgb)
        _, centers = ops.fps(xyz, P)
        e1.record()
        spans["encode"].append((e0, e1))
        labels = torch.ones((Bp, 1), dtype=torch.int64, device=dev)
        cand = None
        for s in range(0, P, Bp):
            e = min(P, s + Bp)
            d0, d1, c1 = ev(), ev(), ev()
            d0.record()
            m, i = model._decode_unchecked(enc, centers[0, s:e].unsqueeze(1), labels[: e - s], None, True)
            d1.record()
            if cand is None:
                K = P * m.shape[1]
                cand = (torch.empty((K, ops.mask_words(N)), dtype=torch.int32, device=dev), torch.empty(K, dtype=torch.int32, device=dev),
                        torch.empty(K, dtype=torch.float32, device=dev), torch.empty(K, dtype=torch.float32, device=dev))
            ops.mask_candidates(m, i, out=cand, base=s * m.shape[1], **rules)
            c1.record()
            spans["decode"].append((d0, d1))
            spans["post"].append((d1, c1))
            logits.append(m)
            ious.append(i)
        n0, n1 = ev(), ev()
        n0.record()
        keep, cnt = ops.mask_nms(cand[0], cand[1], cand[3], gen.mask_nms_thresh)
        n1.record()
        spans["post"].append((n0, n1))
    torch.cuda.synchronize()
    t = {k: sum(x.elapsed_time(y) for x, y in v) for k, v in spans.items()}
    t["nms"] = n0.elapsed_time(n1)
    return t, torch.cat(logits), torch.cat(ious), cand, keep[: int(cnt.item())]


splits = [split_run()[0] for _ in range(3)]
split = {k: float(np.median([s[k] for s in splits])) for k in splits[0]}
_, lg, io, cand, keep = split_run()
C = lg.shape[1]
n_valid = int((cand[3] > float("-inf")).sum().item())

# ---- kernel times: torch.profiler over one generate_packed call -------------------------------------------------------
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    gen.generate_packed(xyz, rgb)
    torch.cuda.synchronize()
kern = {}
for evt in prof.events():
    for tag in ("mask_candidates_kernel", "nms_order_kernel", "nms_pairs_kernel", "nms_scan_kernel"):
        if tag in evt.name and evt.device_type == torch.autograd.DeviceType.CUDA:
            d = kern.setdefault(tag, [0.0, 0])
            d[0] += (getattr(evt, "device_time", None) or evt.cuda_time) / 1e3  # us -> ms
            d[1] += 1
kernel_ms = {k: {"ms_per_cloud": v[0], "launches": v[1]} for k, v in kern.items()}
cand_bytes = lg.numel() * 4 + io.numel() * 4 + cand[0].numel() * 4 + 3 * 4 * cand[1].numel()
if "mask_candidates_kernel" in kern:
    rate = cand_bytes / (kern["mask_candidates_kernel"][0] / 1e3)
    kernel_ms["mask_candidates_kernel"].update(bytes_per_cloud=cand_bytes, achieved_bytes_per_s=rate,
                                               share_of_hbm_peak=rate / HBM_BYTES_PER_S)


# ---- PyTorch-composed arm on the same logits ---------------------------------------------------------------------------
def torch_arm(lg, io):
    K = lg.shape[0] * lg.shape[1]
    flat, iou = lg.reshape(K, N), io.reshape(K)
    t0 = time.perf_counter()
    masks = flat > rules["mask_threshold"]
    area = masks.sum(1)
    hi = (flat > rules["mask_threshold"] + rules["stability_offset"]).sum(1)
    lo = (flat > rules["mask_threshold"] - rules["stability_offset"]).sum(1)
    stab = hi.float() / lo.float()
    ok = ~torch.isnan(iou) & (area >= rules["min_area"]) & (area >= 1)
    if rules["pred_iou_thresh"] > 0:
        ok &= iou > rules["pred_iou_thresh"]
    if rules["stability_thresh"] > 0:
        ok &= stab >= rules["stability_thresh"]
    score = torch.where(ok, iou, torch.full_like(iou, float("-inf")))
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    srt, order = torch.sort(score, descending=True, stable=True)
    order = order[srt > float("-inf")]
    m = masks[order].float()
    inter = m @ m.T  # exact: 0/1 products, sums <= N < 2^24
    a_ = area[order].float()
    sup = (inter / (a_[:, None] + a_[None, :] - inter) > gen.mask_nms_thresh).cpu().numpy()
    order = order.cpu().numpy()
    removed = np.zeros(len(order), dtype=bool)
    keep = []
    for i in range(len(order)):
        if not removed[i]:
            keep.append(int(order[i]))
            removed[i + 1:] |= sup[i, i + 1:]
    t2 = time.perf_counter()
    return keep, (t1 - t0) * 1e3, (t2 - t1) * 1e3


torch.backends.cuda.matmul.allow_tf32 = False
arm = [torch_arm(lg, io) for _ in range(3)]
assert arm[0][0] == keep.cpu().tolist(), "PyTorch-composed arm and kernels disagree"
nms_kernels_ms = sum(kernel_ms.get(k, {}).get("ms_per_cloud", 0.0) for k in ("nms_order_kernel", "nms_pairs_kernel", "nms_scan_kernel"))
med = float(np.median(ms))
line = {
    "workload": f"{'PointCloudSAMHier 2048x32 -> 512x32' if a.hier else 'c2 512x64'}, eva02_large_patch14_448, N={N}, "
                f"points_per_cloud={P}, points_per_batch={Bp}, "
                + ("SAM default thresholds" if a.sam_thresholds else "IoU / stability filters off, mask_nms_thresh 0.7"),
    "device": gpu_info(),
    "ms_per_cloud": med, "ms_per_cloud_range": [min(ms), max(ms)], "steps": a.steps,
    "split_ms": {"encode": split["encode"], "decode": split["decode"], "post": split["post"]},
    "post_share": split["post"] / (split["encode"] + split["decode"] + split["post"]),
    "candidates": P * C, "valid_candidates": n_valid, "kept_masks": kept,
    "kernels": kernel_ms,
    "nms_kernels_ms": nms_kernels_ms,
    "torch_arm_ms": {"candidates": float(np.median([x[1] for x in arm])), "nms": float(np.median([x[2] for x in arm]))},
    "torch_arm_keep_equal": True,
}
line["nms_speedup_vs_torch_arm"] = line["torch_arm_ms"]["nms"] / nms_kernels_ms if nms_kernels_ms else None


# ---- small-region post-processing: with / without alternately, then its kernels ----------------------------------------
def regions_report(A):
    on, off = [], []
    for _ in range(a.warmup):
        gen.generate_packed(xyz, rgb, min_mask_region_area=A)
    torch.cuda.synchronize()
    for _ in range(a.steps):
        for area, dst in ((A, on), (0, off)):
            t0 = time.perf_counter()
            gen.generate_packed(xyz, rgb, min_mask_region_area=area)
            dst.append((time.perf_counter() - t0) * 1e3)
    st = gen._enqueue(xyz, rgb, min_mask_region_area=A)
    n1, n2 = int(st["keep_count"].item()), int(st["region_count"].item())
    changed = int((st["region_score"][:n1] == 0).sum().item())  # rescoring: 0 = changed by the stage
    # kernel times of the stage: each op profiled alone (torch.profiler, separate run) on the generator's own inputs.  The
    # encoder's tokenizer also launches knn_kernel and the first NMS the nms_* kernels, so profiling the whole call could
    # not tell the stage's launches apart.
    k1 = min(gen.region_neighbors + 1, N)
    nbr = ops.knn(xyz, xyz, k1)[0]
    stage = {"knn_graph": (lambda: ops.knn(xyz, xyz, k1), ("knn_kernel",)),
             "mask_regions": (lambda: ops.mask_regions(st["bits"], st["keep"], st["keep_count"], nbr, A), ("mask_regions_kernel",)),
             "second_nms": (lambda: ops.mask_nms(st["region_bits"], st["region_area"], st["region_score"], gen.mask_nms_thresh),
                            ("nms_order_kernel", "nms_pairs_kernel", "nms_scan_kernel"))}
    reps, kernel_ms = 10, {}
    for name, (fn, tags) in stage.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        per = {}
        for evt in prof.events():
            if evt.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for tag in tags:
                if tag in evt.name:
                    per[tag] = per.get(tag, 0.0) + (getattr(evt, "device_time", None) or evt.cuda_time) / 1e3 / reps
        kernel_ms[name] = {"ms": sum(per.values()), "kernels": per}
    return {
        "min_region_area": A,
        "ms_per_cloud_with": float(np.median(on)), "ms_per_cloud_without": float(np.median(off)),
        "ms_per_cloud_with_range": [min(on), max(on)], "ms_per_cloud_without_range": [min(off), max(off)],
        "stage_ms": float(np.median(on) - np.median(off)),
        "kernel_ms": kernel_ms,
        "kept_first_nms": n1, "changed": changed, "kept_after_second_nms": n2,
    }


def profile_ms(fn, tags, reps=10):
    """ms per call of fn's kernels whose names contain one of tags (torch.profiler, fn alone)."""
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for evt in prof.events():
        if evt.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for tag in tags:
            if tag in evt.name:
                per[tag] = per.get(tag, 0.0) + (getattr(evt, "device_time", None) or evt.cuda_time) / 1e3 / reps
    return {"ms": sum(per.values()), "kernels": per}


# ---- crop layers: with / without alternately, the crops, then the new kernels each profiled alone ---------------------
def crops_report(layers, factor):
    ck = dict(crop_n_layers=layers, crop_n_points_downscale_factor=factor)
    ratio, crop_nms, margin = 512 / 1500, 0.7, gen.crop_edge_margin  # SAM's defaults
    for _ in range(a.warmup):
        gen.generate_packed(xyz, rgb, **ck)
    torch.cuda.synchronize()
    on, off = [], []
    for _ in range(a.steps):
        for c, dst in ((ck, on), ({}, off)):
            t0 = time.perf_counter()
            gen.generate_packed(xyz, rgb, **c)
            dst.append((time.perf_counter() - t0) * 1e3)
    st = gen._enqueue(xyz, rgb, **ck, keep_crop_states=True)
    out = gen._finish(st)
    counts = st["crop_counts"].tolist()
    crops = st["crops"]
    sub = [c for c in crops if c["layer"] > 0]
    boxes = st["crop_boxes"]
    gathered = [ops.crop_gather(xyz, rgb, boxes, c["crop"], counts[c["crop"]], margin) for c in sub]
    lifted = tuple(st[k] for k in ("bits", "area", "score", "stability", "prompt", "mask_slot", "crop", "crop_score"))
    offsets = torch.zeros(len(crops) + 1, dtype=torch.int32, device=dev)
    over = torch.zeros(1, dtype=torch.int32, device=dev)

    def uncrop_all():
        for k, c in enumerate(crops):
            ops.crop_uncrop((c["bits"], c["area"], c["stability"], c["score"]), c["keep"], c["keep_count"], c["idx"], c["point_index"],
                            c["slots"], c["crop"], float(c["layer"]), offsets, k, lifted, over, N)

    def edge_all():
        for c, g in zip(sub, gathered):
            ops.crop_edge_filter(c["bits"], c["score"].clone(), g[3])

    k1 = min(gen.region_neighbors + 1, N)
    kernels = {
        "crop_layout": profile_ms(lambda: ops.crop_layout(xyz, layers, ratio), ("crop_layout_kernel", "crop_count_kernel")),
        "crop_gather (all crops)": profile_ms(lambda: [ops.crop_gather(xyz, rgb, boxes, c["crop"], counts[c["crop"]], margin)
                                                       for c in sub], ("crop_gather",)),
        "crop_edge_filter (all crops)": profile_ms(edge_all, ("crop_edge_filter_kernel",)),
        "crop_uncrop (all crops)": profile_ms(uncrop_all, ("crop_uncrop_kernel",)),
        "nms_across_crops": profile_ms(lambda: ops.mask_nms(st["bits"], st["area"], st["crop_score"], crop_nms),
                                       ("nms_order_kernel", "nms_pairs_kernel", "nms_scan_kernel")),
        "knn_graph (min_mask_region_area, not run here)": profile_ms(lambda: ops.knn(xyz, xyz, k1), ("knn_kernel",), reps=3),
    }
    new_ms = sum(v["ms"] for k, v in kernels.items() if not k.startswith("knn_graph"))
    med_on = float(np.median(on))
    return {
        "crop_n_layers": layers, "crop_n_points_downscale_factor": factor,
        "ms_per_cloud_with": med_on, "ms_per_cloud_without": float(np.median(off)),
        "ms_per_cloud_with_range": [min(on), max(on)], "ms_per_cloud_without_range": [min(off), max(off)],
        "crops_run": len(crops), "points_per_crop": [c["points"] for c in crops], "prompts_per_crop": [c["prompts"] for c in crops],
        "crops_skipped": sum(1 for t in range(1, len(counts)) if t not in {c["crop"] for c in crops}),
        "lifted_masks": int(st["lifted_count"].item()), "kept_masks": int(out["area"].shape[0]),
        "kept_from_deeper_layers": int((out["crop_box"] != st["crop_boxes"][0]).any(1).sum().item()),
        "kernel_ms": kernels, "new_kernels_ms": new_ms, "new_kernels_share": new_ms / med_on,
    }


if a.min_region_area > 0:
    line["regions"] = regions_report(a.min_region_area)
if a.crop_n_layers > 0:
    line["crops"] = crops_report(a.crop_n_layers, a.crop_downscale)
print(json.dumps(line))
