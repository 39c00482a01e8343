"""Evaluation driver with the behaviour of the reference's evaluation/eval_kitti.py:284-398 on top of the sm_90a
path: binary PLY crops (fields x y z R G B label) -> normalisation -> per-cloud group-count / group-size override ->
``model.forward_varlen`` on batches of crops of one group shape (``forward(is_eval=True)``'s iterative GT-driven prompting,
one crop per batch by default) -> IoU per prompt iteration, averaged per object class and overall.  The dataset glob is an argument instead of a hard-coded path; every crop is rotated by the reference's
fixed R.from_euler("xyz", [-90, 180, 0]) unless --rotation says otherwise (the network is not rotation invariant)."""
from __future__ import annotations

import argparse
import glob
import os
import sys
from typing import Dict, Hashable, List, Optional, Sequence, Tuple

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pc_sam.model.loss import compute_iou  # noqa: E402
from pc_sam.utils.ply import normalize_colors, normalize_points, read_ply, vertex_count  # noqa: E402
from psam_b200.parallel import plan_eval_batches  # noqa: E402,F401  (the batch plan, shared with the mask generator)


def transform_fn(x: Dict[str, np.ndarray], device="cuda") -> Dict[str, torch.Tensor]:
    """eval_kitti.py:91-114: one cloud with one ground-truth mask -> batched tensors."""
    xyz = normalize_points(np.asarray(x["xyz"]))
    rgb = normalize_colors(np.asarray(x["rgb"]))
    mask = np.asarray(x["mask"])
    xyz = torch.tensor(xyz, dtype=torch.float, device=device)
    rgb = torch.tensor(rgb, dtype=torch.float, device=device)
    mask = torch.tensor(mask, dtype=torch.bool, device=device)
    return {"coords": xyz[None], "features": rgb[None], "gt_masks": mask[None, None]}


def load_crop(path: str, rotation: Optional[np.ndarray] = None) -> Dict[str, np.ndarray]:
    """eval_kitti.py:340-350: structured PLY record -> float32 xyz (optionally rotated), float32 rgb (0..255), int32 label."""
    pc = read_ply(path)
    xyz = np.column_stack([pc["x"], pc["y"], pc["z"]]).astype(np.float32)
    if rotation is not None:
        xyz = np.float32(xyz @ np.asarray(rotation, dtype=np.float64).T)
    rgb = np.column_stack([pc["R"], pc["G"], pc["B"]]).astype(np.float32)
    return {"xyz": xyz, "rgb": rgb, "mask": pc["label"].astype(np.int32)}


REFERENCE_EULER_XYZ_DEG = (-90.0, 180.0, 0.0)  # eval_kitti.py:18: r = R.from_euler("xyz", [-90, 180, 0], degrees=True)


def euler_xyz_matrix(deg: Sequence[float]) -> np.ndarray:
    """scipy's Rotation.from_euler("xyz", deg, degrees=True).as_matrix() (extrinsic x, then y, then z), so that
    ``xyz @ M.T`` equals ``r.apply(xyz)`` of the reference driver (eval_kitti.py:18,347)."""
    a, b, c = (np.deg2rad(float(v)) for v in deg)
    rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    return rz @ ry @ rx


def parse_rotation(spec: Optional[str]) -> Optional[np.ndarray]:
    """--rotation: 'reference' (default: the reference driver's -90,180,0), 'none', or 'ax,ay,az' euler xyz in degrees."""
    if spec is None or spec == "reference":
        return euler_xyz_matrix(REFERENCE_EULER_XYZ_DEG)
    if spec.lower() == "none":
        return None
    vals = [float(v) for v in spec.split(",")]
    if len(vals) != 3:
        raise ValueError("--rotation expects 'reference', 'none' or three comma-separated euler xyz angles in degrees")
    return euler_xyz_matrix(vals)


def group_shape_for(num_points: int) -> Tuple[int, int]:
    """eval_kitti.py:352-362: the (num_groups, group_size) the reference gives a crop of num_points points."""
    if num_points > 30000:
        return 2048, 256
    return min(num_points, 2048), (2 if num_points < 256 else 256)


def set_group_shape(model, num_points: int):
    """The tokenizer's group count / size are runtime attributes chosen per cloud (group_shape_for).  A hierarchical
    tokenizer (PatchEmbedHier: grouper1 / grouper2, which that override does not address) is left as configured."""
    g = getattr(model.pc_encoder.patch_embed, "grouper", None)
    if g is None:
        return
    g.num_groups, g.group_size = group_shape_for(num_points)


def _run_batch(model, data: List[Dict[str, torch.Tensor]]):
    """One batch of transformed crops -> forward_varlen's per-crop lists.  A model with only the reference's forward (no
    forward_varlen) is run on a batch of one crop through forward, whose outputs have the same structure for B = 1."""
    if hasattr(model, "forward_varlen"):
        return model.forward_varlen([d["coords"][0] for d in data], [d["features"][0] for d in data],
                                    [d["gt_masks"][0] for d in data], is_eval=True)
    if len(data) != 1:
        raise TypeError(f"{type(model).__name__} has no forward_varlen: evaluate it with batch_size=1")
    return [model(**data[0], is_eval=True)]


def evaluate(model, files: Sequence[str], rotation: Optional[np.ndarray] = None, log=print, rank: Optional[int] = None,
             world: Optional[int] = None, batch_size: int = 1, max_batch_points: int = 1 << 20) -> Dict[str, object]:
    """Returns {"total": [prompt_iters], "per_object": {name: [prompt_iters]}, "object_mean": [prompt_iters]}.

    Crops run in batches of up to batch_size through model.forward_varlen (batch size 1 included, so there is one code
    path): plan_eval_batches groups them by group shape and size from their PLY headers, and each batch's crops are read
    only when it runs.  A crop whose labels are all 0 or all 1 has no border to sample prompts from and is refused
    (RuntimeError naming it).  IoU rows are kept in file order.

    Crops are independent, so with several processes (one per GPU, torch.distributed initialised) each rank evaluates a
    contiguous slice of `files` and the per-crop IoU rows are all-gathered once at the end; every rank
    returns the same aggregate.  Single process: rank/world default to 0/1."""
    import torch.distributed as dist

    from psam_b200.parallel import gather_metric, shard_range

    files = list(files)
    if world is None:
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank() if world > 1 else 0
    lo, hi = shard_range(len(files), rank or 0, world)
    mine = files[lo:hi]
    sizes = [vertex_count(p) for p in mine]
    flat = getattr(model.pc_encoder.patch_embed, "grouper", None) is not None
    keys = [group_shape_for(n) if flat else None for n in sizes]  # a hierarchical tokenizer keeps one shape
    rows: List[Optional[np.ndarray]] = [None] * len(mine)
    model.eval()
    dev = next(model.parameters()).device
    with torch.no_grad():
        for batch in plan_eval_batches(sizes, keys, batch_size, max_batch_points):
            data = []
            for i in batch:
                crop = load_crop(mine[i], rotation)
                fg = crop["mask"] != 0
                if not fg.any() or fg.all():
                    raise RuntimeError(f"{mine[i]}: every label is {int(fg[0])}, so the ground truth has no border to "
                                       "sample prompts from")
                data.append(transform_fn(crop, device=dev))
            set_group_shape(model, sizes[batch[0]])  # one key per batch
            outs = _run_batch(model, data)
            ious = torch.stack([torch.stack([compute_iou(o["prompt_masks"], d["gt_masks"][0]) for o in out])
                                for out, d in zip(outs, data)])  # [len(batch), prompt_iters, M]
            for i, r in zip(batch, ious.cpu().numpy()):  # one host copy per batch
                rows[i] = r.mean(axis=-1)
            if log:
                log(f"[rank {rank or 0}] current mean IoU: {np.array([r for r in rows if r is not None]).mean(axis=0)}")
    iters = int(getattr(model, "prompt_iters", rows[0].shape[0] if rows else 0))
    local = torch.tensor(np.array(rows), dtype=torch.float32).reshape(len(rows), iters)
    if world > 1:
        gdev = dev if dist.get_backend() == "nccl" else torch.device("cpu")
        local = gather_metric(local.to(gdev), len(files)).cpu()
    ious = local.numpy()
    per_obj: Dict[str, List[np.ndarray]] = {}
    for path, r in zip(files, ious):
        per_obj.setdefault(os.path.basename(path).split("_")[0], []).append(r)
    per = {k: np.array(v).mean(axis=0) for k, v in per_obj.items()}
    return {"total": ious.mean(axis=0) if len(ious) else np.zeros(0),
            "per_object": per,
            "object_mean": np.array(list(per.values())).mean(axis=0) if per else np.zeros(0)}


def main(argv=None):
    from pc_sam.utils.checkpoint import load_model
    from pc_sam.utils.config import compose, instantiate, model_config
    from pc_sam.utils.torch_utils import replace_with_fused_layernorm

    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=str, default="large")
    ap.add_argument("--config_dir", type=str, default=None, help="the reference's configs/ directory (optional)")
    ap.add_argument("--ckpt_path", type=str, default=None)
    ap.add_argument("--data", type=str, required=True, help="glob of binary PLY crops (x y z R G B label)")
    ap.add_argument("--rotation", type=str, default="reference",
                    help="'reference' = euler xyz -90,180,0 deg as eval_kitti.py:18 (default), 'none', or 'ax,ay,az' in degrees")
    ap.add_argument("--batch-size", type=int, default=1,
                    help="crops of the same group shape evaluated together in one padded batch (forward_varlen)")
    ap.add_argument("--max-batch-points", type=int, default=1 << 20,
                    help="cap on crops x largest crop size per batch (bounds the decoder's memory)")
    args, overrides = ap.parse_known_args(argv)
    cfg = compose(args.config_dir, args.config, overrides)["model"] if args.config_dir else model_config(args.config)
    torch.manual_seed(42)
    model = instantiate(cfg)
    model.apply(replace_with_fused_layernorm)
    if args.ckpt_path:
        load_model(model, args.ckpt_path)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:  # torchrun: one process per GPU, crops sharded by rank
        import torch.distributed as dist

        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    model.eval().cuda()
    res = evaluate(model, sorted(glob.glob(args.data)), rotation=parse_rotation(args.rotation), batch_size=args.batch_size,
                   max_batch_points=args.max_batch_points)
    if int(os.environ.get("RANK", "0")) == 0:
        print(f"Total mean IoU: {res['total']}")
        print(f"Object mean IoU: {res['object_mean']}")
    if world > 1:
        dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
