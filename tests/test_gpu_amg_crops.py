"""GPU tests of the crop layers of automatic mask generation (crop_n_layers): the layout, gather, edge-filter and uncrop
kernels equal the numpy oracle bit for bit (N = 33 to 262144, layers 1 and 2, points on crop bounds and margins, flat and
coincident clouds, the lifted-set capacity and one past it), the generator matches the fp32 oracle crop by crop and then
through the merge for both model classes, crop_n_layers = 0 leaves the output as it was, the host synchronises exactly
twice, and the invariants hold at full size (ViT-L, N = 131072, one crop layer)."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_crops_ref, amg_ref, amg_regions_ref, hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
F = np.float32
R = amg_crops_ref.OVERLAP_RATIO
MARGIN = amg_crops_ref.EDGE_MARGIN


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


# ------------------------------------------------------------------------------------------------
# 1. kernel exactness
# ------------------------------------------------------------------------------------------------
def _cloud(N, seed, layers, kind="scene"):
    """A room-like scene (a floor, a wall, objects), with points moved exactly onto crop bounds and onto the edge margins
    of interior faces; or a flat cloud (zero extent along z); or coincident points."""
    rng = np.random.default_rng(seed)
    if kind == "coincident":
        return np.tile(F([[0.3, -0.1, 0.7]]), (N, 1))
    if kind == "nan":  # NaN coordinates are ignored by the bounding box and lie in no crop
        x = _cloud(N, seed, layers)
        x[rng.choice(N, 40, replace=False), rng.integers(0, 3, 40)] = np.nan
        return x
    n1 = N // 3
    floor = np.c_[rng.uniform(-1, 1, (n1, 2)), np.full(n1, -0.2)]
    c = rng.uniform(-0.8, 0.8, (6, 2))
    k = rng.integers(0, 6, N - n1)
    objs = np.c_[c[k] + rng.normal(0, 0.08, (N - n1, 2)), rng.uniform(-0.2, 0.25, N - n1)]
    x = np.clip(np.concatenate([floor, objs]), -1, 1).astype(F)[rng.permutation(N)]
    if kind == "flat":
        x[:, 2] = F(0.125)
        return x
    boxes, _, _ = amg_crops_ref.layout(x, layers, R)
    bb = boxes[0]
    for i in rng.choice(N, min(N // 4, 4096), replace=False):  # on a bound, or on a margin of a face
        t, a = int(rng.integers(1, len(boxes))), int(rng.integers(0, 3))
        m = F(F(MARGIN) * F(bb[3 + a] - bb[a]))
        v = [boxes[t, a], boxes[t, 3 + a], F(boxes[t, a] + m), F(boxes[t, 3 + a] - m)][int(rng.integers(0, 4))]
        x[i, a] = np.clip(v, bb[a], bb[3 + a])
    return x


def _check_layout_and_gather(x, layers, max_crops=None):
    from psam_b200 import ops

    N = len(x)
    rgb = np.random.default_rng(N).uniform(-1, 1, (N, 3)).astype(F)
    xd, rd = torch.from_numpy(x).to(DEV), torch.from_numpy(rgb).to(DEV)
    boxes, counts = ops.crop_layout(xd, layers, R)
    want_boxes, want_counts, _ = amg_crops_ref.layout(x, layers, R)
    assert np.array_equal(boxes.cpu().numpy().view(np.uint32), want_boxes.view(np.uint32))
    assert counts.cpu().numpy().tolist() == want_counts.tolist()
    ts = [t for t in range(len(want_boxes)) if want_counts[t] >= 1][:max_crops]
    near = 0
    for t in ts:
        idx, cx, cr, edge = ops.crop_gather(xd, rd, boxes, t, int(want_counts[t]), MARGIN)
        w_idx, w_x, w_c, w_edge = amg_crops_ref.crop_cloud(x, rgb, want_boxes, t, MARGIN)
        assert idx.cpu().numpy().tolist() == w_idx.tolist(), t
        assert np.array_equal(cx[0].cpu().numpy().view(np.uint32), w_x.view(np.uint32)), t
        assert np.array_equal(cr[0].cpu().numpy(), w_c)
        assert np.array_equal(_u32(edge), amg_ref.pack_bits(w_edge[None])[0]), t
        assert float(cx.abs().max()) <= 1
        near += int(w_edge.sum())
    return want_counts, near


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("N", [33, 2047, 32768, 262144])
def test_layout_and_gather_match_oracle_exactly(N, layers):
    counts, near = _check_layout_and_gather(_cloud(N, N + layers, layers), layers)
    assert counts[0] == N and np.all(counts >= 0)
    if N >= 2047:
        assert near > 0


@pytest.mark.parametrize("kind", ["flat", "coincident", "nan"])
def test_layout_and_gather_on_degenerate_clouds(kind):
    x = _cloud(3000, 1, 2, kind)
    counts, near = _check_layout_and_gather(x, 2)
    if kind == "nan":
        assert counts[0] == 3000 - int(np.isnan(x).any(1).sum()) and np.all(counts >= 0)
        return
    assert (counts == -1).sum() >= (36 if kind == "flat" else 70)  # flat: jz > 0 repeats jz = 0; coincident: one box a layer
    if kind == "coincident":
        assert near == 0


def test_edge_filter_matches_oracle():
    from psam_b200 import ops

    rng = np.random.default_rng(0)
    for K, n in ((1, 33), (300, 2047), (3072, 40000)):
        W = ops.mask_words(n)
        masks = rng.random((K, n)) < rng.uniform(0.0005, 0.02, (K, 1))
        edge = rng.random(n) < 0.01
        bits, eb = amg_ref.pack_bits(masks), amg_ref.pack_bits(edge[None])[0]
        score = rng.uniform(0, 1, K).astype(F)
        score[::7] = -np.inf
        b, s = torch.from_numpy(bits.view(np.int32)).to(DEV), torch.from_numpy(score).to(DEV)
        ops.crop_edge_filter(b, s, torch.from_numpy(eb.view(np.int32)).to(DEV))
        want = amg_crops_ref.edge_filter(bits, score, eb)
        assert np.array_equal(s.cpu().numpy(), want) and W == bits.shape[1]
        if K > 1:
            assert 0 < int((want == -np.inf).sum()) < K


def _lift(per_crop, N, cap):
    from psam_b200 import ops

    W = ops.mask_words(N)
    out = (torch.empty((cap, W), dtype=torch.int32, device=DEV), torch.empty(cap, dtype=torch.int32, device=DEV),
           torch.empty(cap, dtype=torch.float32, device=DEV), torch.empty(cap, dtype=torch.float32, device=DEV),
           torch.empty(cap, dtype=torch.int64, device=DEV), torch.empty(cap, dtype=torch.int32, device=DEV),
           torch.empty(cap, dtype=torch.int32, device=DEV), torch.full((cap,), float("-inf"), dtype=torch.float32, device=DEV))
    offsets = torch.zeros(len(per_crop) + 1, dtype=torch.int32, device=DEV)
    overflow = torch.zeros(1, dtype=torch.int32, device=DEV)
    for k, c in enumerate(per_crop):
        cand = tuple(torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for v in
                     (c["bits"].view(np.int32), c["area"], c["stability"], c["score"]))
        keep = np.zeros(len(c["area"]), np.int32)
        keep[: len(c["keep"])] = c["keep"]
        ops.crop_uncrop(cand, torch.from_numpy(keep).to(DEV), torch.tensor([len(c["keep"])], dtype=torch.int32, device=DEV),
                        torch.from_numpy(c["idx"].astype(np.int32)).to(DEV), torch.from_numpy(c["point_index"]).to(DEV), c["slots"],
                        c["crop"], float(c["layer"]), offsets, k, out, overflow, N)
    torch.cuda.synchronize()
    return out, int(offsets[-1].item()), int(overflow.item())


def test_uncrop_matches_oracle_at_capacity_and_one_past():
    rng = np.random.default_rng(7)
    N, per_crop = 40000, []
    for k, (t, layer, n, P) in enumerate(((0, 0, 40000, 40), (3, 1, 12000, 30), (5, 1, 33, 8), (70, 2, 4100, 20))):
        idx = np.arange(N) if layer == 0 else np.sort(rng.choice(N, n, replace=False))
        K = 3 * P
        masks = rng.random((K, n)) < rng.uniform(0.001, 0.3, (K, 1))
        masks[:, -1] |= rng.random(K) < 0.5  # the last local point (bits up to n)
        keep = rng.permutation(K)[: int(rng.integers(1, K))]
        per_crop.append(dict(crop=t, layer=layer, idx=idx, bits=amg_ref.pack_bits(masks), area=masks.sum(1).astype(np.int32),
                             score=rng.uniform(0, 1, K).astype(F), stability=rng.uniform(0, 1, K).astype(F), keep=keep,
                             point_index=rng.integers(0, n, P).astype(np.int64), slots=3))
    total = sum(len(c["keep"]) for c in per_crop)
    for cap in (total, total - 1):
        out, lifted, over = _lift(per_crop, N, cap)
        want = amg_crops_ref.merge(per_crop, N, 0.7, cap)
        assert lifted == total and over == int(total > cap) and want["overflow"] == (total > cap)
        rows = min(total, cap)
        gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore = (t.cpu().numpy() for t in out)
        assert np.array_equal(gbits[:rows].view(np.uint32), want["bits"])
        for got, key in ((garea, "area"), (giou, "iou"), (gstab, "stability"), (gprompt, "prompt"), (gslot, "mask_slot"),
                         (gcrop, "crop"), (gscore, "layer_score")):
            assert np.array_equal(got[:rows], want[key]), key
        assert np.all(gscore[rows:] == -np.inf)


# ------------------------------------------------------------------------------------------------
# 2. the generator end to end
# ------------------------------------------------------------------------------------------------
# IoU / stability filters off (every non-empty mask is a candidate), so the decisions are a candidate's emptiness, the edge
# filter and the two NMS.  Seeds and thresholds chosen on the CPU oracle so that every NMS decision of every crop and of the
# merge has a margin of at least 1e-2 (asserted below).  Emptiness and the edge filter are decided by single logits, and the
# random tiny models put some logits of most masks within 1e-3 of the threshold, so no margin can be asked of them: the
# test checks those decisions exactly on the device's own masks, and the masks against the oracle's logits.
FIXTURES = {
    "base": dict(seed=5, area=8, crop_nms=0.7, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, stability_score_offset=0.05,
                                                        mask_nms_thresh=0.9)),
    "hier": dict(seed=9, area=8, crop_nms=0.7, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, stability_score_offset=0.05,
                                                        mask_nms_thresh=0.9)),
}
PROMPTS, BATCH, N_E2E = 32, 12, 2048


def _models(kind, seed):
    from pc_sam.model import build_point_sam, build_point_sam_hier

    if kind == "base":
        oracle = torch_ref.build_model("eva02_test_tiny", 64, 32, seed=seed)
        model = build_point_sam("eva02_test_tiny", 64, 32)
    else:
        oracle = hier_ref.build_hier_model("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3, seed=seed)
        model = build_point_sam_hier("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3)
    model.load_state_dict(oracle.state_dict(), strict=True)
    return model.cuda().eval(), oracle


def _np(t):
    return t.cpu().numpy()


def _nms_margin(bits, area, order, nt):
    """Smallest |IoU - nt| of the greedy NMS decisions along `order` (each later candidate against the kept ones)."""
    if len(order) < 2:
        return np.inf
    P = amg_ref.pair_ious(bits, area, order)
    m, kept = [np.inf], []
    for j in range(len(order)):
        ious = P[kept, j]
        sup = ious[ious > nt]
        m.append((sup - nt).max() if len(sup) else (nt - ious).min() if len(ious) else np.inf)
        if not len(sup):
            kept.append(j)
    return float(min(m))


def _crop_margin(w, nt):
    return _nms_margin(w["bits"], w["area"], amg_ref.sort_order(w["score"]), nt)


def _merge_margin(merged, nt):
    return _nms_margin(merged["bits"], merged["area"], amg_ref.sort_order(merged["layer_score"]), nt)


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_generator_crops_match_fp32_oracle(kind):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES[kind]
    model, oracle = _models(kind, fx["seed"])
    xyz, rgb = synth.make_batch(1, N_E2E, fx["seed"])
    want = amg_crops_ref.generate_ref(oracle, xyz, rgb, PROMPTS, PROMPTS, **fx["kw"], crop_n_layers=1, crop_nms_thresh=fx["crop_nms"],
                                      min_points=model._group_shape()[0])
    nt = fx["kw"]["mask_nms_thresh"]
    margins = [_crop_margin(w, nt) for w in want["crops"]]
    merge_margin = _merge_margin(want["merged"], fx["crop_nms"])
    print(f"[amg crops] {kind}: decision margins per crop {np.round(margins, 4).tolist()}, merge {merge_margin:.4g}")
    assert min(margins) >= 1e-2 and merge_margin >= 1e-2
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **fx["kw"])
    crop = dict(crop_n_layers=1, crop_nms_thresh=fx["crop_nms"])
    xd, rd = xyz[0].to(DEV), rgb[0].to(DEV)
    st = gen._enqueue(xd, rd, **crop, keep_crop_states=True)
    got = gen._finish(st)
    assert np.array_equal(_u32(st["crop_boxes"]), want["boxes"].view(np.uint32))
    assert _np(st["crop_counts"]).tolist() == want["counts"].tolist()
    # crop by crop: the same crops ran on the same points, and the device kept the oracle's candidates
    assert [c["crop"] for c in st["crops"]] == [c["crop"] for c in want["crops"]] and len(st["crops"]) > 1
    per, crop_kept = [], 0
    for c, w in zip(st["crops"], want["crops"]):
        n = int(c["keep_count"].item())
        assert _np(c["idx"]).tolist() == np.asarray(w["idx"]).tolist()
        assert _np(c["point_index"]).tolist() == w["point_index"].tolist()
        # the device's candidates are the oracle's: mask bits up to logits within 1e-3 of the threshold, exact areas,
        # predicted IoU within 1e-3
        seg = amg_ref.unpack_bits(_u32(c["bits"]), c["points"])
        lg = w["logits"].reshape(len(seg), -1)
        diff = seg != (lg > 0)
        assert np.all(np.abs(lg[diff]) < 1e-3), f"crop {c['crop']}: {diff.sum()} points differ"
        assert np.array_equal(_np(c["area"]), seg.sum(1))
        score, keep_c = _np(c["score"]), _np(c["keep"])[:n]
        valid = score > -np.inf
        np.testing.assert_allclose(score[valid], w["iou"].reshape(-1)[valid], atol=1e-3, rtol=0)
        # exact on the device's own masks: a non-empty candidate is valid unless it touches the edge bitset, and the crop's
        # NMS keeps the oracle's list in the oracle's order
        edge = np.zeros(c["points"], bool) if w["edge"] is None else w["edge"]
        hit = (seg & edge[None]).any(1)
        assert np.array_equal(valid, (seg.sum(1) >= 1) & ~hit), c["crop"]
        assert keep_c.tolist() == amg_ref.nms(_u32(c["bits"]), _np(c["area"]), score, nt).tolist(), c["crop"]
        # and the same masks as the fp32 oracle's run kept (compared by content: two identical masks with near-equal
        # predicted IoUs may be kept under either slot)
        assert sorted(w["bits"][k].tobytes() for k in keep_c) == sorted(w["bits"][k].tobytes() for k in w["keep"]), c["crop"]
        crop_kept += n if c["layer"] else 0
        per.append(dict(crop=c["crop"], layer=c["layer"], idx=_np(c["idx"]).astype(np.int64), bits=_u32(c["bits"]), area=_np(c["area"]),
                        score=_np(c["score"]), stability=_np(c["stability"]), keep=_np(c["keep"])[:n],
                        point_index=_np(c["point_index"]), slots=c["slots"]))
    print(f"[amg crops] {kind}: {len(per)} crops, {crop_kept} masks kept in layer-1 crops, {len(want['final'])} after the merge")
    assert crop_kept > 0
    # the merge of the device's per-crop results, exactly
    cap = st["bits"].shape[0]
    m = amg_crops_ref.merge(per, N_E2E, fx["crop_nms"], cap)
    L = len(m["area"])
    assert int(st["lifted_count"].item()) == L and not m["overflow"]
    assert np.array_equal(_u32(st["bits"])[:L], m["bits"])
    assert np.array_equal(_np(st["crop_score"])[:L], m["layer_score"])
    keep = m["keep"]
    assert _np(st["keep"])[: int(st["keep_count"].item())].tolist() == keep.tolist()
    assert np.array_equal(_u32(got["bits"]), m["bits"][keep]) and np.array_equal(_np(got["area"]), m["area"][keep])
    assert _np(got["point_index"]).tolist() == m["prompt"][keep].tolist()
    assert _np(got["mask_slot"]).tolist() == m["mask_slot"][keep].tolist()
    assert np.array_equal(_np(got["predicted_iou"]), m["iou"][keep])
    np.testing.assert_array_equal(_np(got["point_coords"]), xyz[0].numpy()[m["prompt"][keep]])
    assert np.array_equal(_np(got["crop_box"]), want["boxes"][m["crop"][keep]])
    assert len({int(c) for c in m["crop"][keep]}) > 1
    # the merge and the kept crops agree with the oracle's own run (decisions with margins)
    assert sorted(m["crop"][keep].tolist()) == sorted(want["merged"]["crop"][want["final"]].tolist())
    # records: SAM's crop_box key
    recs = gen.generate(xd, rd, **crop)
    assert [r["crop_box"] for r in recs] == _np(got["crop_box"]).tolist()
    # small regions on the merged set, over the whole cloud's kNN graph
    from psam_b200 import ops

    A = fx["area"]
    st2 = gen._enqueue(xd, rd, min_mask_region_area=A, **crop)
    got2 = gen._finish(st2)
    nbr = ops.knn(xd[None], xd[None], amg_regions_ref.REGION_NEIGHBORS + 1)[0][0].cpu().numpy()
    post = amg_regions_ref.postprocess_small_regions(m["bits"], keep, nbr, A, fx["kw"]["mask_nms_thresh"])
    assert np.array_equal(_u32(got2["bits"]), post["bits"][post["keep"]])
    assert _np(got2["point_index"]).tolist() == m["prompt"][keep[post["keep"]]].tolist()


def test_generator_without_crops_is_unchanged():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import native

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t[0].to(DEV) for t in synth.make_batch(1, N_E2E, fx["seed"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=16, **fx["kw"])
    gen.generate_packed(xyz, rgb)  # packs the weights
    n0 = native.LAUNCHES[0]
    a = gen.generate_packed(xyz, rgb)
    n1 = native.LAUNCHES[0]
    b = gen.generate_packed(xyz, rgb, crop_n_layers=0, crop_nms_thresh=0.1, crop_overlap_ratio=0.9, crop_n_points_downscale_factor=3)
    assert native.LAUNCHES[0] - n1 == n1 - n0  # nothing new is launched
    assert a.keys() == b.keys() and "crop_box" not in a
    for k in ("bits", "area", "point_index", "point_coords", "mask_slot"):
        assert torch.equal(a[k], b[k]), k
    for k in ("predicted_iou", "stability_score"):  # the decoder's fp32 reductions may round differently from run to run
        torch.testing.assert_close(a[k], b[k], atol=1e-5, rtol=0)


def test_crops_synchronise_twice():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t[0].to(DEV) for t in synth.make_batch(1, N_E2E, fx["seed"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **fx["kw"])
    first = gen.generate_packed(xyz, rgb, crop_n_layers=2)  # packs the weights
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            got = gen.generate_packed(xyz, rgb, crop_n_layers=2)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
    assert len(syncs) == 2, [str(w.message) for w in caught]
    assert torch.equal(first["bits"], got["bits"]) and torch.equal(first["crop_box"], got["crop_box"])


def test_generator_raises_when_lifted_masks_overflow():
    """The kernel sets the overflow flag at capacity + 1 (test above); the final read turns the flag into ValueError."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t[0].to(DEV) for t in synth.make_batch(1, N_E2E, fx["seed"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **fx["kw"])
    st = gen._enqueue(xyz, rgb, crop_n_layers=1)
    assert int(st["overflow"].item()) == 0 and int(st["lifted_count"].item()) <= st["bits"].shape[0]
    st["overflow"].fill_(1)
    with pytest.raises(ValueError, match="lifted"):
        gen._finish(st)


# ------------------------------------------------------------------------------------------------
# 3. full size, once
# ------------------------------------------------------------------------------------------------
def test_crops_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    xyz, rgb = synth.make_batch(1, 131072, 3, "kitti")
    xd, rd = xyz[0].to(DEV), rgb[0].to(DEV)
    ct = 0.7
    gen = PointCloudMaskGenerator(model, points_per_cloud=1024, points_per_batch=32, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05)
    st = gen._enqueue(xd, rd, crop_n_layers=1, crop_nms_thresh=ct)
    out = gen._finish(st)
    boxes = _np(st["crop_boxes"])
    crop = _np(st["crop"])[_np(st["keep"])[: out["area"].shape[0]]]
    print(f"[amg crops] full size: {len(st['crops'])} crops, {int(st['lifted_count'].item())} lifted, {len(crop)} kept, "
          f"{int((crop > 0).sum())} from layer 1, points per crop {_np(st['crop_counts']).tolist()}")
    assert len(st["crops"]) > 1 and (crop > 0).any() and (crop == 0).any()
    # no two kept masks overlap above crop_nms_thresh (fp32 IoU of exact counts, as the kernel compares)
    m = torch.from_numpy(amg_ref.unpack_bits(_u32(out["bits"]), 131072)).to(DEV).float()
    inter = (m @ m.T).round().long().cpu().numpy()
    area = _np(out["area"]).astype(np.int64)
    assert np.array_equal(np.diag(inter), area)
    iou = inter.astype(F) / (area[:, None] + area[None, :] - inter).astype(F)
    np.fill_diagonal(iou, 0)
    assert iou.max() <= ct
    # no kept mask of a layer-1 crop touches an interior face of its crop
    x = xyz[0].numpy()
    seg = m.bool().cpu().numpy()
    for t in np.unique(crop[crop > 0]):
        idx, _, _, edge = amg_crops_ref.crop_cloud(x, x, boxes, int(t))
        g = np.zeros(len(x), bool)
        g[idx[edge]] = True
        assert not (seg[crop == t] & g[None]).any(), t
