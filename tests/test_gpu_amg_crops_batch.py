"""GPU tests of crop layers on a batch of clouds: the batched layout, gather, edge filter and uncrop equal the single-crop
kernels bit for bit (equal N and padded lists with padding built to win if read, 1024-point chunk boundaries, degenerate
clouds with duplicate boxes, the uncrop capacity exactly reached and one past with only the overflowing cloud flagged);
generate_packed_batch_crops on three clouds of different sizes matches the fp32 oracle (amg_crops_ref.generate_ref) crop
by crop and through the merge, with decision margins asserted, and generate_packed's crop path bit for bit up to the
encoder, for both model classes and 1 or 2 layers; a real overflow is flagged on its own cloud only; a cloud
with no layer-1 crop skips the merge next to clouds that have crops; two host synchronisations per call; crop_n_layers = 0
is generate_packed_batch launch for launch; and the full-size invariants hold for two ViT-L clouds."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_crops_ref, amg_ref, hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
F = np.float32
R = amg_crops_ref.OVERLAP_RATIO
MARGIN = amg_crops_ref.EDGE_MARGIN


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _np(t):
    return t.cpu().numpy()


def _scene(N, seed, kind="scene"):
    rng = np.random.default_rng(seed)
    if kind == "coincident":
        return np.tile(F([[0.3, -0.1, 0.7]]), (N, 1))
    n1 = N // 3
    floor = np.c_[rng.uniform(-1, 1, (n1, 2)), np.full(n1, -0.2)]
    c = rng.uniform(-0.8, 0.8, (6, 2))
    k = rng.integers(0, 6, N - n1)
    objs = np.c_[c[k] + rng.normal(0, 0.08, (N - n1, 2)), rng.uniform(-0.2, 0.25, N - n1)]
    x = np.clip(np.concatenate([floor, objs]), -1, 1).astype(F)[rng.permutation(N)]
    if kind == "flat":
        x[:, 2] = F(0.125)
    return x


def _padded(clouds, pad):
    """[B, N_max, 3] with rows past each cloud filled by `pad` (values that would win the bounding box or every count)."""
    N = max(len(x) for x in clouds)
    out = np.empty((len(clouds), N, 3), F)
    for b, x in enumerate(clouds):
        out[b, :len(x)] = x
        out[b, len(x):] = pad
    return out


# ------------------------------------------------------------------------------------------------
# 1. the batched kernels against the single-crop kernels
# ------------------------------------------------------------------------------------------------
CASES = {
    "equal": ([3000, 3000, 3000], None, 1),
    "padded": ([1023, 1025, 4097, 2048], F(1e30), 2),
    "padded_nan": ([2047, 5000, 1024], F(np.nan), 1),
    "padded_inside": ([3000, 700, 2049], F(0.01), 2),  # padding inside every box: would be counted if read
}


@pytest.mark.parametrize("case", list(CASES))
def test_layout_and_gather_batched_equal_single(case):
    from psam_b200 import ops

    sizes, pad, layers = CASES[case]
    clouds = [_scene(n, 10 * b + n) for b, n in enumerate(sizes)]
    rgbs = [np.random.default_rng(n).uniform(-1, 1, (n, 3)).astype(F) for n in sizes]
    if pad is None:
        xd, rd, lengths = torch.from_numpy(np.stack(clouds)).to(DEV), torch.from_numpy(np.stack(rgbs)).to(DEV), None
    else:
        xd, rd = torch.from_numpy(_padded(clouds, pad)).to(DEV), torch.from_numpy(_padded(rgbs, F(-7.0))).to(DEV)
        lengths = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    boxes, counts = ops.crop_layout_batched(xd, layers, R, lengths)
    pairs = []
    for b, x in enumerate(clouds):
        xb, rb = torch.from_numpy(x).to(DEV), torch.from_numpy(rgbs[b]).to(DEV)
        sb, sc = ops.crop_layout(xb, layers, R)
        assert np.array_equal(_u32(boxes[b]), _u32(sb)) and _np(counts[b]).tolist() == _np(sc).tolist(), b
        assert int(counts[b, 0]) == sizes[b]
        pairs += [(b, t, int(c)) for t, c in enumerate(_np(sc)) if c >= 1]
    # every (cloud, crop) pair with points, in one padded batch, against crop_gather of that cloud alone
    idx, cx, cr, edge, clen = ops.crop_gather_batched(xd, rd, boxes, pairs, MARGIN, lengths)
    n_max = max(c for _, _, c in pairs)
    assert tuple(idx.shape) == (len(pairs), n_max) and tuple(edge.shape) == (len(pairs), ops.mask_words(n_max))
    assert _np(clen).tolist() == [c for _, _, c in pairs]
    near = 0
    for p, (b, t, c) in enumerate(pairs):
        xb, rb = torch.from_numpy(clouds[b]).to(DEV), torch.from_numpy(rgbs[b]).to(DEV)
        si, sx, sr, se = ops.crop_gather(xb, rb, boxes[b], t, c, MARGIN)
        assert torch.equal(idx[p, :c], si), (b, t)
        assert np.array_equal(_u32(cx[p, :c]), _u32(sx[0])) and np.array_equal(_u32(cr[p, :c]), _u32(sr[0])), (b, t)
        W = ops.mask_words(c)
        assert np.array_equal(_u32(edge[p, :W]), _u32(se)), (b, t)
        assert not _u32(edge[p, W:]).any()
        assert not _np(idx[p, c:]).any() and not _np(cx[p, c:]).any() and not _np(cr[p, c:]).any()
        near += int(np.unpackbits(_u32(se).view(np.uint8)).sum())
    assert near > 0


def test_layout_and_gather_batched_on_degenerate_clouds():
    """Duplicate boxes (count -1) on a flat and a coincident cloud, next to a scene, padded."""
    from psam_b200 import ops

    clouds = [_scene(3000, 1, "flat"), _scene(1500, 2, "coincident"), _scene(2500, 3)]
    sizes = [len(x) for x in clouds]
    xd = torch.from_numpy(_padded(clouds, F(-1e30))).to(DEV)
    rd = torch.from_numpy(_padded(clouds, F(0))).to(DEV)
    lengths = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    boxes, counts = ops.crop_layout_batched(xd, 2, R, lengths)
    pairs = []
    for b, x in enumerate(clouds):
        sb, sc = ops.crop_layout(torch.from_numpy(x).to(DEV), 2, R)
        assert np.array_equal(_u32(boxes[b]), _u32(sb)) and _np(counts[b]).tolist() == _np(sc).tolist()
        want_boxes, want_counts, _ = amg_crops_ref.layout(x, 2, R)
        assert _np(counts[b]).tolist() == want_counts.tolist()
        pairs += [(b, t, int(c)) for t, c in enumerate(want_counts) if c >= 1]
    assert (_np(counts[:2]) == -1).sum() >= 36 + 70
    idx, cx, cr, edge, _ = ops.crop_gather_batched(xd, rd, boxes, pairs, MARGIN, lengths)
    for p, (b, t, c) in enumerate(pairs):
        w_idx, w_x, _, w_edge = amg_crops_ref.crop_cloud(clouds[b], clouds[b], _np(boxes[b]), t, MARGIN)
        assert _np(idx[p, :c]).tolist() == w_idx.tolist()
        assert np.array_equal(_u32(cx[p, :c]), w_x.view(np.uint32))
        assert np.array_equal(_u32(edge[p, :ops.mask_words(c)]), amg_ref.pack_bits(w_edge[None])[0])


def test_edge_filter_batched_equals_single():
    from psam_b200 import ops

    rng = np.random.default_rng(3)
    T, K, n = 5, 300, 2047
    W = ops.mask_words(n)
    masks = rng.random((T, K, n)) < rng.uniform(0.0005, 0.02, (T, K, 1))
    edges = rng.random((T, n)) < 0.01
    bits = torch.from_numpy(np.stack([amg_ref.pack_bits(m) for m in masks]).view(np.int32)).to(DEV)
    edge = torch.from_numpy(amg_ref.pack_bits(edges).view(np.int32)).to(DEV)
    score = rng.uniform(0, 1, (T, K)).astype(F)
    score[:, ::7] = -np.inf
    got = torch.from_numpy(score).to(DEV)
    ops.crop_edge_filter_batched(bits, got, edge)
    for t in range(T):
        s = torch.from_numpy(score[t].copy()).to(DEV)
        ops.crop_edge_filter(bits[t], s, edge[t])
        assert torch.equal(got[t], s), t
    assert 0 < int((got == -np.inf).sum()) < T * K and W == bits.shape[2]


def _runs(rng, N, specs):
    """Synthetic per-crop states for the uncrop: specs of (crop, layer, n, prompts)."""
    out = []
    for t, layer, n, P in specs:
        idx = np.arange(N) if layer == 0 else np.sort(rng.choice(N, n, replace=False))
        K = 3 * P
        masks = rng.random((K, n)) < rng.uniform(0.001, 0.3, (K, 1))
        masks[:, -1] |= rng.random(K) < 0.5
        keep = rng.permutation(K)[: int(rng.integers(1, K))]
        out.append(dict(crop=t, layer=layer, idx=idx, bits=amg_ref.pack_bits(masks), area=masks.sum(1).astype(np.int32),
                        score=rng.uniform(0, 1, K).astype(F), stability=rng.uniform(0, 1, K).astype(F), keep=keep,
                        point_index=rng.integers(0, n, P).astype(np.int64), slots=3))
    return out


def _dev_run(c, cloud, cap):
    cand = tuple(torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for v in (c["bits"].view(np.int32), c["area"], c["stability"], c["score"]))
    keep = np.zeros(len(c["area"]), np.int32)
    keep[: len(c["keep"])] = c["keep"]
    return dict(cand=cand, keep=torch.from_numpy(keep).to(DEV), keep_count=torch.tensor([len(c["keep"])], dtype=torch.int32, device=DEV),
                idx=torch.from_numpy(c["idx"].astype(np.int32)).to(DEV), prompt_index=torch.from_numpy(c["point_index"]).to(DEV),
                slots=3, crop=c["crop"], layer=c["layer"], cloud=cloud, capacity=cap)


def _out(B, cap, W):
    return (torch.empty((B, cap, W), dtype=torch.int32, device=DEV), torch.empty((B, cap), dtype=torch.int32, device=DEV),
            torch.empty((B, cap), dtype=torch.float32, device=DEV), torch.empty((B, cap), dtype=torch.float32, device=DEV),
            torch.empty((B, cap), dtype=torch.int64, device=DEV), torch.empty((B, cap), dtype=torch.int32, device=DEV),
            torch.empty((B, cap), dtype=torch.int32, device=DEV), torch.full((B, cap), float("-inf"), dtype=torch.float32, device=DEV))


@pytest.mark.parametrize("over", [None, 0, 1])
def test_uncrop_batched_equals_single_at_capacity_and_one_past(over):
    """Two clouds (N_max = 40000, the second of 33000 points): cloud b's capacity is its total kept count, or one less for
    the cloud `over`; only that cloud is flagged, and every cloud's rows equal psam_crop_uncrop over its crops in order."""
    from psam_b200 import ops

    rng = np.random.default_rng(11)
    Ns = [40000, 33000]
    clouds = [_runs(rng, Ns[0], ((0, 0, 40000, 40), (3, 1, 12000, 30), (5, 1, 33, 8), (70, 2, 4100, 20))),
              _runs(rng, Ns[1], ((0, 0, 33000, 24), (2, 1, 9000, 16), (8, 1, 1025, 12)))]
    totals = [sum(len(c["keep"]) for c in cl) for cl in clouds]
    caps = [t - (b == over) for b, t in enumerate(totals)]
    W = ops.mask_words(Ns[0])
    out = _out(2, max(caps), W)
    runs = [_dev_run(c, b, caps[b]) for b, cl in enumerate(clouds) for c in cl]
    lifted, flags = ops.crop_uncrop_batched(runs, out, Ns[0])
    assert _np(lifted).tolist() == totals
    assert _np(flags).tolist() == [int(b == over) for b in range(2)]
    for b, cl in enumerate(clouds):
        single = _out(1, caps[b], W)
        single = tuple(t[0] for t in single)
        offsets = torch.zeros(len(cl) + 1, dtype=torch.int32, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        for k, c in enumerate(cl):
            r = _dev_run(c, b, caps[b])
            ops.crop_uncrop(r["cand"], r["keep"], r["keep_count"], r["idx"], r["prompt_index"], 3, c["crop"], float(c["layer"]), offsets,
                            k, single, flag, Ns[0])
        rows = min(totals[b], caps[b])
        assert int(flag) == int(b == over) and int(offsets[-1]) == totals[b]
        for got, want in zip(out, single):
            assert np.array_equal(_np(got[b, :rows]).view(np.uint8), _np(want[:rows]).view(np.uint8))
        assert np.all(_np(out[7][b, rows:]) == -np.inf)
        m = amg_crops_ref.merge(cl, Ns[0], 0.7, caps[b])  # and the oracle's lifted rows
        assert np.array_equal(_u32(out[0][b, :rows]), m["bits"]) and np.array_equal(_np(out[4][b, :rows]), m["prompt"])


# ------------------------------------------------------------------------------------------------
# 2. the generator
# ------------------------------------------------------------------------------------------------
KW = dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, stability_score_offset=0.05, mask_nms_thresh=0.9)
PROMPTS, BATCH = 32, 12


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


def _clouds(sizes, seed):
    out = [synth.make_batch(1, n, seed + b) for b, n in enumerate(sizes)]
    return [x[0].to(DEV) for x, _ in out], [c[0].to(DEV) for _, c in out]


def _per_crop_np(crops, N):
    per = []
    for c in crops:
        n = int(c["keep_count"].item())
        per.append(dict(crop=c["crop"], layer=c["layer"], idx=_np(c["idx"]).astype(np.int64), bits=_u32(c["bits"]), area=_np(c["area"]),
                        score=_np(c["score"]), stability=_np(c["stability"]), keep=_np(c["keep"])[:n], point_index=_np(c["point_index"]),
                        slots=c["slots"]))
    return per


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


# (points, synth seed) of the three clouds of each case.  IoU / stability filters off; seeds chosen on the CPU oracle so
# that every NMS decision of every crop and of the merge of every cloud has a margin of at least 1e-2 (asserted below), as
# in test_gpu_amg_crops.py.  Emptiness and the edge filter are decided by single logits: checked exactly on the device's
# own masks, and the masks against the oracle's logits.
ORACLE_CLOUDS = {
    ("base", 1): [(2048, 101), (3000, 100), (1500, 100)],
    ("hier", 1): [(2048, 108), (3000, 101), (1500, 101)],
    ("base", 2): [(2048, 101), (3000, 100), (1500, 103)],
    ("hier", 2): [(2048, 108), (3000, 101), (1500, 106)],
}
CROP_NMS = 0.7


def _check_against_oracle(kind, layers, b, crops, lifted, want, N):
    """Cloud b's crops (keep_crop_states) against generate_ref's, crop by crop, then its merge."""
    from psam_b200 import ops

    nt = KW["mask_nms_thresh"]
    margins = [_nms_margin(w["bits"], w["area"], amg_ref.sort_order(w["score"]), nt) for w in want["crops"]]
    merged = want["merged"]
    merge_margin = _nms_margin(merged["bits"], merged["area"], amg_ref.sort_order(merged["layer_score"]), CROP_NMS)
    print(f"[amg crops batch] {kind} L{layers} cloud {b}: {len(want['crops'])} crops, decision margins: crops "
          f"{min(margins):.4g}, merge {merge_margin:.4g}")
    assert min(margins) >= 1e-2 and merge_margin >= 1e-2
    assert [c["crop"] for c in crops] == [c["crop"] for c in want["crops"]]
    kept_deeper = 0
    for c, w in zip(crops, want["crops"]):
        n = int(c["keep_count"].item())
        assert _np(c["idx"]).tolist() == np.asarray(w["idx"]).tolist(), c["crop"]
        P = len(w["point_index"])
        assert _np(c["point_index"])[:P].tolist() == w["point_index"].tolist(), c["crop"]
        # the crop batch may give a crop more slots than its own prompts (a batch's P is the largest): they score -inf
        K, score_all = P * c["slots"], _np(c["score"])
        assert np.all(score_all[K:] == -np.inf), c["crop"]
        words = _u32(c["bits"])[:K]
        full = amg_ref.unpack_bits(words, words.shape[1] * 32)
        assert not full[:, c["points"]:].any(), c["crop"]  # nothing of the padding, whatever the batch's n_max
        seg = full[:, :c["points"]]
        lg = w["logits"].reshape(len(seg), -1)
        diff = seg != (lg > 0)
        assert np.all(np.abs(lg[diff]) < 1e-3), f"crop {c['crop']}: {diff.sum()} points differ"
        assert np.array_equal(_np(c["area"])[:K], seg.sum(1))
        score = score_all[:K]
        valid = score > -np.inf
        np.testing.assert_allclose(score[valid], w["iou"].reshape(-1)[valid], atol=1e-3, rtol=0)
        edge = np.zeros(c["points"], bool) if w["edge"] is None else w["edge"]
        hit = (seg & edge[None]).any(1)
        assert np.array_equal(valid, (seg.sum(1) >= 1) & ~hit), c["crop"]
        keep_c = _np(c["keep"])[:n]
        assert keep_c.tolist() == amg_ref.nms(_u32(c["bits"]), _np(c["area"]), score_all, nt).tolist(), c["crop"]
        assert sorted(w["bits"][k].tobytes() for k in keep_c) == sorted(w["bits"][k].tobytes() for k in w["keep"]), c["crop"]
        kept_deeper += n if c["layer"] else 0
    # the lifted list in crop order and the merge: exactly the oracle merge of this call's own per-crop results, and the
    # same crops kept as the oracle's own run
    m = amg_crops_ref.merge(_per_crop_np(crops, N), N, CROP_NMS, lifted["capacity"])
    L = len(m["area"])
    assert lifted["count"] == L and not m["overflow"]
    Wb = ops.mask_words(N)  # the lifted rows have the words of N_max; the cloud's own come first, the rest are zero
    assert np.array_equal(lifted["bits"][:L, :Wb], m["bits"]) and not lifted["bits"][:L, Wb:].any()
    assert np.array_equal(lifted["crop"][:L], m["crop"]) and np.array_equal(lifted["prompt"][:L], m["prompt"])
    assert lifted["keep"].tolist() == m["keep"].tolist()
    assert sorted(m["crop"][m["keep"]].tolist()) == sorted(merged["crop"][want["final"]].tolist())
    return m, kept_deeper


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("kind", ["base", "hier"])
def test_generator_batch_crops_match_fp32_oracle(kind, layers):
    """Three clouds of different sizes in one call: each against amg_crops_ref.generate_ref crop by crop and through the
    merge, and against generate_packed's crop path bit for bit up to the encoder."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import ops

    model, oracle = _models(kind, 5 if kind == "base" else 9)
    clouds = [synth.make_batch(1, n, seed) for n, seed in ORACLE_CLOUDS[kind, layers]]
    xs, cs = [x[0].to(DEV) for x, _ in clouds], [c[0].to(DEV) for _, c in clouds]
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    crop = dict(crop_n_layers=layers, crop_nms_thresh=CROP_NMS)
    st = gen._enqueue_batch_crops(xs, cs, **crop, keep_crop_states=True)
    outs = gen._finish_batch_crops(st)
    assert len(st["crop_batches"]) >= 1
    for lay, pairs, n_max in st["crop_batches"]:  # one layer per crop batch, at most points_per_batch crops
        assert all(ops.crop_total(lay - 1) <= t < ops.crop_total(lay) for _, t, _ in pairs) and len(pairs) <= BATCH
        assert n_max == max(c for _, _, c in pairs)
    assert any(len({c for _, _, c in pairs}) > 1 for _, pairs, _ in st["crop_batches"])  # crops of different sizes share a batch
    kept_deeper = 0
    for b, ((xc, rc), x, c) in enumerate(zip(clouds, xs, cs)):
        N = x.shape[0]
        want = amg_crops_ref.generate_ref(oracle, xc, rc, PROMPTS, BATCH, **KW, **crop, min_points=model._group_shape()[0])
        assert np.array_equal(_u32(st["crop_boxes"][b]), want["boxes"].view(np.uint32))
        assert _np(st["crop_counts"][b]).tolist() == want["counts"].tolist()
        n_keep = int(st["keep_count"][b])
        lifted = dict(capacity=st["capacity"][b], count=int(st["lifted_count"][b]), bits=_u32(st["bits"][b]), crop=_np(st["crop"][b]),
                      prompt=_np(st["prompt"][b]), keep=_np(st["keep"][b])[:n_keep])
        m, kd = _check_against_oracle(kind, layers, b, st["crops"][b], lifted, want, N)
        kept_deeper += kd
        out = outs[b]
        assert out["bits"].shape[1] == ops.mask_words(N)
        assert np.array_equal(_u32(out["bits"]), m["bits"][m["keep"]])
        assert _np(out["point_index"]).tolist() == m["prompt"][m["keep"]].tolist()
        assert np.array_equal(_np(out["crop_box"]), want["boxes"][m["crop"][m["keep"]]])
        np.testing.assert_array_equal(_np(out["point_coords"]), xc[0].numpy()[m["prompt"][m["keep"]]])
        # generate_packed's crop path on this cloud alone: the same fields and dtypes, the same capacity, and bit for bit
        # the same crops, points, renormalised coordinates, edge bits and prompts
        single = gen._enqueue(x, c, **crop, keep_crop_states=True)
        ref = gen._finish(single)
        assert out.keys() == ref.keys() and all(out[k].dtype == ref[k].dtype for k in out)
        assert st["capacity"][b] == single["bits"].shape[0]
        assert [(k["crop"], k["layer"], k["points"], k["prompts"]) for k in st["crops"][b]] == \
               [(k["crop"], k["layer"], k["points"], k["prompts"]) for k in single["crops"]]
        for got, sw in zip(st["crops"][b], single["crops"]):
            assert torch.equal(got["idx"], sw["idx"]), got["crop"]
            assert torch.equal(got["point_index"][:sw["prompts"]], sw["point_index"]), got["crop"]
            if got["layer"]:
                _, want_x, _, want_edge = ops.crop_gather(x, c, single["crop_boxes"], got["crop"], got["points"], MARGIN)
                assert np.array_equal(_u32(got["xyz"]), _u32(want_x[0])) and torch.equal(got["edge"], want_edge)
    assert kept_deeper > 0
    # records, with crop_box
    recs = gen.generate_batch_crops(xs, cs, **crop)
    assert [len(r) for r in recs] == [o["area"].shape[0] for o in outs]
    assert all(len(r["segmentation"]) == x.shape[0] and len(r["crop_box"]) == 6 for rr, x in zip(recs, xs) for r in rr)


def test_generator_batch_crops_with_regions_equals_oracle_of_its_merge():
    from oracle import amg_regions_ref
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import ops

    model, _ = _models("base", 5)
    xs, cs = _clouds([2048, 2600], 21)
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    st = gen._enqueue_batch_crops(xs, cs, crop_n_layers=1, min_mask_region_area=8, keep_crop_states=True)
    outs = gen._finish_batch_crops(st)
    for b, x in enumerate(xs):
        N = x.shape[0]
        m = amg_crops_ref.merge(_per_crop_np(st["crops"][b], N), N, 0.7, st["capacity"][b])
        nbr = ops.knn(x[None], x[None], amg_regions_ref.REGION_NEIGHBORS + 1)[0][0].cpu().numpy()
        post = amg_regions_ref.postprocess_small_regions(m["bits"], m["keep"], nbr, 8, KW["mask_nms_thresh"])
        assert np.array_equal(_u32(outs[b]["bits"]), post["bits"][post["keep"]][:, :ops.mask_words(N)])
        assert _np(outs[b]["point_index"]).tolist() == m["prompt"][m["keep"][post["keep"]]].tolist()


def test_one_cloud_list_equals_generate_packed_up_to_the_encoder():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model, _ = _models("base", 5)
    xs, cs = _clouds([2048], 5)
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    st = gen._enqueue_batch_crops(xs, cs, crop_n_layers=2, keep_crop_states=True)
    single = gen._enqueue(xs[0], cs[0], crop_n_layers=2, keep_crop_states=True)
    assert np.array_equal(_u32(st["crop_boxes"][0]), _u32(single["crop_boxes"]))
    assert len(st["crops"][0]) == len(single["crops"])
    for got, want in zip(st["crops"][0], single["crops"]):
        assert got["crop"] == want["crop"] and torch.equal(got["idx"], want["idx"])
        assert torch.equal(got["point_index"][: want["prompts"]], want["point_index"])
    a, b = gen._finish_batch_crops(st)[0], gen._finish(single)
    assert a.keys() == b.keys()


def test_cloud_without_layer1_crops_skips_the_merge_next_to_clouds_with_crops():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model, _ = _models("base", 5)
    # 70 points: every layer-1 crop holds fewer than the 64 first-level groups, so only layer 0 runs on that cloud
    xs, cs = _clouds([2048, 70, 1800], 31)
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    ct = 0.05  # a merge threshold that would drop most of a layer-0-only cloud's masks
    st = gen._enqueue_batch_crops(xs, cs, crop_n_layers=1, crop_nms_thresh=ct, keep_crop_states=True)
    outs = gen._finish_batch_crops(st)
    assert [len(c) for c in st["crops"]][1] == 1 and len(st["crops"][0]) > 1 and len(st["crops"][2]) > 1
    single = gen._enqueue(xs[1], cs[1], crop_n_layers=1, crop_nms_thresh=ct, keep_crop_states=True)
    ref = gen._finish(single)
    L = int(st["lifted_count"][1])
    assert _np(st["keep"][1])[: int(st["keep_count"][1])].tolist() == list(range(L))  # every lifted mask, in order
    assert outs[1]["area"].shape[0] == L == ref["area"].shape[0]
    assert _np(outs[1]["point_index"]).tolist() == _np(ref["point_index"]).tolist()
    nms = amg_ref.nms(_u32(st["bits"][1, :L]), _np(st["area"][1, :L]), _np(st["crop_score"][1, :L]), ct)
    assert len(nms) < L  # running the merge there would have dropped masks


def test_batch_crops_synchronise_twice():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model, _ = _models("base", 5)
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    for B in (1, 4):
        xs, cs = _clouds([2048, 1500, 3000, 2500][:B], 7)
        first = gen.generate_packed_batch_crops(xs, cs, crop_n_layers=2)
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                got = gen.generate_packed_batch_crops(xs, cs, crop_n_layers=2)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        syncs = [w for w in caught if "called a synchronizing" in str(w.message)]
        assert len(syncs) == 2, (B, [str(w.message) for w in caught])
        for a, b in zip(first, got):
            assert torch.equal(a["crop_box"], b["crop_box"]) and a["bits"].shape[1] == b["bits"].shape[1]


def test_batch_crops_overflow_names_the_cloud():
    """A real overflow: cloud 0 (8000 points, 5400 prompts, IoU / stability / NMS filters off and no edge margin) keeps more
    masks over its crops than the 16384 lifted slots; cloud 1 (300 points) stays within its own capacity.  Only cloud 0 is
    flagged, and the final read names it."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import ops

    model, _ = _models("base", 5)
    xs, cs = _clouds([8000, 300], 41)
    gen = PointCloudMaskGenerator(model, points_per_cloud=5400, points_per_batch=128, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  mask_nms_thresh=1.0)
    gen.crop_edge_margin = 0.0
    st = gen._enqueue_batch_crops(xs, cs, crop_n_layers=1)
    caps, lifted = st["capacity"], _np(st["lifted_count"]).tolist()
    print(f"[amg crops batch] overflow: capacities {caps}, lifted {lifted}")
    assert caps[0] == ops.NMS_MAX_CANDIDATES and caps[1] < caps[0]
    assert lifted[0] > caps[0] and lifted[1] <= caps[1]
    assert _np(st["overflow"]).tolist() == [1, 0]
    with pytest.raises(ValueError, match="cloud 0"):
        gen._finish_batch_crops(st)


def test_batch_crops_refuse_out_of_range_clouds():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model, _ = _models("base", 5)
    xs, cs = _clouds([2048, 1500], 7)
    gen = PointCloudMaskGenerator(model, points_per_cloud=PROMPTS, points_per_batch=BATCH, **KW)
    with pytest.raises(ValueError, match="normalized"):
        gen.generate_packed_batch_crops([xs[0], xs[1] * 3], cs)
    gen.generate_packed_batch_crops(xs, cs)  # the flag was reset


def test_zero_layers_is_generate_packed_batch():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import native

    model, _ = _models("base", 5)
    xs, cs = _clouds([2048, 1500, 1900], 3)
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=16, **KW)
    gen.generate_packed_batch(xs, cs)  # packs the weights
    n0 = native.LAUNCHES[0]
    gen.generate_packed_batch(xs, cs, min_mask_region_area=4)
    n1 = native.LAUNCHES[0]
    gen.generate_packed_batch_crops(xs, cs, crop_n_layers=0, crop_nms_thresh=0.1, min_mask_region_area=4)
    assert native.LAUNCHES[0] - n1 == n1 - n0  # the same launches
    # the same results.  The encoder's float atomics can move a logit by about 1e-5 from one run to the next, so both calls
    # decode one encoder output: the second call reuses the first call's encode of the same padded batch.
    real, memo = model._encode, []

    def encode_once(coords, features, lengths=None):
        for c, f, n, out in memo:
            if torch.equal(c, coords) and torch.equal(f, features) and torch.equal(n, lengths):
                return out
        out = real(coords, features, lengths)
        memo.append((coords.clone(), features.clone(), lengths.clone(), out))
        return out

    model._encode = encode_once
    try:
        a = gen.generate_packed_batch(xs, cs, min_mask_region_area=4)
        b = gen.generate_packed_batch_crops(xs, cs, crop_n_layers=0, crop_nms_thresh=0.1, min_mask_region_area=4)
    finally:
        del model._encode
    assert len(memo) == 1
    for x, y in zip(a, b):
        assert x.keys() == y.keys() and "crop_box" not in y
        for k in ("bits", "area", "point_index", "point_coords", "mask_slot"):
            assert torch.equal(x[k], y[k]), k
        for k in ("predicted_iou", "stability_score"):  # the decoder's fp32 reductions may round differently from run to run
            torch.testing.assert_close(x[k], y[k], atol=1e-5, rtol=0)


# ------------------------------------------------------------------------------------------------
# 3. full size, once
# ------------------------------------------------------------------------------------------------
def test_batch_crops_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    xs, cs = [], []
    for b, n in enumerate((131072, 127000)):
        x, c = synth.make_batch(1, n, 3 + b, "kitti")
        xs.append(x[0].to(DEV))
        cs.append(c[0].to(DEV))
    ct = 0.7
    gen = PointCloudMaskGenerator(model, points_per_cloud=1024, points_per_batch=32, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05)
    st = gen._enqueue_batch_crops(xs, cs, crop_n_layers=1, crop_nms_thresh=ct)
    outs = gen._finish_batch_crops(st)
    for b, (x, out) in enumerate(zip(xs, outs)):
        N = x.shape[0]
        boxes = _np(st["crop_boxes"][b])
        crop = _np(st["crop"][b])[_np(st["keep"][b])[: out["area"].shape[0]]]
        print(f"[amg crops batch] full size cloud {b}: {len(st['crops'][b])} crops, {int(st['lifted_count'][b])} lifted, {len(crop)} kept, "
              f"{int((crop > 0).sum())} from layer 1")
        assert len(st["crops"][b]) > 1 and (crop > 0).any() and (crop == 0).any()
        m = torch.from_numpy(amg_ref.unpack_bits(_u32(out["bits"]), N)).to(DEV).float()
        inter = (m @ m.T).round().long().cpu().numpy()
        area = _np(out["area"]).astype(np.int64)
        assert np.array_equal(np.diag(inter), area)
        iou = inter.astype(F) / (area[:, None] + area[None, :] - inter).astype(F)
        np.fill_diagonal(iou, 0)
        assert iou.max() <= ct
        xn = x.cpu().numpy()
        seg = m.bool().cpu().numpy()
        for t in np.unique(crop[crop > 0]):
            idx, _, _, edge = amg_crops_ref.crop_cloud(xn, xn, boxes, int(t))
            g = np.zeros(N, bool)
            g[idx[edge]] = True
            assert not (seg[crop == t] & g[None]).any(), t
