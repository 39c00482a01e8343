"""GPU tests of automatic mask generation on a batch of clouds: the batched candidate, NMS and small-region launches equal
the numpy oracles per cloud and the single-cloud kernels on each cloud's slice, bit for bit; B = 1 is the single-cloud
path; B clouds per call match the fp32 oracle end to end (PointCloudSAM and PointCloudSAMHier, with and without
min_mask_region_area); the call synchronises with the host once; and it holds at full size (ViT-L, 4 x 32768 points)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_ref, amg_regions_ref, hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
K1 = amg_regions_ref.REGION_NEIGHBORS + 1
RULES = dict(mask_threshold=0.0, stability_offset=1.0, pred_iou_thresh=0.88, stability_thresh=0.5, min_area=3)


# ------------------------------------------------------------------------------------------------
# 1. candidates and NMS on synthetic logits
# ------------------------------------------------------------------------------------------------
def _synthetic(Z, N, seed):
    """Z x 3 candidate rows (test_gpu_amg.py's): overlapping interval-shaped masks with near and exact duplicates, empty
    rows, logits exactly on the thresholds (0, +-offset) and predicted IoUs with ties and values exactly on
    pred_iou_thresh.  Returns logits [Z, 3, N], iou [Z, 3]."""
    K = 3 * Z
    rng = np.random.default_rng(seed)
    n = np.arange(N, dtype=np.float32)
    protos = max(2, K // 6)
    c = rng.uniform(0, N, protos).astype(np.float32)
    w = rng.uniform(0.05, 0.5, protos).astype(np.float32) * N
    p = rng.integers(0, protos, K)
    lg = (w[p, None] - np.abs(n[None, :] - c[p, None])) / np.float32(max(N / 16, 1)) + rng.normal(0, 0.3, (K, N))
    lg = lg.astype(np.float32)
    lg[rng.random((K, N)) < 0.02] = 0.0
    lg[rng.random((K, N)) < 0.02] = 1.0
    lg[rng.random((K, N)) < 0.02] = -1.0
    if K > 4:
        lg[1] = lg[0]
        lg[4] = -2.0
    if K > 8 and N >= 40:  # stability exactly 0.5 = stability_thresh
        lg[8] = -2.0
        lg[8, :20] = 2.0
        lg[8, 20:40] = 0.5
    iou = rng.choice(np.float32([0.5, 0.8, 0.88, 0.9, 0.95, 0.97]), size=K).astype(np.float32)
    iou[1::5] = np.float32(0.88)
    if K > 8:
        iou[8] = np.float32(0.99)
    return lg.reshape(Z, 3, N), iou.reshape(Z, 3)


def _batch_rows(per_cloud, s, e):
    """Rows [s, e) of every cloud in the decoder's layout: row b * (e - s) + j is row s + j of cloud b."""
    return torch.from_numpy(np.concatenate([x[s:e] for x in per_cloud])).to(DEV)


def _alloc(B, K, N):
    from psam_b200 import ops

    return (torch.empty((B, K, ops.mask_words(N)), dtype=torch.int32, device=DEV), torch.empty((B, K), dtype=torch.int32, device=DEV),
            torch.empty((B, K), dtype=torch.float32, device=DEV), torch.empty((B, K), dtype=torch.float32, device=DEV))


@pytest.mark.parametrize("B,N,Z,chunk,empty", [(1, 2048, 64, 64, None), (3, 33, 5461, 2000, 1), (5, 2047, 100, 37, 4),
                                                (3, 2048, 21, 8, 0), (3, 32768, 8, 3, 2), (5, 33, 40, 40, None)])
def test_candidates_and_nms_match_oracle_per_cloud(B, N, Z, chunk, empty):
    """B clouds of Z prompts (K = 3Z slots each) in decode chunks of `chunk` prompts per cloud (the last one short); cloud
    `empty` has no valid candidate.  K = 16383 at Z = 5461."""
    from psam_b200 import ops

    C, K = 3, 3 * Z
    data = [_synthetic(Z, N, 1000 * b + N + Z) for b in range(B)]
    if empty is not None:
        data[empty][1][:] = np.float32(np.nan)  # a NaN predicted IoU is never kept
    lgs, ious = [d[0] for d in data], [d[1] for d in data]
    cand = _alloc(B, K, N)
    for s in range(0, Z, chunk):
        e = min(Z, s + chunk)
        ops.mask_candidates_batched(_batch_rows(lgs, s, e), _batch_rows(ious, s, e), B, out=cand, base=s * C, **RULES)
    for nt in (0.7, 1.0):
        keep, cnt = ops.mask_nms_batched(cand[0], cand[1], cand[3], nt)
        torch.cuda.synchronize()
        counts = cnt.cpu().numpy()
        for b in range(B):
            want = amg_ref.candidates(lgs[b], ious[b], **RULES)
            bits, area, stab, score = (t[b].cpu().numpy() for t in cand)
            assert np.array_equal(bits.view(np.uint32), want["bits"]), b
            assert np.array_equal(area, want["area"])
            np.testing.assert_array_equal(stab, want["stability"])
            np.testing.assert_array_equal(score, want["score"])
            want_keep = amg_ref.nms(want["bits"], want["area"], want["score"], nt)
            assert keep[b, : counts[b]].cpu().numpy().tolist() == want_keep.tolist(), (b, nt)
            if b == empty:
                assert counts[b] == 0
            # the single-cloud kernels on the cloud's own rows and slice
            one = ops.mask_candidates(torch.from_numpy(lgs[b]).to(DEV), torch.from_numpy(ious[b]).to(DEV), **RULES)
            for t1, tb in zip(one, cand):
                assert torch.equal(t1.view(torch.int32), tb[b].view(torch.int32))
            k1, c1 = ops.mask_nms(cand[0][b], cand[1][b], cand[3][b], nt)
            assert int(c1.item()) == counts[b] and torch.equal(k1[: counts[b]], keep[b, : counts[b]])
    assert sum(int((amg_ref.candidates(lgs[b], ious[b], **RULES)["score"] > -np.inf).sum()) for b in range(B)) > 0


def test_nms_batched_without_candidates():
    from psam_b200 import ops

    e = torch.empty((3, 0, 1), dtype=torch.int32, device=DEV)
    keep, cnt = ops.mask_nms_batched(e, e[..., 0], e[..., 0].float(), 0.7)
    assert cnt.tolist() == [0, 0, 0]


# ------------------------------------------------------------------------------------------------
# 2. small-region stage
# ------------------------------------------------------------------------------------------------
def _cloud(N, seed):
    """test_gpu_amg_regions.py's synthetic cloud: separated Gaussian blobs, points on line segments and coincident
    duplicates.  Returns xyz [N, 3] fp32 and a part label per point."""
    rng = np.random.default_rng(seed)
    nb, nl = 10, 3
    centers = rng.uniform(-0.8, 0.8, (nb, 3))
    n_line, n_dup = N // 8, N // 16
    n_blob = N - n_line - n_dup
    lab_b = rng.integers(0, nb, n_blob)
    pb = centers[lab_b] + rng.normal(0, 1, (n_blob, 3)) * rng.uniform(0.01, 0.06, nb)[lab_b, None]
    lab_l = rng.integers(0, nl, n_line)
    ends = rng.uniform(-0.9, 0.9, (nl, 2, 3))
    t = rng.random((n_line, 1))
    pl = ends[lab_l, 0] * (1 - t) + ends[lab_l, 1] * t
    xyz = np.concatenate([pb, pl]).astype(np.float32)
    lab = np.concatenate([lab_b, nb + lab_l])
    src = rng.integers(0, len(xyz), n_dup)
    xyz, lab = np.concatenate([xyz, xyz[src]]), np.concatenate([lab, lab[src]])
    perm = rng.permutation(N)
    return np.clip(xyz[perm], -1, 1), lab[perm]


def _masks(xyz, lab, S, seed):
    """S masks: unions of parts with stray points and punched holes; slot 0 the whole cloud, the last two a five-point and
    a one-point mask."""
    rng = np.random.default_rng(seed)
    N = len(lab)
    parts = int(lab.max()) + 1
    out = np.zeros((S, N), bool)
    for s in range(S):
        m = np.isin(lab, rng.choice(parts, int(rng.integers(1, 4)), replace=False))
        m[rng.integers(0, N, int(rng.integers(0, 6)))] = True
        if m.any() and rng.random() < 0.7:
            c = xyz[rng.choice(np.nonzero(m)[0])]
            r = rng.uniform(0.005, 0.05)
            m &= ((xyz - c) ** 2).sum(1) > r * r
        m[rng.integers(0, N, int(rng.integers(0, 6)))] = False
        out[s] = m
    out[0] = True
    out[S - 2] = False
    out[S - 2, rng.integers(0, N, 5)] = True
    out[S - 1] = False
    out[S - 1, rng.integers(0, N)] = True
    out[out.sum(1) == 0, 0] = True
    return out


@pytest.mark.parametrize("B,N", [(3, 2047), (4, 32768), (3, 65536)])
def test_regions_match_oracle_per_cloud(B, N):
    """Both label stores: shared memory (N <= 49152) and workspace slices shared by the launch (N > 49152).  Every cloud
    has its own cloud, masks, keep subset and count (one cloud keeps nothing)."""
    from psam_b200 import ops

    S = 10 if N <= 32768 else 6
    Kk = S - 2  # keep entries per cloud
    clouds = [_cloud(N, N + 17 * b) for b in range(B)]
    xyz_d = torch.from_numpy(np.stack([c[0] for c in clouds])).to(DEV)
    nbr_d, _ = ops.knn(xyz_d, xyz_d, K1)
    W = ops.mask_words(N)
    bits = np.stack([amg_ref.pack_bits(_masks(x, l, S, N + 31 * b), W) for b, (x, l) in enumerate(clouds)])
    rng = np.random.default_rng(N)
    keep = np.stack([rng.permutation(S)[:Kk] for _ in range(B)]).astype(np.int32)  # unsorted subsets of the slots
    counts = np.array([Kk, 0] + [int(rng.integers(1, Kk + 1)) for _ in range(B - 2)], dtype=np.int32)
    bits_d = torch.from_numpy(bits.view(np.int32)).to(DEV)
    keep_d, cnt_d = torch.from_numpy(keep).to(DEV), torch.from_numpy(counts).to(DEV)
    nt = 0.7
    changed = 0
    for A in (4, max(4, N // 4)):
        rb, ra, rs = ops.mask_regions_batched(bits_d, keep_d, cnt_d, nbr_d, A)
        keep2, c2 = ops.mask_nms_batched(rb, ra, rs, nt)
        torch.cuda.synchronize()
        c2 = c2.cpu().numpy()
        for b in range(B):
            n = counts[b]
            want = amg_regions_ref.postprocess_small_regions(bits[b], keep[b, :n], nbr_d[b].cpu().numpy(), A, nt)
            assert np.array_equal(rb[b, :n].cpu().numpy().view(np.uint32), want["bits"]), (A, b)
            assert np.array_equal(ra[b, :n].cpu().numpy(), want["area"])
            assert np.array_equal(rs[b, :n].cpu().numpy(), want["score"])
            assert np.all(rs[b, n:].cpu().numpy() == -np.inf)
            assert keep2[b, : c2[b]].cpu().numpy().tolist() == want["keep"].tolist()
            changed += int((want["score"] == 0).sum())
            # the single-cloud launch on the cloud's own slice
            sb, sa, ss = ops.mask_regions(bits_d[b], keep_d[b], cnt_d[b:b + 1], nbr_d[b], A)
            assert torch.equal(sb[:n], rb[b, :n]) and torch.equal(sa[:n], ra[b, :n]) and torch.equal(ss, rs[b])
    assert changed >= 2


# ------------------------------------------------------------------------------------------------
# 3-5. the generator
# ------------------------------------------------------------------------------------------------
# test_gpu_amg.py's model fixtures with three clouds each, seeds chosen on the CPU oracle so that every filter and NMS
# decision of every cloud has a margin >= 1e-2 (valid scores >= 2e-3 apart)
FIXTURES = {
    "base": dict(seed=5, clouds=(5, 6, 49), kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.475, stability_score_offset=0.02,
                                                   mask_nms_thresh=0.9)),
    "hier": dict(seed=8, clouds=(26, 32, 36), kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.55, stability_score_offset=0.05,
                                                   mask_nms_thresh=0.9)),
}
N_E2E, AREA = 2048, 8


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


def _clouds(seeds, N=N_E2E):
    xs, rs = zip(*[synth.make_batch(1, N, s) for s in seeds])
    return torch.cat(xs), torch.cat(rs)


def _margins(want, st, nt):
    io, stab, area = want["iou"].ravel(), want["stability"], want["area"]
    fm = min((abs(stab[k] - np.float32(st)) if not np.isnan(stab[k]) else np.inf) for k in range(len(io)) if area[k] >= 1)
    order = amg_ref.sort_order(want["score"])
    sc = want["score"][order]
    P = amg_ref.pair_ious(want["bits"], area, order)
    nm, kept = [], []
    for j in range(len(order)):
        ious = P[kept, j]
        sup = ious[ious > nt]
        nm.append((sup - nt).max() if len(sup) else (nt - ious).min() if len(ious) else np.inf)
        if not len(sup):
            kept.append(j)
    return fm, min(nm), (np.diff(-sc).min() if len(sc) > 1 else np.inf), len(order), len(kept)


def _pairs(out):
    return list(zip(out["point_index"].tolist(), out["mask_slot"].tolist()))


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_batch_matches_fp32_oracle_per_cloud(kind):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES[kind]
    model, oracle = _models(kind, fx["seed"])
    xyz, rgb = _clouds(fx["clouds"])
    nt = fx["kw"]["mask_nms_thresh"]
    wants = []
    for b in range(len(fx["clouds"])):
        want = amg_regions_ref.generate_ref(oracle, xyz[b:b + 1], rgb[b:b + 1], 64, 64, **fx["kw"], min_mask_region_area=AREA)
        fm, nm, gap, valid, kept = _margins(want, fx["kw"]["stability_score_thresh"], nt)
        print(f"[amg batch] {kind} cloud {b}: valid {valid} kept {kept}; margins filter {fm:.3g} nms {nm:.3g} gap {gap:.3g}")
        assert fm >= 1e-2 and nm >= 1e-2 and gap >= 2e-3 and kept >= 1
        wants.append(want)
    # 64 prompts per cloud, 24 rows per decode batch: 8 prompts of each of the 3 clouds per batch, 8 batches
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])
    outs = gen.generate_packed_batch(xyz.to(DEV), rgb.to(DEV))
    assert len(outs) == len(wants)
    for b, (got, want) in enumerate(zip(outs, wants)):
        C = want["slots"]
        assert _pairs(got) == [(int(want["point_index"][k // C]), int(k % C)) for k in want["keep"]], b
        np.testing.assert_allclose(got["predicted_iou"].cpu().numpy(), want["iou"].reshape(-1)[want["keep"]], atol=1e-3, rtol=0)
        seg = amg_ref.unpack_bits(got["bits"].cpu().numpy().view(np.uint32), N_E2E)
        lg = want["logits"].reshape(-1, N_E2E)[want["keep"]]
        diff = seg != (lg > 0)
        assert np.all(np.abs(lg[diff]) < 1e-3), f"cloud {b}: {diff.sum()} points differ"
        assert np.array_equal(got["area"].cpu().numpy(), seg.sum(1))
        np.testing.assert_array_equal(got["point_coords"].cpu().numpy(), xyz[b].numpy()[got["point_index"].cpu().numpy()])
        assert got["bits"].dtype == torch.int32 and got["point_index"].dtype == torch.int64 and got["mask_slot"].dtype == torch.int64
    recs = gen.generate_batch(xyz.to(DEV), rgb.to(DEV))
    assert [[r["point_index"] for r in rb] for rb in recs] == [[p for p, _ in _pairs(o)] for o in outs]
    assert all(r["segmentation"].shape == (N_E2E,) for rb in recs for r in rb)
    # with the small-region stage: the device's first-stage masks are the oracle's up to logits within 1e-3 of the
    # threshold, so the stage is checked exactly on the device's own kept masks, and against the oracle's run where the
    # first-stage masks agree bit for bit
    st = gen._enqueue_batch(xyz.to(DEV), rgb.to(DEV), min_mask_region_area=AREA)
    got_r = gen._finish_batch(st)
    from psam_b200 import ops

    nbr = ops.knn(xyz.to(DEV), xyz.to(DEV), K1)[0].cpu().numpy()
    exact = 0
    for b, (got, want) in enumerate(zip(got_r, wants)):
        n = int(st["keep_count"][b].item())
        keep = st["keep"][b, :n].cpu().numpy()
        assert keep.tolist() == want["keep"].tolist(), b
        bits = st["bits"][b].cpu().numpy().view(np.uint32)
        post = amg_regions_ref.postprocess_small_regions(bits, keep, nbr[b], AREA, nt)
        assert np.array_equal(got["bits"].cpu().numpy().view(np.uint32), post["bits"][post["keep"]]), b
        assert np.array_equal(got["area"].cpu().numpy(), post["area"][post["keep"]])
        C = want["slots"]
        assert _pairs(got) == [(int(want["point_index"][k // C]), int(k % C)) for k in keep[post["keep"]]]
        if np.array_equal(bits[keep], want["bits"][want["keep"]]):
            exact += 1
            assert np.array_equal(post["bits"], want["regions"]["bits"])
            assert _pairs(got) == [(int(want["point_index"][k // C]), int(k % C)) for k in want["final_slots"]]
    print(f"[amg batch] {kind}: first-stage masks equal to the oracle's on {exact} of {len(wants)} clouds")
    assert exact >= 1


@pytest.mark.parametrize("area", [0, AREA])
def test_one_cloud_batch_is_the_single_cloud_path(area):
    """generate_packed_batch(xyz[None], rgb[None])[0] equals generate_packed(xyz, rgb) bit for bit in every field.  Both
    calls get the same model outputs (the first call's encode and decode results are replayed to the second, which must
    ask for them with the same inputs), because the encoder's split-K reductions may round differently from run to run."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from psam_b200 import native

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t[0].to(DEV) for t in synth.make_batch(1, N_E2E, fx["seed"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])
    gen.generate_packed(xyz, rgb)  # packs the weights
    enc_fn, dec_fn, log, model_launches = model._encode, model._decode_unchecked, [], [0]

    def record_encode(*a):
        n = native.LAUNCHES[0]
        log.append(("enc", [t.clone() for t in a], enc_fn(*a)))
        model_launches[0] += native.LAUNCHES[0] - n
        return log[-1][2]

    def record_decode(enc, coords, labels, masks, multi):
        n = native.LAUNCHES[0]
        log.append(("dec", [coords.clone(), labels.clone()], dec_fn(enc, coords, labels, masks, multi)))
        model_launches[0] += native.LAUNCHES[0] - n
        return log[-1][2]

    replay = iter(())

    def replay_call(kind):
        def fn(*a):
            k, args, out = next(replay)
            assert k == kind
            mine = [a[0], a[1]] if kind == "enc" else [a[1], a[2]]
            assert all(torch.equal(x, y) for x, y in zip(mine, args))
            return out
        return fn

    try:
        model._encode, model._decode_unchecked = record_encode, record_decode
        n0 = native.LAUNCHES[0]
        one = gen.generate_packed(xyz, rgb, min_mask_region_area=area)
        n1 = native.LAUNCHES[0]
        replay = iter(log)
        model._encode, model._decode_unchecked = replay_call("enc"), replay_call("dec")
        (bat,) = gen.generate_packed_batch(xyz[None], rgb[None], min_mask_region_area=area)
        n2 = native.LAUNCHES[0]
        assert next(replay, None) is None  # the same encode and decode calls
    finally:
        del model._encode, model._decode_unchecked
    assert n2 - n1 == n1 - n0 - model_launches[0] and model_launches[0] > 0  # the same launches besides the model's
    assert list(one.keys()) == list(bat.keys())
    for k in one:
        assert one[k].dtype == bat[k].dtype and torch.equal(one[k], bat[k]), k
    assert one["area"].shape[0] >= 1


def test_batch_enqueues_without_host_sync_and_checks_range():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t.to(DEV) for t in _clouds(fx["clouds"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=16, **fx["kw"])
    first = gen.generate_packed_batch(xyz, rgb, min_mask_region_area=AREA)  # packs the weights
    torch.cuda.synchronize()
    for area in (0, AREA):
        torch.cuda.set_sync_debug_mode("error")
        try:
            st = gen._enqueue_batch(xyz, rgb, min_mask_region_area=area)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        got = gen._finish_batch(st)
        assert len(got) == 3
    assert [g["area"].shape[0] for g in got] == [f["area"].shape[0] for f in first]
    bad = xyz.clone()
    bad[1] *= 1.5  # one cloud's FPS prompt points outside [-1, 1]
    with pytest.raises(ValueError):
        gen.generate_packed_batch(bad, rgb)
    again = gen.generate_packed_batch(xyz, rgb, min_mask_region_area=AREA)  # the flag was reset
    assert [g["area"].shape[0] for g in again] == [f["area"].shape[0] for f in first]


# ------------------------------------------------------------------------------------------------
# 6. full size, once
# ------------------------------------------------------------------------------------------------
def test_batch_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    B, N, P, Bp, nt = 4, 32768, 1024, 64, 0.7
    xyz, rgb = (t.to(DEV) for t in synth.make_batch(B, N, 3))
    gen = PointCloudMaskGenerator(model, points_per_cloud=P, points_per_batch=Bp, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05, mask_nms_thresh=nt)
    # keep the batched path's own logits: every decode batch holds 16 prompts of each of the 4 clouds
    dec_fn, logits = model._decode_unchecked, []

    def keep_logits(*a):
        m, i = dec_fn(*a)
        logits.append((m.cpu().numpy(), i.cpu().numpy()))
        return m, i

    model._decode_unchecked = keep_logits
    try:
        st = gen._enqueue_batch(xyz, rgb)
        outs = gen._finish_batch(st)
    finally:
        del model._decode_unchecked
    Zc = Bp // B
    assert len(logits) == P // Zc
    counts = st["keep_count"].cpu().numpy()
    for b in range(B):
        lg = np.concatenate([m.reshape(B, Zc, 3, N)[b] for m, _ in logits])
        io = np.concatenate([i.reshape(B, Zc, 3)[b] for _, i in logits])
        rules = dict(mask_threshold=0.0, stability_offset=0.05, pred_iou_thresh=0.0, stability_thresh=0.0, min_area=0)
        want = amg_ref.candidates(lg, io, **rules)
        assert np.array_equal(st["bits"][b].cpu().numpy().view(np.uint32), want["bits"]), b
        assert np.array_equal(st["area"][b].cpu().numpy(), want["area"])
        np.testing.assert_array_equal(st["stability"][b].cpu().numpy(), want["stability"])
        np.testing.assert_array_equal(st["score"][b].cpu().numpy(), want["score"])
        want_keep = amg_ref.nms(want["bits"], want["area"], want["score"], nt)
        assert st["keep"][b, : counts[b]].cpu().numpy().tolist() == want_keep.tolist(), b
        out = outs[b]
        bits, area, sc = out["bits"].cpu().numpy().view(np.uint32), out["area"].cpu().numpy(), out["predicted_iou"].cpu().numpy()
        print(f"[amg batch] full size cloud {b}: {int((want['score'] > -np.inf).sum())} valid, {len(sc)} kept")
        assert len(sc) >= 1 and np.all(np.diff(sc) <= 0)
        if len(sc) > 1:
            iou = amg_ref.pair_ious(bits, area, np.arange(len(sc)))
            np.fill_diagonal(iou, 0)
            assert iou.max() <= nt
