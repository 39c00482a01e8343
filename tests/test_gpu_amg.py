"""GPU tests of automatic mask generation: the candidate and NMS kernels equal the numpy oracle exactly, the generator
matches the fp32 oracle end to end (PointCloudSAM and PointCloudSAMHier), it enqueues without host synchronisation, and it
holds at full size (ViT-L, N = 32768, 1024 prompts)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_ref, hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------
# 1. kernel exactness on synthetic logits
# ------------------------------------------------------------------------------------------------
def _synthetic(K, N, seed):
    """K = Z*3 candidate rows: overlapping interval-shaped masks with near and exact duplicates, empty rows, logits exactly
    on the thresholds (0, +-offset) and predicted IoUs with ties and values exactly on pred_iou_thresh."""
    rng = np.random.default_rng(seed)
    n = np.arange(N, dtype=np.float32)
    protos = max(2, K // 6)
    c = rng.uniform(0, N, protos).astype(np.float32)
    w = rng.uniform(0.05, 0.5, protos).astype(np.float32) * N
    p = rng.integers(0, protos, K)
    lg = (w[p, None] - np.abs(n[None, :] - c[p, None])) / np.float32(max(N / 16, 1)) + rng.normal(0, 0.3, (K, N))
    lg = lg.astype(np.float32)
    lg[rng.random((K, N)) < 0.02] = 0.0          # exactly on the mask threshold (not in the mask)
    lg[rng.random((K, N)) < 0.02] = 1.0          # exactly on +offset (not counted)
    lg[rng.random((K, N)) < 0.02] = -1.0         # exactly on -offset (not counted)
    if K > 4:
        lg[1] = lg[0]                            # identical masks
        lg[4] = -2.0                             # empty mask
    if K > 8 and N >= 40:                        # stability exactly 0.5 = stability_thresh: 20 points > 1, 40 points > -1
        lg[8] = -2.0
        lg[8, :20] = 2.0
        lg[8, 20:40] = 0.5
    iou = rng.choice(np.float32([0.5, 0.8, 0.88, 0.9, 0.95, 0.97]), size=K).astype(np.float32)
    iou[1::5] = np.float32(0.88)                 # exactly on pred_iou_thresh: dropped (> is strict)
    if K > 8:
        iou[8] = np.float32(0.99)
    return lg.reshape(-1, 3, N) if K % 3 == 0 else lg.reshape(K, 1, N), iou.reshape(K // (3 if K % 3 == 0 else 1), -1)


RULES = dict(mask_threshold=0.0, stability_offset=1.0, pred_iou_thresh=0.88, stability_thresh=0.5, min_area=3)


def _run_kernels(lg, iou, nms_thresh, chunk=None):
    from psam_b200 import ops

    Z, C, N = lg.shape
    K = Z * C
    out = (torch.empty((K, ops.mask_words(N)), dtype=torch.int32, device=DEV), torch.empty(K, dtype=torch.int32, device=DEV),
           torch.empty(K, dtype=torch.float32, device=DEV), torch.empty(K, dtype=torch.float32, device=DEV))
    lgd, iod = torch.from_numpy(lg).to(DEV), torch.from_numpy(iou).to(DEV)
    chunk = chunk or Z
    for s in range(0, Z, chunk):
        ops.mask_candidates(lgd[s:s + chunk], iod[s:s + chunk], out=out, base=s * C, **RULES)
    keep, cnt = ops.mask_nms(*out[0:2], out[3], nms_thresh)
    torch.cuda.synchronize()
    n = int(cnt.item())
    return [t.cpu().numpy() for t in out], keep[:n].cpu().numpy()


def _check_exact(lg, iou, nms_thresh, chunk=None):
    (bits, area, stab, score), keep = _run_kernels(lg, iou, nms_thresh, chunk)
    want = amg_ref.candidates(lg, iou, **{k: RULES[k] for k in RULES})
    assert np.array_equal(bits.view(np.uint32), want["bits"])
    assert np.array_equal(area, want["area"])
    np.testing.assert_array_equal(stab, want["stability"])  # NaN (0/0) positions included
    np.testing.assert_array_equal(score, want["score"])
    want_keep = amg_ref.nms(want["bits"], want["area"], want["score"], nms_thresh)
    assert keep.tolist() == want_keep.tolist()
    return want, keep


@pytest.mark.parametrize("N,K", [(33, 1), (33, 63), (2047, 64), (2048, 65), (32768, 3), (2047, 3072), (33, 16384)])
def test_kernels_match_oracle_exactly(N, K):
    lg, iou = _synthetic(K, N, N + K)
    for thr in (0.7, 1.0):
        want, keep = _check_exact(lg, iou, thr, chunk=max(1, lg.shape[0] // 3))
        if thr == 1.0:  # nothing suppressed
            assert keep.tolist() == amg_ref.sort_order(want["score"]).tolist()
    if K >= 9 and N >= 40:
        assert want["stability"][8] == np.float32(0.5) and want["score"][8] == np.float32(0.99)


def test_kernels_full_nms_width_and_empty():
    """K = 16383 candidates over N = 2048 (nearly all pairwise tiles run), and K = 0."""
    from psam_b200 import ops

    lg, iou = _synthetic(16383, 2048, 5)
    _check_exact(lg, np.maximum(iou, np.float32(0.9)), 0.5, chunk=1024)
    e = torch.empty((0, 1), dtype=torch.int32, device=DEV)
    keep, cnt = ops.mask_nms(e, e[:, 0], e[:, 0].float(), 0.7)
    assert int(cnt.item()) == 0


# ------------------------------------------------------------------------------------------------
# 2. end to end against the fp32 oracle
# ------------------------------------------------------------------------------------------------
def _decision_margins(cand, iou, st, nt):
    """Smallest margin of every filter decision (a candidate fails some test by at least the margin, or passes all of them by
    at least the margin), of every NMS decision (a later candidate's IoU with the kept ones vs nms_thresh) and the smallest
    gap between the scores of valid candidates."""
    io, stab, area = np.asarray(iou, np.float32).ravel(), cand["stability"], cand["area"]
    fm = []
    for k in range(len(io)):
        if area[k] < 1:
            continue
        fm.append(abs(stab[k] - np.float32(st)) if not np.isnan(stab[k]) else np.inf)  # the only active filter
    order = amg_ref.sort_order(cand["score"])
    sc = cand["score"][order]
    P = amg_ref.pair_ious(cand["bits"], area, order)
    nm, kept = [], []
    for j in range(len(order)):
        ious = P[kept, j]
        sup = ious[ious > nt]
        nm.append((sup - nt).max() if len(sup) else (nt - ious).min() if len(ious) else np.inf)
        if not len(sup):
            kept.append(j)
    return min(fm), min(nm), (np.diff(-sc).min() if len(sc) > 1 else np.inf), len(order), len(kept)


# seeds and thresholds chosen (on the CPU oracle) so that every decision has a margin >= 1e-2; pred_iou_thresh = 0 (off)
FIXTURES = {
    "base": dict(seed=5, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.475, stability_score_offset=0.02, mask_nms_thresh=0.9)),
    "hier": dict(seed=8, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.55, stability_score_offset=0.05, mask_nms_thresh=0.9)),
}


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


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_generator_matches_fp32_oracle(kind):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES[kind]
    model, oracle = _models(kind, fx["seed"])
    xyz, rgb = synth.make_batch(1, 2048, fx["seed"])
    want = amg_ref.generate_ref(oracle, xyz, rgb, 64, 64, **fx["kw"])
    fm, nm, gap, valid, kept = _decision_margins(want, want["iou"], fx["kw"]["stability_score_thresh"], fx["kw"]["mask_nms_thresh"])
    print(f"[amg] {kind}: oracle valid {valid} kept {kept}; margins filter {fm:.3g} nms {nm:.3g} score gap {gap:.3g}")
    assert fm >= 1e-2 and nm >= 1e-2 and gap >= 2e-3 and kept >= 2 and valid > kept
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])  # 3 chunks, last one short
    got = gen.generate_packed(xyz[0].to(DEV), rgb[0].to(DEV))
    C = want["slots"]
    want_pairs = [(int(want["point_index"][k // C]), int(k % C)) for k in want["keep"]]
    got_pairs = list(zip(got["point_index"].tolist(), got["mask_slot"].tolist()))
    assert got_pairs == want_pairs
    np.testing.assert_allclose(got["predicted_iou"].cpu().numpy(), want["iou"].reshape(-1)[want["keep"]], atol=1e-3, rtol=0)
    seg = amg_ref.unpack_bits(got["bits"].cpu().numpy().view(np.uint32), 2048)
    lg = want["logits"].reshape(-1, 2048)[want["keep"]]
    diff = seg != (lg > 0)
    assert np.all(np.abs(lg[diff]) < 1e-3), f"{diff.sum()} points differ"
    assert np.array_equal(got["area"].cpu().numpy(), seg.sum(1))
    np.testing.assert_array_equal(got["point_coords"].cpu().numpy(), xyz[0].numpy()[got["point_index"].cpu().numpy()])
    recs = gen.generate(xyz[0].to(DEV), rgb[0].to(DEV))
    assert [(r["point_index"]) for r in recs] == [p for p, _ in want_pairs]
    assert all(r["segmentation"].dtype == bool and r["segmentation"].shape == (2048,) for r in recs)


def test_generator_enqueues_without_host_sync_and_checks_range():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model, _ = _models("base", 5)
    xyz, rgb = synth.make_batch(1, 2048, 5)
    xyz, rgb = xyz.to(DEV), rgb.to(DEV)
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=16, **FIXTURES["base"]["kw"])
    first = gen.generate_packed(xyz, rgb)  # packs the weights
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st = gen._enqueue(xyz, rgb)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    got = gen._finish(st)
    assert got["area"].shape[0] == first["area"].shape[0]
    with pytest.raises(ValueError):
        gen.generate_packed(xyz * 1.5, rgb)  # FPS prompt points outside [-1, 1]
    assert gen.generate_packed(xyz, rgb)["area"].shape[0] == first["area"].shape[0]  # the flag was reset


# ------------------------------------------------------------------------------------------------
# 4. full size, once
# ------------------------------------------------------------------------------------------------
def test_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam
    from psam_b200 import ops

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    xyz, rgb = synth.make_batch(1, 32768, 3)
    xyz, rgb = xyz.to(DEV), rgb.to(DEV)
    P, Bp, nt = 1024, 64, 0.7
    rules = dict(mask_threshold=0.0, stability_offset=0.05, pred_iou_thresh=0.0, stability_thresh=0.0, min_area=0)
    with torch.no_grad():
        enc = model._encode(xyz, rgb)
        _, centers = ops.fps(xyz, P)
        labels = torch.ones((Bp, 1), dtype=torch.int64, device=DEV)
        logits, ious = [], []
        for s in range(0, P, Bp):
            m, i = model._decode_unchecked(enc, centers[0, s:s + Bp].unsqueeze(1), labels, None, True)
            logits.append(m)
            ious.append(i)
        lg, io = torch.cat(logits), torch.cat(ious)
        cand = ops.mask_candidates(lg, io, **rules)
        keep, cnt = ops.mask_nms(cand[0], cand[1], cand[3], nt)
    n = int(cnt.item())
    lg_np, io_np = lg.cpu().numpy(), io.cpu().numpy()
    want = amg_ref.candidates(lg_np, io_np, **rules)
    assert np.array_equal(cand[0].cpu().numpy().view(np.uint32), want["bits"])
    assert np.array_equal(cand[1].cpu().numpy(), want["area"])
    np.testing.assert_array_equal(cand[2].cpu().numpy(), want["stability"])
    np.testing.assert_array_equal(cand[3].cpu().numpy(), want["score"])
    want_keep = amg_ref.nms(want["bits"], want["area"], want["score"], nt)
    print(f"[amg] full size: {int((want['score'] > -np.inf).sum())} valid candidates, {n} kept")
    assert keep[:n].cpu().numpy().tolist() == want_keep.tolist()
    # the generator itself: no two kept masks overlap above the threshold, scores non-increasing
    gen = PointCloudMaskGenerator(model, points_per_cloud=P, points_per_batch=Bp, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05, mask_nms_thresh=nt)
    out = gen.generate_packed(xyz, rgb)
    bits, area, sc = out["bits"].cpu().numpy().view(np.uint32), out["area"].cpu().numpy(), out["predicted_iou"].cpu().numpy()
    assert len(sc) >= 1 and np.all(np.diff(sc) <= 0)
    if len(sc) > 1:
        iou = amg_ref.pair_ious(bits, area, np.arange(len(sc)))
        np.fill_diagonal(iou, 0)
        assert iou.max() <= nt
