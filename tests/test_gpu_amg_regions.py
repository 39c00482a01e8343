"""GPU tests of the small-region post-processing of automatic mask generation (min_mask_region_area): psam_mask_regions
and the second NMS equal the scipy oracle exactly on synthetic clouds (both label stores: shared memory up to 49152
points, the workspace beyond), the kNN graph equals the C oracle's, the generator matches the fp32 oracle end to end for
both model classes, it enqueues without host synchronisation, and the stage holds at full size (ViT-L, N = 32768)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_ref, amg_regions_ref, hier_ref, synth, tokenizer_ref, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
K1 = amg_regions_ref.REGION_NEIGHBORS + 1


# ------------------------------------------------------------------------------------------------
# 1. kernel exactness on synthetic clouds
# ------------------------------------------------------------------------------------------------
def _cloud(N, seed):
    """Separated Gaussian blobs, points on line segments and coincident duplicates.  Returns xyz [N, 3] fp32 and a part
    label per point (blob or line)."""
    rng = np.random.default_rng(seed)
    nb, nl = 10, 3
    centers = rng.uniform(-0.8, 0.8, (nb, 3))
    n_line = N // 8
    n_dup = N // 16
    n_blob = N - n_line - n_dup
    lab_b = rng.integers(0, nb, n_blob)
    pb = centers[lab_b] + rng.normal(0, 1, (n_blob, 3)) * rng.uniform(0.01, 0.06, nb)[lab_b, None]
    lab_l = rng.integers(0, nl, n_line)
    ends = rng.uniform(-0.9, 0.9, (nl, 2, 3))
    t = rng.random((n_line, 1))
    pl = ends[lab_l, 0] * (1 - t) + ends[lab_l, 1] * t
    xyz = np.concatenate([pb, pl]).astype(np.float32)
    lab = np.concatenate([lab_b, nb + lab_l])
    src = rng.integers(0, len(xyz), n_dup)  # exact duplicates: distance-0 neighbours, ties broken by index
    xyz, lab = np.concatenate([xyz, xyz[src]]), np.concatenate([lab, lab[src]])
    perm = rng.permutation(N)
    return np.clip(xyz[perm], -1, 1), lab[perm]


def _masks(xyz, lab, S, seed):
    """S masks: unions of parts, plus stray points, minus punched holes (a ball around a mask point, or scattered
    points); slot 0 the whole cloud (each point and its 8 neighbours share a component, so no component is smaller than
    9 points), slot 1 a plain union of parts, one stray-only mask and one single-point mask."""
    rng = np.random.default_rng(seed)
    N = len(lab)
    parts = int(lab.max()) + 1
    out = np.zeros((S, N), bool)
    for s in range(S):
        m = np.isin(lab, rng.choice(parts, int(rng.integers(1, 4)), replace=False))
        m[rng.integers(0, N, int(rng.integers(0, 6)))] = True  # strays (islands of one point, mostly)
        if m.any() and rng.random() < 0.7:  # a punched ball
            c = xyz[rng.choice(np.nonzero(m)[0])]
            r = rng.uniform(0.005, 0.05)
            m &= ((xyz - c) ** 2).sum(1) > r * r
        m[rng.integers(0, N, int(rng.integers(0, 6)))] = False  # scattered holes
        out[s] = m
    out[0] = True
    out[1] = np.isin(lab, rng.choice(parts, 2, replace=False))
    out[S - 2] = False
    out[S - 2, rng.integers(0, N, 5)] = True
    out[S - 1] = False
    out[S - 1, rng.integers(0, N)] = True
    out[out.sum(1) == 0, 0] = True  # candidates are never empty
    return out


def _run(bits, keep, count, nbr, A, nt):
    from psam_b200 import ops

    b = torch.from_numpy(bits.view(np.int32)).to(DEV)
    k = torch.from_numpy(keep.astype(np.int32)).to(DEV)
    c = torch.tensor([count], dtype=torch.int32, device=DEV)
    rb, ra, rs = ops.mask_regions(b, k, c, nbr, A)
    keep2, c2 = ops.mask_nms(rb, ra, rs, nt)
    torch.cuda.synchronize()
    return (rb.cpu().numpy().view(np.uint32), ra.cpu().numpy(), rs.cpu().numpy(), keep2[: int(c2.item())].cpu().numpy())


@pytest.mark.parametrize("N", [33, 2047, 32768, 49152, 49153, 131072])
def test_mask_regions_match_oracle_exactly(N):
    from psam_b200 import ops

    xyz, lab = _cloud(N, N)
    xyz_d = torch.from_numpy(xyz).to(DEV)[None]
    nbr_d, _ = ops.knn(xyz_d, xyz_d, K1)
    nbr = nbr_d[0].cpu().numpy()
    if N <= 32768:  # the C oracle is quadratic
        assert np.array_equal(nbr, tokenizer_ref.knn(xyz[None], xyz[None], K1)[0][0])
    S = 12 if N <= 49153 else 6
    masks = _masks(xyz, lab, S, N + 1)
    W = ops.mask_words(N) + (1 if N == 2047 else 0)  # a padding word past ceil(N / 32) stays zero
    bits = amg_ref.pack_bits(masks, W)
    rng = np.random.default_rng(N + 2)
    keep = np.concatenate([[1], 2 + rng.permutation(S - 2)[: S - 4], [0]])  # an unsorted subset of the slots
    nt = 0.7
    changed = unchanged = 0
    for A, count in ((4, len(keep)), (max(4, N // 4), len(keep) - 1), (3, 0)):
        rb, ra, rs, keep2 = _run(bits, keep, count, nbr_d[0], A, nt)
        want = amg_regions_ref.postprocess_small_regions(bits, keep[:count], nbr, A, nt)
        assert np.array_equal(rb[:count], want["bits"]), (A, count)
        assert np.array_equal(ra[:count], want["area"])
        assert np.array_equal(rs[:count], want["score"])
        assert np.all(rs[count:] == -np.inf)
        assert keep2.tolist() == want["keep"].tolist()
        assert np.all(ra[:count] >= 1)
        changed += int((want["score"] == 0).sum())
        unchanged += int((want["score"] == 1).sum())
        if count:  # the same call again gives the same bits
            assert np.array_equal(_run(bits, keep, count, nbr_d[0], A, nt)[0], rb)
    assert changed >= 2 and unchanged >= 1, (changed, unchanged)


# ------------------------------------------------------------------------------------------------
# 2. end to end against the fp32 oracle
# ------------------------------------------------------------------------------------------------
# the fixtures of test_gpu_amg.py (every filter / NMS decision has a margin >= 1e-2, valid scores are >= 2e-3 apart), with
# min_mask_region_area chosen on the CPU oracle so that it changes at least one kept mask and leaves at least one unchanged
FIXTURES = {
    "base": dict(seed=5, N=2048, area=8, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.475, stability_score_offset=0.02,
                                                 mask_nms_thresh=0.9)),
    "hier": dict(seed=8, N=2048, area=8, kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.55, stability_score_offset=0.05,
                                                 mask_nms_thresh=0.9)),
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
def test_generator_regions_match_fp32_oracle(kind):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES[kind]
    N, A = fx["N"], fx["area"]
    model, oracle = _models(kind, fx["seed"])
    xyz, rgb = synth.make_batch(1, N, fx["seed"])
    want = amg_regions_ref.generate_ref(oracle, xyz, rgb, 64, 64, **fx["kw"], min_mask_region_area=A)
    post = want["regions"]
    print(f"[amg regions] {kind}: kept {len(want['keep'])}, changed {int((post['score'] == 0).sum())}, final {len(post['keep'])}")
    assert 0 < int((post["score"] == 0).sum()) < len(post["score"])
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])
    st = gen._enqueue(xyz[0].to(DEV), rgb[0].to(DEV), min_mask_region_area=A)
    got = gen._finish(st)
    # a logit on the other side of the threshold would change connectivity, so the comparison below is exact only when
    # the first-stage kept masks are: check that directly (the random tiny models put a few logits of every mask within
    # 1e-3 of the threshold, so a margin cannot be asked of them)
    first = st["keep"][: len(want["keep"])].long()
    assert int(st["keep_count"].item()) == len(want["keep"])
    assert st["keep"][: len(want["keep"])].tolist() == want["keep"].tolist()
    assert np.array_equal(st["bits"][first].cpu().numpy().view(np.uint32), want["bits"][want["keep"]])
    C = want["slots"]
    want_pairs = [(int(want["point_index"][k // C]), int(k % C)) for k in want["final_slots"]]
    got_pairs = list(zip(got["point_index"].tolist(), got["mask_slot"].tolist()))
    assert got_pairs == want_pairs
    assert np.array_equal(got["bits"].cpu().numpy().view(np.uint32), post["bits"][post["keep"]])
    assert np.array_equal(got["area"].cpu().numpy(), post["area"][post["keep"]])
    np.testing.assert_allclose(got["predicted_iou"].cpu().numpy(), want["iou"].reshape(-1)[want["final_slots"]], atol=1e-3, rtol=0)
    np.testing.assert_allclose(got["stability_score"].cpu().numpy(), want["stability"][want["final_slots"]], atol=1e-6, rtol=0)
    recs = gen.generate(xyz[0].to(DEV), rgb[0].to(DEV), min_mask_region_area=A)
    assert [r["point_index"] for r in recs] == [p for p, _ in want_pairs]
    assert [r["area"] for r in recs] == post["area"][post["keep"]].tolist()
    # the default leaves the output as it was: the first NMS order and the candidate masks
    plain = gen.generate_packed(xyz[0].to(DEV), rgb[0].to(DEV))
    assert list(zip(plain["point_index"].tolist(), plain["mask_slot"].tolist())) == \
        [(int(want["point_index"][k // C]), int(k % C)) for k in want["keep"]]
    assert np.array_equal(plain["bits"].cpu().numpy().view(np.uint32), want["bits"][want["keep"]])


def test_generator_regions_enqueue_without_host_sync():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = synth.make_batch(1, fx["N"], fx["seed"])
    xyz, rgb = xyz.to(DEV), rgb.to(DEV)
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=16, **fx["kw"])
    first = gen.generate_packed(xyz, rgb, min_mask_region_area=fx["area"])  # packs the weights
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st = gen._enqueue(xyz, rgb, min_mask_region_area=fx["area"])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    got = gen._finish(st)
    assert torch.equal(got["bits"], first["bits"]) and torch.equal(got["point_index"], first["point_index"])


# ------------------------------------------------------------------------------------------------
# 4. full size, once
# ------------------------------------------------------------------------------------------------
def test_regions_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam
    from psam_b200 import ops

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    xyz, rgb = synth.make_batch(1, 32768, 3)
    xyz, rgb = xyz.to(DEV), rgb.to(DEV)
    P, Bp, nt, A = 1024, 64, 0.7, 64
    gen = PointCloudMaskGenerator(model, points_per_cloud=P, points_per_batch=Bp, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05, mask_nms_thresh=nt)
    st = gen._enqueue(xyz, rgb, min_mask_region_area=A)
    nbr, _ = ops.knn(xyz, xyz, K1)
    out = gen._finish(st)
    n = int(st["keep_count"].item())
    n2 = int(st["region_count"].item())
    keep = st["keep"][:n].cpu().numpy()
    want = amg_regions_ref.postprocess_small_regions(st["bits"].cpu().numpy().view(np.uint32), keep, nbr[0].cpu().numpy(), A, nt)
    assert np.array_equal(st["region_bits"].cpu().numpy().view(np.uint32)[:n], want["bits"])
    assert np.array_equal(st["region_area"].cpu().numpy()[:n], want["area"])
    assert st["region_keep"][:n2].cpu().numpy().tolist() == want["keep"].tolist()
    print(f"[amg regions] full size: {n} kept, {int((want['score'] == 0).sum())} changed, {n2} after the second NMS")
    bits, area = out["bits"].cpu().numpy().view(np.uint32), out["area"].cpu().numpy()
    assert np.array_equal(bits, want["bits"][want["keep"]]) and np.array_equal(area, want["area"][want["keep"]])
    if len(area) > 1:
        iou = amg_ref.pair_ious(bits, area, np.arange(len(area)))
        np.fill_diagonal(iou, 0)
        assert iou.max() <= nt
