"""GPU tests of clouds of different sizes in one padded batch: the four length-aware launches (FPS, kNN, mask candidates,
small regions) equal the single-cloud kernels on every unpadded cloud bit for bit, whatever the padding holds;
predict_masks_varlen matches predict_masks and the fp32 oracles per cloud; generate_packed_batch on a ragged list matches
the oracle per cloud, is the single-cloud path for one cloud, synchronises once, and holds at full size."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import amg_ref, amg_regions_ref, hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
ATOL, RTOL = 1e-3, 1e-2  # test_gpu_model.py's
K1 = amg_regions_ref.REGION_NEIGHBORS + 1
RULES = dict(mask_threshold=0.0, stability_offset=1.0, pred_iou_thresh=0.88, stability_thresh=0.5, min_area=3)


def _pad(rows, fill):
    """rows: list of [N_b, ...] numpy arrays -> padded [B, N_max, ...] with fill(b, n_pad) in the padding, lengths."""
    n_max = max(len(r) for r in rows)
    out = np.stack([np.concatenate([r, fill(b, n_max - len(r)).astype(r.dtype)]) for b, r in enumerate(rows)])
    lengths = torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV)
    return torch.from_numpy(out).to(DEV), lengths


def _far(b, n):
    """Padding that wins every farthest-point step if read: far outside the cloud, each row farther than the last."""
    return np.stack([np.arange(n) + 100.0 + b, np.full(n, 50.0), np.full(n, -75.0)], 1) if n else np.zeros((0, 3))


def _ball(n, seed, quant=None, dup=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, 3))
    if quant:
        x = np.round(x * quant) / quant  # many equal distances: the block size T decides the winner
    if dup:
        x[rng.integers(0, n, dup)] = x[rng.integers(0, n, dup)]
    return x.astype(np.float32)


# ------------------------------------------------------------------------------------------------
# 1. farthest-point sampling
# ------------------------------------------------------------------------------------------------
FPS_CASES = {
    "T-boundaries": ([32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1000], 24, None),
    "register-resident": ([3000, 1, 2047, 2048, 2049, 1234], 64, None),
    "16-cta": ([70000, 65536, 40000, 3], 48, None),
    "streaming": ([131073, 70001, 600], 32, None),
    "ties": ([300, 257, 700, 64, 65, 33], 40, 4),
    "short": ([10, 40, 100, 64, 1], 64, None),
}


@pytest.mark.parametrize("case", list(FPS_CASES))
def test_fps_varlen_equals_fps_per_cloud(case):
    from psam_b200 import ops

    sizes, G, quant = FPS_CASES[case]
    clouds = [_ball(n, 7 * b + n, quant, dup=n // 8) for b, n in enumerate(sizes)]
    xyz, lengths = _pad(clouds, _far)
    idx, cen = ops.fps(xyz, G, lengths=lengths)
    for b, c in enumerate(clouds):
        g = min(G, len(c))
        ri, rc = ops.fps(torch.from_numpy(c)[None].to(DEV), g)
        assert torch.equal(idx[b, :g], ri[0]), (case, b)
        assert torch.equal(cen[b, :g].view(torch.int32), rc[0].view(torch.int32)), (case, b)
        assert torch.all(idx[b, g:] == 0) and torch.equal(cen[b, g:], cen[b, :1].expand(G - g, 3)), (case, b)
        if g > 1 and len(c) > g:  # prefix property: a longer run starts with the shorter one
            ri2, _ = ops.fps(torch.from_numpy(c)[None].to(DEV), g - 1)
            assert torch.equal(ri2[0], ri[0, : g - 1])


# ------------------------------------------------------------------------------------------------
# 2. kNN
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sizes,K", [([100, 1000, 4099, 2048], 16), ([40, 33, 9000], 9), ([2048, 2047], 1), ([5000, 1100], 64)])
def test_knn_varlen_equals_knn_per_cloud(sizes, K):
    from psam_b200 import ops

    Q = 37
    clouds = [_ball(n, n + b, quant=8, dup=n // 4) for b, n in enumerate(sizes)]
    rng = np.random.default_rng(len(sizes))
    queries = np.stack([c[rng.integers(0, len(c), Q)] for c in clouds])
    # padding: copies of the queries themselves, nearer to every centre than any real point except its duplicates
    key, lengths = _pad(clouds, lambda b, n: queries[b][np.arange(n) % Q] + np.float32(1e-7))
    q = torch.from_numpy(queries).to(DEV)
    idx, d2 = ops.knn(q, key, K, want_d2=True, lengths=lengths)
    for b, c in enumerate(clouds):
        ri, rd = ops.knn(q[b:b + 1], torch.from_numpy(c)[None].to(DEV), K, want_d2=True)
        assert torch.equal(idx[b], ri[0]), b
        assert torch.equal(d2[b].view(torch.int32), rd[0].view(torch.int32)), b
        assert int(idx[b].max()) < len(c)


# ------------------------------------------------------------------------------------------------
# 3. candidates, NMS, small regions
# ------------------------------------------------------------------------------------------------
def _synthetic(Z, N, seed):
    """Overlapping interval-shaped masks with duplicates, logits on the thresholds and tied predicted IoUs."""
    K = 3 * Z
    rng = np.random.default_rng(seed)
    n = np.arange(N, dtype=np.float32)
    protos = max(2, K // 6)
    c = rng.uniform(0, N, protos).astype(np.float32)
    w = rng.uniform(0.05, 0.5, protos).astype(np.float32) * N
    p = rng.integers(0, protos, K)
    lg = ((w[p, None] - np.abs(n[None, :] - c[p, None])) / np.float32(max(N / 16, 1)) + rng.normal(0, 0.3, (K, N))).astype(np.float32)
    for v in (0.0, 1.0, -1.0):
        lg[rng.random((K, N)) < 0.02] = v
    if K > 4:
        lg[1] = lg[0]
    iou = rng.choice(np.float32([0.5, 0.8, 0.88, 0.9, 0.95, 0.97]), size=K).astype(np.float32)
    iou[1::5] = np.float32(0.88)
    return lg.reshape(Z, 3, N), iou.reshape(Z, 3)


@pytest.mark.parametrize("sizes,Z,chunk", [([33, 2047, 2048], 40, 16), ([2047, 1000, 5, 1500], 24, 24), ([4096, 100], 64, 10)])
def test_candidates_and_nms_varlen_equal_single_cloud(sizes, Z, chunk):
    from psam_b200 import ops

    B, C, K = len(sizes), 3, 3 * Z
    n_max = max(sizes)
    W = ops.mask_words(n_max)
    data = [_synthetic(Z, n, 100 * b + n) for b, n in enumerate(sizes)]
    # padded logits are +1e9: a count or a bit that included them would show
    lg_pad = [np.concatenate([lg, np.full((Z, C, n_max - lg.shape[2]), 1e9, np.float32)], 2) for lg, _ in data]
    cand = (torch.empty((B, K, W), dtype=torch.int32, device=DEV), torch.empty((B, K), dtype=torch.int32, device=DEV),
            torch.empty((B, K), dtype=torch.float32, device=DEV), torch.empty((B, K), dtype=torch.float32, device=DEV))
    lengths = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    for s in range(0, Z, chunk):
        e = min(Z, s + chunk)
        rows = torch.from_numpy(np.concatenate([x[s:e] for x in lg_pad])).to(DEV)
        ious = torch.from_numpy(np.concatenate([d[1][s:e] for d in data])).to(DEV)
        ops.mask_candidates_batched(rows, ious, B, out=cand, base=s * C, lengths=lengths, num_prompts=Z, **RULES)
    keep, cnt = ops.mask_nms_batched(cand[0], cand[1], cand[3], 0.7)
    counts = cnt.cpu().tolist()
    for b, (lg, io) in enumerate(data):
        n, P = sizes[b], min(Z, sizes[b])
        Wb, Kb = ops.mask_words(n), 3 * P
        one = ops.mask_candidates(torch.from_numpy(lg[:P]).to(DEV), torch.from_numpy(io[:P]).to(DEV), **RULES)
        assert torch.equal(cand[0][b, :Kb, :Wb], one[0]) and torch.all(cand[0][b, :, Wb:] == 0), b
        assert torch.equal(cand[1][b, :Kb], one[1]) and torch.equal(cand[2][b, :Kb].view(torch.int32), one[2].view(torch.int32))
        assert torch.equal(cand[3][b, :Kb], one[3]), b
        assert torch.all(cand[3][b, Kb:] == -np.inf), b  # prompts past min(P, N_b)
        want = amg_ref.candidates(lg[:P], io[:P], **RULES)
        assert np.array_equal(one[0].cpu().numpy().view(np.uint32), want["bits"])
        k1, c1 = ops.mask_nms(one[0], one[1], one[3], 0.7)
        assert int(c1.item()) == counts[b] and torch.equal(keep[b, : counts[b]], k1[: counts[b]]), b
    assert sum(counts) > 0


def _cloud(N, seed):
    """Gaussian blobs plus coincident duplicates (test_gpu_amg_regions.py's kind of cloud) and a part label per point."""
    rng = np.random.default_rng(seed)
    nb = 8
    centers = rng.uniform(-0.8, 0.8, (nb, 3))
    lab = rng.integers(0, nb, N)
    xyz = centers[lab] + rng.normal(0, 1, (N, 3)) * rng.uniform(0.01, 0.06, nb)[lab, None]
    src = rng.integers(0, N, N // 16)
    xyz[rng.integers(0, N, N // 16)] = xyz[src]
    return np.clip(xyz, -1, 1).astype(np.float32), lab


def _masks(xyz, lab, S, seed):
    rng = np.random.default_rng(seed)
    N = len(lab)
    out = np.zeros((S, N), bool)
    for s in range(S):
        m = np.isin(lab, rng.choice(int(lab.max()) + 1, int(rng.integers(1, 4)), replace=False))
        m[rng.integers(0, N, 5)] = True
        if m.any():
            c = xyz[rng.choice(np.nonzero(m)[0])]
            m &= ((xyz - c) ** 2).sum(1) > rng.uniform(0.005, 0.05) ** 2
        out[s] = m
    out[0] = True
    out[S - 1] = False
    out[S - 1, rng.integers(0, N, 3)] = True
    out[out.sum(1) == 0, 0] = True
    return out


@pytest.mark.parametrize("sizes", [[2047, 500, 1200], [50000, 60000, 30000]])
def test_regions_varlen_equal_single_cloud(sizes):
    """Both label stores: shared memory (N_max <= 49152) and workspace slices (N_max > 49152)."""
    from psam_b200 import ops

    S, Kk = 8, 6
    B, n_max = len(sizes), max(sizes)
    W = ops.mask_words(n_max)
    clouds = [_cloud(n, n + b) for b, n in enumerate(sizes)]
    # padding inside the clouds' extent: a region pass that walked it would join it to every component
    xyz, lengths = _pad([c[0] for c in clouds], lambda b, n: np.zeros((n, 3)))
    nbr, _ = ops.knn(xyz, xyz, K1, lengths=lengths)
    masks = [_masks(x, l, S, 3 * b) for b, (x, l) in enumerate(clouds)]
    bits = np.stack([amg_ref.pack_bits(m, W) for m in masks])
    rng = np.random.default_rng(len(sizes))
    keep = np.stack([rng.permutation(S)[:Kk] for _ in range(B)]).astype(np.int32)
    counts = np.array([Kk, 0] + [3] * (B - 2), dtype=np.int32)
    bits_d = torch.from_numpy(bits.view(np.int32)).to(DEV)
    keep_d, cnt_d = torch.from_numpy(keep).to(DEV), torch.from_numpy(counts).to(DEV)
    changed = 0
    for A in (4, 200):
        rb, ra, rs = ops.mask_regions_batched(bits_d, keep_d, cnt_d, nbr, A, lengths=lengths)
        for b, n in enumerate(sizes):
            c = int(counts[b])
            x1 = torch.from_numpy(clouds[b][0])[None].to(DEV)
            nbr1, _ = ops.knn(x1, x1, K1)
            assert torch.equal(nbr[b, :n], nbr1[0]), b
            Wb = ops.mask_words(n)
            bits1 = torch.from_numpy(amg_ref.pack_bits(masks[b], Wb).view(np.int32)).to(DEV)
            sb, sa, ss = ops.mask_regions(bits1, keep_d[b], cnt_d[b:b + 1], nbr1[0], A)
            assert torch.equal(rb[b, :c, :Wb], sb[:c]) and torch.all(rb[b, :c, Wb:] == 0), (A, b)
            assert torch.equal(ra[b, :c], sa[:c]) and torch.equal(rs[b], ss), (A, b)
            changed += int((ss[:c] == 0).sum())
    assert changed >= 2


# ------------------------------------------------------------------------------------------------
# 4. the model
# ------------------------------------------------------------------------------------------------
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
def test_predict_masks_varlen_per_cloud(kind):
    model, oracle = _models(kind, 3)
    sizes, M, Q = [2048, 3000, 4100], 2, 2
    clouds = [synth.make_batch(1, n, 10 + b) for b, n in enumerate(sizes)]
    prompts = [synth.make_prompts(x, M * Q, 4 + b) for b, (x, _) in enumerate(clouds)]
    pc = torch.stack([p[0].reshape(M, Q, 3) for p in prompts])
    pl = torch.stack([p[1].reshape(M, Q) for p in prompts])
    xyz = [x[0].to(DEV) for x, _ in clouds]
    rgb = [f[0].to(DEV) for _, f in clouds]
    with torch.no_grad():
        got = model.predict_masks_varlen(xyz, rgb, pc.to(DEV), pl.to(DEV), None, True)
        pms = [g[0][:, 1].contiguous() for g in got]
        got2 = model.predict_masks_varlen(xyz, rgb, pc.to(DEV), pl.to(DEV), pms, False)
        for b, ((x, f), n) in enumerate(zip(clouds, sizes)):
            m, i = got[b]
            assert m.shape == (M, 3, n) and i.shape == (M, 3)
            one_m, one_i = model.predict_masks(x.to(DEV), f.to(DEV), pc[b].to(DEV), pl[b].to(DEV), None, True)
            np.testing.assert_allclose(m.cpu().numpy(), one_m.cpu().numpy(), atol=ATOL, rtol=RTOL)
            np.testing.assert_allclose(i.cpu().numpy(), one_i.cpu().numpy(), atol=ATOL, rtol=RTOL)
            want_m, want_i = oracle.predict_masks(x, f, pc[b], pl[b], None, True)
            np.testing.assert_allclose(m.cpu().numpy(), want_m.numpy(), atol=ATOL, rtol=RTOL)
            np.testing.assert_allclose(i.cpu().numpy(), want_i.numpy(), atol=ATOL, rtol=RTOL)
            want2, _ = oracle.predict_masks(x, f, pc[b], pl[b], pms[b].cpu(), False)
            assert got2[b][0].shape == (M, 1, n)
            np.testing.assert_allclose(got2[b][0].cpu().numpy(), want2.numpy(), atol=ATOL, rtol=RTOL)


# ------------------------------------------------------------------------------------------------
# 5. the generator
# ------------------------------------------------------------------------------------------------
# test_gpu_amg_batch.py's fixtures; each cloud is cut to its own size, and a cloud whose filter or NMS decisions come
# within the margins below of a threshold on the oracle is refused rather than compared
FIXTURES = {
    "base": dict(seed=5, clouds=(5, 6, 49), kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.475, stability_score_offset=0.02,
                                                   mask_nms_thresh=0.9)),
    "hier": dict(seed=8, clouds=(26, 32, 36), kw=dict(pred_iou_thresh=0.0, stability_score_thresh=0.55, stability_score_offset=0.05,
                                                   mask_nms_thresh=0.9)),
}
SIZES, AREA = (2048, 1500, 1800), 8


def _ragged(seeds, sizes=SIZES):
    xs, rs = zip(*[synth.make_batch(1, n, s) for s, n in zip(seeds, sizes)])
    return [x[0] for x in xs], [r[0] for r in rs]


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
    return fm, min(nm), (np.diff(-sc).min() if len(sc) > 1 else np.inf), len(kept)


def _pairs(out):
    return list(zip(out["point_index"].tolist(), out["mask_slot"].tolist()))


@pytest.mark.parametrize("kind", ["base", "hier"])
@pytest.mark.parametrize("area", [0, AREA])
def test_ragged_batch_matches_fp32_oracle_per_cloud(kind, area):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES[kind]
    model, oracle = _models(kind, fx["seed"])
    xyz, rgb = _ragged(fx["clouds"])
    nt = fx["kw"]["mask_nms_thresh"]
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])
    outs = gen.generate_packed_batch([x.to(DEV) for x in xyz], [r.to(DEV) for r in rgb], min_mask_region_area=area)
    compared = 0
    for b, (got, n) in enumerate(zip(outs, SIZES)):
        assert got["bits"].shape[1] == (n + 31) // 32 and got["bits"].dtype == torch.int32
        want = amg_regions_ref.generate_ref(oracle, xyz[b][None], rgb[b][None], 64, 64, **fx["kw"], min_mask_region_area=area)
        fm, nm, gap, kept = _margins(want, fx["kw"]["stability_score_thresh"], nt)
        print(f"[varlen] {kind} area {area} cloud {b} (N={n}): margins filter {fm:.3g} nms {nm:.3g} gap {gap:.3g}, kept {kept}")
        if not (fm >= 1e-2 and nm >= 1e-2 and gap >= 2e-3 and kept >= 1):
            continue
        C = want["slots"]
        seg = amg_ref.unpack_bits(got["bits"].cpu().numpy().view(np.uint32), n)
        assert np.array_equal(got["area"].cpu().numpy(), seg.sum(1))
        np.testing.assert_array_equal(got["point_coords"].cpu().numpy(), xyz[b].numpy()[got["point_index"].cpu().numpy()])
        if area == 0:
            assert _pairs(got) == [(int(want["point_index"][k // C]), int(k % C)) for k in want["keep"]], b
            np.testing.assert_allclose(got["predicted_iou"].cpu().numpy(), want["iou"].reshape(-1)[want["keep"]], atol=1e-3, rtol=0)
            lg = want["logits"].reshape(-1, n)[want["keep"]]
            diff = seg != (lg > 0)
            assert np.all(np.abs(lg[diff]) < 1e-3), f"cloud {b}: {diff.sum()} points differ"
        else:
            # the region stage is exact on the first-stage masks; compared where those equal the oracle's bit for bit
            first = gen.generate_packed_batch([x.to(DEV) for x in xyz[b:b + 1]], [r.to(DEV) for r in rgb[b:b + 1]])[0]
            if not np.array_equal(first["bits"].cpu().numpy().view(np.uint32), want["bits"][want["keep"]]):
                continue
            assert _pairs(got) == [(int(want["point_index"][k // C]), int(k % C)) for k in want["final_slots"]], b
            assert np.array_equal(got["bits"].cpu().numpy().view(np.uint32), want["regions"]["bits"][want["regions"]["keep"]])
        compared += 1
    print(f"[varlen] {kind} area {area}: {compared} of {len(SIZES)} clouds compared")
    assert compared >= 1
    recs = gen.generate_batch([x.to(DEV) for x in xyz], [r.to(DEV) for r in rgb], min_mask_region_area=area)
    assert [[r["segmentation"].shape for r in rb] for rb in recs] == [[(n,)] * len(rb) for rb, n in zip(recs, SIZES)]


@pytest.mark.parametrize("area", [0, AREA])
def test_one_cloud_list_is_the_single_cloud_path(area):
    """generate_packed_batch([xyz], [rgb])[0] equals generate_packed(xyz, rgb) bit for bit in every field, with the first
    call's encode and decode outputs replayed to the second (the encoder's split-K reductions may round differently)."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = (t[0].to(DEV) for t in synth.make_batch(1, 1999, fx["seed"]))
    gen = PointCloudMaskGenerator(model, points_per_cloud=64, points_per_batch=24, **fx["kw"])
    gen.generate_packed(xyz, rgb)  # packs the weights
    enc_fn, dec_fn, log = model._encode, model._decode_unchecked, []

    def record_encode(*a):
        log.append(("enc", [t.clone() for t in a[:2]], enc_fn(*a)))
        return log[-1][2]

    def record_decode(enc, coords, labels, masks, multi):
        log.append(("dec", [coords.clone(), labels.clone()], dec_fn(enc, coords, labels, masks, multi)))
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
        one = gen.generate_packed(xyz, rgb, min_mask_region_area=area)
        replay = iter(log)
        model._encode, model._decode_unchecked = replay_call("enc"), replay_call("dec")
        (bat,) = gen.generate_packed_batch([xyz], [rgb], min_mask_region_area=area)
        assert next(replay, None) is None
    finally:
        del model._encode, model._decode_unchecked
    assert list(one.keys()) == list(bat.keys())
    for k in one:
        assert one[k].dtype == bat[k].dtype and torch.equal(one[k], bat[k]), k
    assert one["area"].shape[0] >= 1


def test_ragged_batch_enqueues_without_host_sync_and_checks_range():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    fx = FIXTURES["base"]
    model, _ = _models("base", fx["seed"])
    xyz, rgb = _ragged(fx["clouds"])
    xyz, rgb = [x.to(DEV) for x in xyz], [r.to(DEV) for r in rgb]
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
    bad = [x.clone() for x in xyz]
    bad[1] *= 1.5  # one cloud's FPS prompt points outside [-1, 1]
    with pytest.raises(ValueError):
        gen.generate_packed_batch(bad, rgb)
    again = gen.generate_packed_batch(xyz, rgb, min_mask_region_area=AREA)  # the flag was reset
    assert [g["area"].shape[0] for g in again] == [f["area"].shape[0] for f in first]


# ------------------------------------------------------------------------------------------------
# 6. full size, once
# ------------------------------------------------------------------------------------------------
def test_ragged_batch_full_size_vit_l():
    """ViT-L, 4 clouds of 20000 .. 32768 points, 1024 prompts: the candidates and NMS of the batched path equal the oracle
    on its own logits cut to each cloud, and each cloud's masks agree with its own generate_packed."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam
    from psam_b200 import ops

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    sizes, P, Bp, nt = [32768, 20000, 27001, 24576], 1024, 64, 0.7
    B, n_max = len(sizes), max(sizes)
    xyz, rgb = _ragged((3, 4, 5, 6), sizes)
    xyz, rgb = [x.to(DEV) for x in xyz], [r.to(DEV) for r in rgb]
    gen = PointCloudMaskGenerator(model, points_per_cloud=P, points_per_batch=Bp, pred_iou_thresh=0.0, stability_score_thresh=0.0,
                                  stability_score_offset=0.05, mask_nms_thresh=nt)
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
    counts = st["keep_count"].cpu().numpy()
    rules = dict(mask_threshold=0.0, stability_offset=0.05, pred_iou_thresh=0.0, stability_thresh=0.0, min_area=0)
    for b, n in enumerate(sizes):
        lg = np.concatenate([m.reshape(B, Zc, 3, n_max)[b, :, :, :n] for m, _ in logits])
        io = np.concatenate([i.reshape(B, Zc, 3)[b] for _, i in logits])
        want = amg_ref.candidates(lg, io, **rules)
        W = ops.mask_words(n)
        assert np.array_equal(st["bits"][b, :, :W].cpu().numpy().view(np.uint32), want["bits"]), b
        assert np.array_equal(st["area"][b].cpu().numpy(), want["area"])
        np.testing.assert_array_equal(st["score"][b].cpu().numpy(), want["score"])
        want_keep = amg_ref.nms(want["bits"], want["area"], want["score"], nt)
        assert st["keep"][b, : counts[b]].cpu().numpy().tolist() == want_keep.tolist(), b
        one = gen.generate_packed(xyz[b], rgb[b])
        got = outs[b]
        assert got["bits"].shape[1] == W
        fps_idx, _ = ops.fps(xyz[b][None], P)
        assert torch.equal(st["point_index"][b], fps_idx[0]), b  # the same prompts
        a, c = set(_pairs(one)), set(_pairs(got))
        jac = len(a & c) / max(1, len(a | c))
        print(f"[varlen] full size cloud {b} (N={n}): {len(c)} kept, {len(a)} by generate_packed, overlap {jac:.3f}")
        assert len(c) >= 1 and jac >= 0.8, b
