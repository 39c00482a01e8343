"""GPU tests of dense-scan segmentation: the voxel subsample equals the numpy oracle bit for bit (P = 1 to 2^24 + 3, S from 1
to beyond P, volume, surface, line, single-point, LiDAR-like and cell-edge inputs, two seeds, repeated runs), the grid
nearest search equals the brute-force psam_nn_distance_f32 bit for bit (random clouds, mesh vertices and face centres
against surface samples, lattice ties, duplicates, NaN / inf, far queries, overflowing and subnormal distances, n2 = 1,
n2 = 2^20 with n1 = 10^7) and the C oracle at small sizes, ScanSegmenter is exact end to end for both model classes with
one host synchronisation per scan and none in the lifting, and the invariants hold at full size (ViT-L, 10^7 points)."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hier_ref, mesh_ref, scan_ref, tokenizer_ref, torch_ref  # noqa: E402
from psam_b200 import synth  # noqa: E402

DEV = torch.device("cuda:0")
F32 = np.float32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ------------------------------------------------------------------------------------------------
# voxel subsample
# ------------------------------------------------------------------------------------------------
def _scan_input(kind, P, seed):
    rng = np.random.default_rng(seed)
    if kind == "volume":
        return rng.uniform(-1, 1, (P, 3)).astype(F32)
    if kind == "surface":
        d = rng.normal(size=(P, 3))
        return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)
    if kind == "line":
        t = rng.uniform(-1, 1, P)
        return np.stack([t, 0.3 * t, -0.2 * t], 1).astype(F32)
    if kind == "single":
        return np.tile(F32([[0.1, -0.7, 0.4]]), (P, 1))
    if kind == "lidar":
        x, _ = synth.make_scan(P, seed)
        v = np.isfinite(x).all(1)
        c = x[v].astype(np.float64)
        c -= c.mean(0)
        x[v] = (c / np.linalg.norm(c, axis=1).max()).astype(F32)
        return x
    if kind == "edges":  # every coordinate on a cell edge of some level, plus +-1 and values just inside
        k = rng.integers(-2 ** 10, 2 ** 10, (P, 3))
        x = (k * 2.0 ** -10).astype(F32)
        x[:: 7] = F32(1)
        x[1:: 7] = F32(-1)
        x[2:: 11] = np.nextafter(x[2:: 11], F32(0))
        return x
    raise ValueError(kind)


def _check_subsample(xyz, S, seed):
    from psam_b200 import ops

    idx, stats = ops.voxel_subsample(_t(xyz), S, seed)
    w_idx, w_stats = scan_ref.subsample(xyz, S, seed)
    assert stats.cpu().numpy().tolist() == w_stats.tolist()
    assert np.array_equal(idx.cpu().numpy(), w_idx)
    again = ops.voxel_subsample(_t(xyz), S, seed)
    assert torch.equal(idx, again[0]) and torch.equal(stats, again[1])
    return w_stats


@pytest.mark.parametrize("kind,P", [("volume", 1), ("volume", 1000), ("surface", 100003), ("line", 50000), ("single", 4097),
                                    ("lidar", 300000), ("edges", 65536)])
@pytest.mark.parametrize("seed", [0, 0xDEADBEEFCAFEF00D])
def test_voxel_subsample_bit_exact(kind, P, seed):
    xyz = _scan_input(kind, P, 11 + P)
    for S in (1, 512, 32768, P, P + 5):
        _check_subsample(xyz, S, seed)


def test_voxel_subsample_bit_exact_large():
    _check_subsample(_scan_input("volume", 2 ** 24 + 3, 5), 32768, 0xDEADBEEFCAFEF00D)


def test_voxel_subsample_invalid_rows():
    xyz = _scan_input("volume", 20000, 3)
    xyz[::13, 1] = np.nan
    xyz[5::17, 2] = np.inf
    st = _check_subsample(xyz, 1024, 9)
    assert st[0] == np.isfinite(xyz).all(1).sum()
    st = _check_subsample(np.full((100, 3), np.nan, F32), 16, 0)
    assert st.tolist() == [0, 21, 0, 0]


# ------------------------------------------------------------------------------------------------
# grid nearest search
# ------------------------------------------------------------------------------------------------
def _brute(q, k):
    from psam_b200 import native as nv

    qt, kt = _t(np.asarray(q, F32)), _t(np.asarray(k, F32))
    d = torch.empty(len(q), dtype=torch.float32, device=DEV)
    i = torch.empty(len(q), dtype=torch.int64, device=DEV)
    nv.check(nv.lib().psam_nn_distance_f32(nv.ptr(qt), nv.ptr(kt), len(q), len(k), nv.ptr(d), nv.ptr(i), nv.stream()), "nn_distance")
    return d, i


def _check_grid(q, k, c_oracle=False):
    from psam_b200 import ops

    d, i = ops.nearest_grid(_t(np.asarray(q, F32)), _t(np.asarray(k, F32)))
    bd, bi = _brute(q, k)
    assert torch.equal(i, bi), int((i != bi).sum())
    assert np.array_equal(_u32(d.cpu().numpy()), _u32(bd.cpu().numpy()))
    if c_oracle:
        w = tokenizer_ref.knn(np.asarray(q, F32)[None], np.asarray(k, F32)[None], 1)[0][0, :, 0]
        ok = np.isfinite(np.asarray(q)).all(1)
        assert np.array_equal(i.cpu().numpy()[ok], w[ok])
    return i.cpu().numpy()


@pytest.mark.parametrize("n1,n2", [(1, 1), (1000, 1), (5000, 7), (20000, 3000), (100000, 32768)])
def test_grid_random_clouds(n1, n2):
    rng = np.random.default_rng(n1 + n2)
    k = rng.uniform(-1, 1, (n2, 3)).astype(F32)
    q = rng.uniform(-1.2, 1.2, (n1, 3)).astype(F32)
    _check_grid(q, k, c_oracle=n1 * n2 <= 10 ** 8)
    _check_grid(q, k[:, [0, 1, 1]] * F32([1, 1, 0]))  # planar keys


def test_grid_mesh_targets_against_surface_samples():
    from pc_sam.mesh import sample_surface
    from pc_sam.utils.ply import normalize_points
    from psam_b200 import ops

    v, f, _ = synth.make_mesh(200000, 2)
    vn = normalize_points(v.astype(np.float64)).astype(F32)
    xyz, _, _ = sample_surface(_t(vn), _t(f), 32768, seed=3)
    centers = ops.mesh_face_centers(_t(vn), _t(f)).cpu().numpy()
    xs = xyz.cpu().numpy()
    _check_grid(vn, xs)
    _check_grid(centers, xs)
    _check_grid(vn[:3000], xs, c_oracle=True)


def test_grid_adversarial():
    rng = np.random.default_rng(7)
    # keys on a lattice aligned with the cell edges, queries at lattice midpoints: ties everywhere
    g = np.arange(-8, 8, dtype=F32) / F32(8)
    k = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    mid = (np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + F32(1 / 16)).astype(F32)
    _check_grid(np.concatenate([mid, k, k[::-1] + F32(1 / 16)]), k, c_oracle=True)
    # duplicate keys: the lower index wins
    kd = np.concatenate([k, k, k[::3]])
    perm = rng.permutation(len(kd))
    _check_grid(np.concatenate([k, mid]), kd[perm], c_oracle=True)
    # NaN and inf in keys and queries
    kn = rng.uniform(-1, 1, (5000, 3)).astype(F32)
    kn[::7, 0] = np.nan
    kn[3::11, 2] = np.inf
    kn[5::13, 1] = -np.inf
    qn = rng.uniform(-1, 1, (4000, 3)).astype(F32)
    qn[::5, 1] = np.nan
    qn[2::9, 0] = np.inf
    idx = _check_grid(qn, kn)
    assert (idx[::5] == -1).all() and (idx[2::9] == -1).all()
    _check_grid(qn, np.full((10, 3), np.nan, F32))  # no finite key at all
    # queries 10^3 times outside the keys' box
    kb = rng.uniform(-1, 1, (20000, 3)).astype(F32)
    far = rng.normal(size=(300, 3))
    far = (far / np.linalg.norm(far, axis=1, keepdims=True) * rng.uniform(10, 1000, (300, 1))).astype(F32)
    _check_grid(far, kb, c_oracle=True)
    # coordinates so large that d overflows, for some keys or for all of them
    big = (rng.uniform(-1, 1, (3000, 3)) * 3e38).astype(F32)
    _check_grid(big[:1000], big)
    _check_grid((rng.uniform(-1, 1, (1000, 3)) * 1e19).astype(F32), (rng.uniform(-1, 1, (3000, 3)) * 1e19).astype(F32))
    # tiny coordinates: subnormal and zero distances
    tiny = (rng.uniform(-1, 1, (3000, 3)) * 1e-22).astype(F32)
    _check_grid(tiny[:1500], tiny[1500:])
    sub = (rng.integers(-40, 40, (3000, 3)) * 2.0 ** -149).astype(F32)
    _check_grid(sub[:1000], sub)
    # one key
    _check_grid(rng.uniform(-5, 5, (1000, 3)).astype(F32), F32([[0.3, 0.2, -0.1]]), c_oracle=True)


def test_grid_large():
    from psam_b200 import ops

    rng = np.random.default_rng(1)
    k = rng.uniform(-1, 1, (2 ** 20, 3)).astype(F32)
    q = rng.uniform(-1, 1, (10 ** 7, 3)).astype(F32)
    kt, qt = _t(k), _t(q)
    d, i = ops.nearest_grid(qt, kt)
    sel = rng.choice(len(q), 20000, replace=False)
    bd, bi = _brute(q[sel], k)
    assert torch.equal(i[_t(sel)], bi) and torch.equal(d[_t(sel)], bd)
    _check_grid(q[:200000], k[: 2 ** 16])


# ------------------------------------------------------------------------------------------------
# end to end
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
    return model.cuda().eval()


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_scan_segmenter_end_to_end(kind):
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.scan import ScanSegmenter

    model = _models(kind, 3)
    xyz, rgb = synth.make_scan(200000, 5)
    xyz = xyz * F32(7.0) + F32([10, -3, 2])  # not normalised: the segmenter normalises over the valid points
    valid = np.isfinite(xyz).all(1)
    S = 2048
    seg = ScanSegmenter(model, num_points=S, seed=7)

    def syncs(fn):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return sum("called a synchronizing" in str(x.message) for x in w)

    xd, rd = _t(xyz), _t(rgb)
    torch.cuda.synchronize()
    n_scan = syncs(lambda: seg.set_scan(xd, rd))
    n_encode = syncs(lambda: model.set_pointcloud(seg.xyz.clone(), seg.rgb.clone()))  # the model's own, on fresh tensors
    assert n_scan == 1 + n_encode, (n_scan, n_encode)
    seg.set_scan(xyz, rgb)  # numpy input: the same result
    x64 = xyz[valid].astype(np.float64)
    assert np.allclose(seg.shift, x64.mean(0)) and np.isclose(seg.scale, np.linalg.norm(x64 - seg.shift, axis=1).max())
    pts = seg.points.cpu().numpy()
    assert np.isnan(pts[~valid]).all() and np.isfinite(pts[valid]).all()
    w_idx, w_st = scan_ref.subsample(pts, S, 7)
    kept = w_idx[w_idx >= 0]
    assert np.array_equal(seg.sample_index.cpu().numpy(), kept)
    assert np.array_equal(seg.xyz[0].cpu().numpy(), pts[kept]) and np.array_equal(seg.rgb[0].cpu().numpy(), rgb[kept])
    near = seg.point_nearest.cpu().numpy()
    _, bi = _brute(pts, pts[kept])
    assert np.array_equal(near, bi.cpu().numpy()) and (near[~valid] == -1).all() and (near[valid] >= 0).all()

    gen = PointCloudMaskGenerator(model, points_per_cloud=32, points_per_batch=12, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    for kw in ({}, dict(crop_n_layers=1, min_mask_region_area=8)):
        ref = gen.generate_packed(seg.xyz, seg.rgb, **kw)
        out = seg.lift_packed(ref)  # the generator's output unchanged, plus the lifted fields
        assert all(out[k] is ref[k] for k in ref)
        whole = seg.generate_packed(gen, **kw)  # a second decode may round differently: compare the fields, not the values
        assert set(whole) == set(out)
        assert ("crop_box" in out) == ("crop_n_layers" in kw)
        bits, area = _u32(ref["bits"].cpu().numpy()), ref["area"].cpu().numpy()
        assert len(bits) > 0
        w_bits, w_area = mesh_ref.lift(bits, near, len(kept))
        assert np.array_equal(_u32(out["point_bits"].cpu().numpy()), w_bits)
        assert np.array_equal(out["point_area"].cpu().numpy(), w_area)
        labels = mesh_ref.label_map(bits, area, len(kept))
        assert np.array_equal(out["sample_labels"].cpu().numpy(), labels)
        want = np.where(near >= 0, labels[np.maximum(near, 0)], -1)
        assert np.array_equal(out["point_labels"].cpu().numpy(), want)
        assert torch.equal(out["sample_index"], seg.sample_index)

    # lifting and labels enqueue work only
    out = gen.generate_packed(seg.xyz, seg.rgb)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lifted = seg.lift_packed(out)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert lifted["point_bits"].shape == (len(out["area"]), (len(xyz) + 31) // 32)

    # prompted masks in scan coordinates; invalid points get -inf
    prompts = xyz[np.flatnonzero(valid)[[10, 4000, 9000]]]
    res = seg.predict_masks(prompts, np.array([1, 1, 0]))
    lg = res["logits"].cpu().numpy()
    pl = res["point_logits"].cpu().numpy()
    assert np.array_equal(pl[:, valid], lg[:, near[valid]]) and np.isneginf(pl[:, ~valid]).all()


def test_scan_segmenter_rejects_bad_scans():
    from pc_sam.scan import ScanSegmenter

    seg = ScanSegmenter(_models("base", 1), num_points=2048)
    with pytest.raises(ValueError, match="finite"):
        seg.set_scan(np.full((100, 3), np.nan, F32))
    with pytest.raises(ValueError, match="patches"):
        seg.set_scan(np.random.default_rng(0).uniform(-1, 1, (40, 3)).astype(F32))


def test_scan_segmenter_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam
    from pc_sam.scan import ScanSegmenter

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    xyz, rgb = synth.make_scan(10 ** 7, 11)
    valid = np.isfinite(xyz).all(1)
    seg = ScanSegmenter(model, num_points=32768, seed=1)
    seg.set_scan(_t(xyz), _t(rgb))
    gen = PointCloudMaskGenerator(model, points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    out = seg.generate_packed(gen)
    K = len(out["area"])
    assert K > 0
    near = seg.point_nearest.cpu().numpy()
    assert (near[valid] >= 0).all() and (near[~valid] == -1).all()
    lab = out["point_labels"].cpu().numpy()
    assert lab.shape == (len(xyz),) and lab.min() >= -1 and lab.max() < K and (lab[~valid] == -1).all()
    pb = out["point_bits"]
    pc = torch.zeros(K, dtype=torch.int64, device=DEV)
    for b in range(32):  # popcount of every row
        pc += ((pb >> b) & 1).sum(1)
    assert torch.equal(pc.to(torch.int32), out["point_area"])
