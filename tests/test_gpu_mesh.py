"""GPU tests of mesh segmentation: the surface sampler equals the numpy oracle bit for bit (F = 1 to 2^20 + 3, degenerate,
NaN and tiny faces, every colour source, two seeds, repeated runs), bad meshes raise ValueError, mask lifting and label maps
equal the oracle bit for bit (K up to 16384, M up to 10^6, out-of-range nearest entries), nearest samples equal the C
oracle, MeshSegmenter returns the generator's output plus exact liftings for both model classes without extra host
synchronisation, and the invariants hold at full size (ViT-L, about 500k faces, 1024 prompts)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hier_ref, mesh_ref, tokenizer_ref, torch_ref  # noqa: E402
from psam_b200 import synth  # noqa: E402

DEV = torch.device("cuda:0")
F32 = np.float32


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _soup(F, seed, specials=True):
    """F random triangles over F + 2 vertices in [-1, 1], with degenerate, NaN-bearing and tiny faces mixed in."""
    rng = np.random.default_rng(seed)
    V = F + 2
    v = rng.uniform(-1, 1, (V, 3)).astype(F32)
    f = rng.integers(0, V, (F, 3)).astype(np.int32)
    if specials and F >= 7:
        f[1] = [f[1, 0], f[1, 0], f[1, 2]]                       # repeated vertex: zero area
        v[f[2, 1]] = v[f[2, 0]]                                  # coincident vertices
        v[f[3, 2]] = F32(np.nan)                                 # NaN vertex
        v[f[4, 1]] = v[f[4, 0]] + F32(1e-7)                      # tiny, possibly below 2^-32 of the largest
        v[f[4, 2]] = v[f[4, 0]] + F32([0, 1e-7, 0])
        v[f[5, 2]] = (v[f[5, 0]] + v[f[5, 1]]) * F32(0.5)        # collinear
    return v, f


def _check_sample(v, f, S, seed, **colour):
    from psam_b200 import ops

    dev_col = {k: _t(x) for k, x in colour.items()}
    xyz, rgb, face, stats = ops.mesh_sample(_t(v), _t(f), S, seed, **dev_col)
    w_xyz, w_rgb, w_face, w_stats = mesh_ref.sample(v, f, S, seed, **colour)
    assert stats.cpu().numpy().tolist() == w_stats.tolist()
    assert np.array_equal(face.cpu().numpy(), w_face)
    assert np.array_equal(_u32(xyz.cpu().numpy()), _u32(w_xyz))
    assert np.array_equal(_u32(rgb.cpu().numpy()), _u32(w_rgb))
    again = ops.mesh_sample(_t(v), _t(f), S, seed, **dev_col)
    assert all(torch.equal(a, b) for a, b in zip((xyz, rgb, face, stats), again))
    return w_face, w_stats


@pytest.mark.parametrize("F", [1, 7, 1000, 2 ** 20 + 3])
@pytest.mark.parametrize("seed", [0, 0xDEADBEEFCAFEF00D])
def test_sampler_bit_exact(F, seed):
    v, f = _soup(F, F)
    S = 32768 if F > 1000 else 4096
    face, stats = _check_sample(v, f, S, seed)
    if F >= 7:
        assert stats[1] >= 3  # the zero-area faces and the NaN face
        assert not np.isin([1, 2, 3], face).any()


@pytest.mark.parametrize("source", ["vertex", "texture3", "texture4"])
def test_sampler_colour_sources(source):
    v, f = _soup(1000, 5)
    rng = np.random.default_rng(9)
    if source == "vertex":
        _check_sample(v, f, 8192, 3, vertex_colors=rng.uniform(0, 1, (len(v), 3)).astype(F32))
    else:
        C = 3 if source == "texture3" else 4
        uv = rng.uniform(-0.1, 1.1, (len(v), 2)).astype(F32)  # some outside the image: clamped to the border texels
        uv[:8] = F32([[0, 0], [1, 1], [0, 1], [1, 0], [0.5, 0.5], [np.nan, 0.2], [0.999, 0.001], [1e-4, 0.9999]])
        _check_sample(v, f, 8192, 3, uv=uv, texture=rng.integers(0, 256, (37, 53, C)).astype(np.uint8))


def test_sampler_mesh_normalised_stays_in_unit_ball():
    from pc_sam.mesh import sample_surface

    v, f, _ = synth.make_mesh(20000, 1)
    from pc_sam.utils.ply import normalize_points

    vn = normalize_points(v.astype(np.float64)).astype(F32)
    xyz, _, face = sample_surface(_t(vn), _t(f), 32768, seed=4)
    assert float(xyz.abs().max()) <= 1
    w_xyz, _, w_face, _ = mesh_ref.sample(vn, f, 32768, 4)
    assert np.array_equal(_u32(xyz.cpu().numpy()), _u32(w_xyz)) and np.array_equal(face.cpu().numpy(), w_face)


def test_bad_meshes_raise():
    from pc_sam.mesh import sample_surface

    v, f = synth.make_sphere(6, 8)
    bad = f.copy()
    bad[3, 1] = len(v)
    with pytest.raises(ValueError, match="index"):
        sample_surface(_t(v), _t(bad), 64)
    bad[3, 1] = -1
    with pytest.raises(ValueError, match="index"):
        sample_surface(_t(v), _t(bad), 64)
    flat = np.zeros_like(v)
    with pytest.raises(ValueError, match="area"):
        sample_surface(_t(flat), _t(f), 64)
    from psam_b200 import ops

    xyz, rgb, face, stats = ops.mesh_sample(_t(flat), _t(f), 64)  # the kernel itself: face -1 and zeros
    assert (face == -1).all() and float(xyz.abs().max()) == 0 and float(rgb.abs().max()) == 0
    assert stats.tolist() == [0, len(f), 0]


def test_face_centers_bit_exact():
    from psam_b200 import ops

    v, f = _soup(5000, 2)
    f[7, 2] = len(v) + 3
    c = ops.mesh_face_centers(_t(v), _t(f)).cpu().numpy()
    w = mesh_ref.face_centers(v, f)
    nan = np.isnan(w)  # the bad face, and faces on the soup's NaN vertex (NaN payloads may differ)
    assert nan[7].all() and np.array_equal(np.isnan(c), nan)
    assert np.array_equal(_u32(c)[~nan], _u32(w)[~nan])


# ------------------------------------------------------------------------------------------------
# lifting and labels
# ------------------------------------------------------------------------------------------------
def _random_bits(K, S, seed):
    """K random masks over S points (S % 32 == 0) as words, of varied density; with K > 2 row 1 is empty and row 2 equals
    row 0 (equal areas: ties go to the lower index)."""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 2 ** 32, (K, S // 32), dtype=np.uint32)
    w[::2] &= rng.integers(0, 2 ** 32, (len(w[::2]), S // 32), dtype=np.uint32)
    w[::3] &= rng.integers(0, 2 ** 32, (len(w[::3]), S // 32), dtype=np.uint32)
    if K > 2:
        w[1] = 0
        w[2] = w[0]
    return w


@pytest.mark.parametrize("K,M", [(0, 33), (1, 1), (1, 1000000), (300, 33), (300, 1000000), (16384, 1), (16384, 33)])
def test_lift_and_labels_bit_exact(K, M):
    from psam_b200 import ops

    S = 32768
    rng = np.random.default_rng(K * 7 + M)
    bits = _random_bits(K, S, K)
    near = rng.integers(0, S, M).astype(np.int64)
    near[rng.uniform(0, 1, M) < 0.05] = -1                            # a target without a nearest sample
    near[rng.uniform(0, 1, M) < 0.02] = S + rng.integers(0, 5)        # out of range
    bd = _t(bits.view(np.int32))
    out, area = ops.mask_lift(bd, _t(near), S)
    w_out, w_area = mesh_ref.lift(bits, near, S)
    assert out.shape == (K, (M + 31) // 32)
    assert np.array_equal(_u32(out.cpu().numpy()), w_out) and np.array_equal(area.cpu().numpy(), w_area)
    if K <= 300:  # the label map over the lifted masks, priority = area (ties at rows 0 and 2)
        lab = ops.mask_label_map(out, area, M).cpu().numpy()
        assert np.array_equal(lab, mesh_ref.label_map(w_out, w_area, M))
    # and over the samples with random priorities, many equal
    pr = rng.integers(-3, 3, K).astype(np.int32)
    lab = ops.mask_label_map(bd, _t(pr), S).cpu().numpy()
    if K <= 300:
        assert np.array_equal(lab, mesh_ref.label_map(bits, pr, S))
    else:  # the oracle's dense form is too large here: check each label's rule directly on a sample of points
        idx = rng.choice(S, 256, replace=False)
        words = bits[:, idx >> 5] >> (idx & 31).astype(np.uint32) & 1
        for j, n in enumerate(idx):
            ks = np.flatnonzero(words[:, j])
            want = -1 if len(ks) == 0 else int(ks[np.lexsort((ks, pr[ks]))[0]])
            assert lab[n] == want


def test_nearest_samples_match_c_oracle():
    from pc_sam.mesh import nearest_samples, sample_surface

    v, f, _ = synth.make_mesh(20000, 3)
    from pc_sam.utils.ply import normalize_points

    vn = normalize_points(v.astype(np.float64)).astype(F32)
    xyz, _, _ = sample_surface(_t(vn), _t(f), 32768, seed=2)
    xs = xyz.cpu().numpy()
    # vertices, plus targets placed exactly on samples (one of them duplicated, so the lower index must win)
    rng = np.random.default_rng(0)
    on = xs[rng.choice(len(xs), 500, replace=False)]
    tgt = np.concatenate([vn, on, xs[:1]])
    got = nearest_samples(xyz, _t(tgt)).cpu().numpy()
    want = tokenizer_ref.knn(tgt[None], xs[None], 1)[0][0, :, 0]
    assert np.array_equal(got, want)


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
def test_mesh_segmenter_lifts_its_generator_call(kind):
    """MeshSegmenter end to end: the samples and nearest samples against the oracles, generate_packed = the generator's
    own call on the samples (recorded: its arguments, and every output key bit for bit) plus the lifted masks and labels
    against the oracles, no host synchronisation in the lifting, and prompted masks.  The generator's output is taken
    from the segmenter's own call rather than from a second run: the encoder's split-K GEMMs accumulate with float
    atomics, so two runs may differ in the last bits of a logit, and a mask bit whose logit lies that close to 0 with it."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.mesh import MeshSegmenter
    from pc_sam.utils.ply import normalize_points

    model = _models(kind, 3)
    v, f, col = synth.make_mesh(20000, 5)
    v = v * F32(3.5) + F32([1, -2, 0.5])  # not normalised: the segmenter normalises
    S = 2048
    seg = MeshSegmenter(model, num_points=S, seed=7)
    seg.set_mesh(v, f, vertex_colors=col)
    vn = normalize_points(v.astype(np.float64)).astype(F32)
    w_xyz, w_rgb, _, _ = mesh_ref.sample(vn, f, S, 7, vertex_colors=col)
    assert np.array_equal(_u32(seg.xyz[0].cpu().numpy()), _u32(w_xyz)) and np.array_equal(seg.rgb[0].cpu().numpy(), w_rgb)
    near_v = seg.vertex_nearest.cpu().numpy()
    near_f = seg.face_nearest.cpu().numpy()
    assert np.array_equal(near_v, tokenizer_ref.knn(vn[None], w_xyz[None], 1)[0][0, :, 0])
    assert np.array_equal(near_f, tokenizer_ref.knn(mesh_ref.face_centers(vn, f)[None], w_xyz[None], 1)[0][0, :, 0])

    gen = PointCloudMaskGenerator(model, points_per_cloud=32, points_per_batch=12, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    for kw in ({}, dict(crop_n_layers=1, min_mask_region_area=8)):
        calls = []
        run = gen.generate_packed

        def record(xyz, rgb, **k):
            assert xyz is seg.xyz and rgb is seg.rgb and k == kw
            res = run(xyz, rgb, **k)
            calls.append({name: t.clone() if torch.is_tensor(t) else t for name, t in res.items()})  # before the lifting
            return res

        gen.generate_packed = record
        try:
            out = seg.generate_packed(gen, **kw)
        finally:
            del gen.generate_packed
        assert len(calls) == 1
        ref = calls[0]
        assert set(ref) <= set(out)
        for k in ref:
            assert torch.equal(out[k], ref[k]) if torch.is_tensor(ref[k]) else out[k] == ref[k], k
        assert ("crop_box" in out) == ("crop_n_layers" in kw)
        bits = _u32(ref["bits"].cpu().numpy())
        area = ref["area"].cpu().numpy()
        assert len(bits) > 0
        for name, near, n in (("vertex", near_v, len(v)), ("face", near_f, len(f))):
            w_bits, w_area = mesh_ref.lift(bits, near, S)
            assert np.array_equal(_u32(out[f"{name}_bits"].cpu().numpy()), w_bits)
            assert np.array_equal(out[f"{name}_area"].cpu().numpy(), w_area)
        labels = mesh_ref.label_map(bits, area, S)
        assert np.array_equal(out["sample_labels"].cpu().numpy(), labels)
        assert np.array_equal(out["vertex_labels"].cpu().numpy(), labels[near_v])
        assert np.array_equal(out["face_labels"].cpu().numpy(), labels[near_f])
        assert np.allclose(out["shift"], v.astype(np.float64).mean(0)) and out["scale"] > 0

    # lifting and labels enqueue work only
    out = gen.generate_packed(seg.xyz, seg.rgb)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lifted = seg.lift_packed(out)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert lifted["vertex_bits"].shape == (len(out["area"]), (len(v) + 31) // 32)

    # prompted masks: prompts in mesh coordinates, logits gathered through the nearest samples
    prompts = v[[10, 4000, 9000]]
    res = seg.predict_masks(prompts, np.array([1, 1, 0]))
    logits, _, _ = model.predict_masks(_t(seg.normalize(prompts))[None], _t(np.array([[1, 1, 0]])), None, True)
    torch.testing.assert_close(res["logits"], logits[0], atol=1e-4, rtol=1e-4)
    lg = res["logits"].cpu().numpy()
    assert np.array_equal(res["vertex_logits"].cpu().numpy(), lg[:, near_v])
    assert np.array_equal(res["face_logits"].cpu().numpy(), lg[:, near_f])
    assert res["scores"].shape == (lg.shape[0],)


def test_mesh_segmenter_full_size_vit_l():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.mesh import MeshSegmenter
    from pc_sam.model import build_point_sam

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 512, 64).to(DEV).eval()
    v, f, col = synth.make_mesh(500000, 11)
    S = 32768
    seg = MeshSegmenter(model, num_points=S, seed=1)
    seg.set_mesh(v, f, vertex_colors=col)
    gen = PointCloudMaskGenerator(model, points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    out = seg.generate_packed(gen)
    K = len(out["area"])
    assert K > 0
    bits = _u32(out["bits"].cpu().numpy())
    for name, near, n in (("vertex", seg.vertex_nearest, len(v)), ("face", seg.face_nearest, len(f))):
        near = near.cpu().numpy()
        lab = out[f"{name}_labels"].cpu().numpy()
        lifted = _u32(out[f"{name}_bits"].cpu().numpy())
        area = out[f"{name}_area"].cpu().numpy()
        assert lab.shape == (n,) and lab.min() >= -1 and lab.max() < K
        # a labelled element lies in its mask
        e = np.flatnonzero(lab >= 0)
        assert ((lifted[lab[e], e >> 5] >> (e & 31).astype(np.uint32)) & 1).all()
        # area[k] = the elements whose nearest sample lies in sample mask k (rows in chunks)
        for k0 in range(0, K, 128):
            rows = bits[k0:k0 + 128]
            inside = (rows[:, near >> 5] >> (near & 31).astype(np.uint32)) & 1
            assert np.array_equal(inside.sum(1), area[k0:k0 + 128])
