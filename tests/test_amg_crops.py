"""CPU tests of the crop layers of automatic mask generation (crop_n_layers): the oracle's layout (coverage, layer 0 = the
cloud, the box formula, duplicate boxes on degenerate clouds), the renormalised crop cloud, the edge flags against a
per-point loop, uncrop against a plain scatter, the merge across crops, the generator's new parameters and argument
validation of the new C-ABI entries (before any CUDA call)."""
import ctypes
import inspect

import numpy as np
import pytest

from oracle import amg_crops_ref, amg_ref

F = np.float32


def _scene(N, seed):
    """A room-like cloud: a floor, two walls and boxes on the floor, thin along z."""
    rng = np.random.default_rng(seed)
    n1, n2 = N // 3, N // 3
    floor = np.c_[rng.uniform(-1, 1, (n1, 2)), np.full(n1, -0.2)]
    wall = np.c_[rng.uniform(-1, 1, n2), np.full(n2, 0.9), rng.uniform(-0.2, 0.25, n2)]
    c = rng.uniform(-0.8, 0.8, (6, 2))
    rest = N - n1 - n2
    k = rng.integers(0, 6, rest)
    objs = np.c_[c[k] + rng.uniform(-0.1, 0.1, (rest, 2)), rng.uniform(-0.2, 0.1, rest)]
    return np.concatenate([floor, wall, objs]).astype(F)[rng.permutation(N)]


@pytest.mark.parametrize("seed,layers,ratio", [(0, 1, amg_crops_ref.OVERLAP_RATIO), (1, 2, amg_crops_ref.OVERLAP_RATIO),
                                               (2, 3, 0.1), (3, 2, 0.9), (4, 1, 0.5)])
def test_layout_covers_every_point_and_layer0_is_the_cloud(seed, layers, ratio):
    rng = np.random.default_rng(seed)
    x = _scene(3000, seed) if seed % 2 else (rng.normal(0, 1, (3000, 3)) * [3, 1, 0.1] + [5, -2, 100]).astype(F)
    boxes, counts, layer = amg_crops_ref.layout(x, layers, ratio)
    assert len(boxes) == sum(8 ** i for i in range(layers + 1))
    bb = amg_crops_ref.bounding_box(x)
    assert np.array_equal(boxes[0], bb) and counts[0] == len(x)
    for lay in range(1, layers + 1):
        ts = np.nonzero(layer == lay)[0]
        assert len(ts) == 8 ** lay and np.all(counts[ts] >= 0)  # no zero-extent axis: no duplicates
        covered = np.zeros(len(x), bool)
        for t in ts:
            m = amg_crops_ref.members(x, boxes[t])
            assert m.sum() == counts[t]
            covered |= m
        assert covered.all(), lay
        lo, hi = boxes[ts, :3], boxes[ts, 3:]
        assert np.all(lo >= bb[:3]) and np.all(hi <= bb[3:] + 1e-5)
        assert np.all(lo.min(0) == bb[:3]) and np.all(hi.max(0) == bb[3:])  # first / last crops sit on the box exactly


def test_layout_box_formula():
    # unit cube, n = 2, r = 0.5: o = 0.5, s = 0.75 -> [0, 0.75] and [0.25, 1] on every axis; crop index (jx*2 + jy)*2 + jz
    x = np.array([[0, 0, 0], [1, 1, 1]], F)
    boxes, counts, _ = amg_crops_ref.layout(x, 1, 0.5)
    assert boxes[1].tolist() == [0, 0, 0, 0.75, 0.75, 0.75]
    assert boxes[1 + 4].tolist() == [0.25, 0, 0, 1, 0.75, 0.75]  # jx = 1
    assert boxes[1 + 1].tolist() == [0, 0, 0.25, 0.75, 0.75, 1]  # jz = 1
    assert boxes[8].tolist() == [0.25, 0.25, 0.25, 1, 1, 1]
    assert counts[1:].tolist() == [1, 0, 0, 0, 0, 0, 0, 1]
    # points exactly on a bound are members (closed boxes)
    assert amg_crops_ref.members(np.array([[0.75, 0.75, 0.75], [0.25, 0.25, 0.25]], F), boxes[1]).all()


def test_degenerate_clouds_give_deduplicated_boxes():
    rng = np.random.default_rng(0)
    flat = np.c_[rng.uniform(-1, 1, (500, 2)), np.zeros(500)].astype(F)  # zero extent along z
    boxes, counts, layer = amg_crops_ref.layout(flat, 2, amg_crops_ref.OVERLAP_RATIO)
    for lay, n in ((1, 2), (2, 4)):
        ts = np.nonzero(layer == lay)[0]
        jz = (ts - ts[0]) % n
        assert np.all(counts[ts[jz == 0]] >= 0) and np.all(counts[ts[jz > 0]] == -1)
        assert np.all(boxes[ts, 2] == 0) and np.all(boxes[ts, 5] == 0)
    same = np.tile(F([[0.25, -0.5, 0.125]]), (64, 1))  # coincident points: one box per layer
    boxes, counts, layer = amg_crops_ref.layout(same, 2, amg_crops_ref.OVERLAP_RATIO)
    for lay in (1, 2):
        ts = np.nonzero(layer == lay)[0]
        assert counts[ts[0]] == 64 and np.all(counts[ts[1:]] == -1)
    idx, xyz, _, edge = amg_crops_ref.crop_cloud(same, same, boxes, 1)
    assert len(idx) == 64 and np.all(xyz == 0) and not edge.any()  # scale 0 -> coordinates 0; no interior face


def test_nan_coordinates_are_ignored_by_the_box_and_lie_in_no_crop():
    x = _scene(2000, 3)
    x[[5, 17, 400]] = np.nan
    x[[9, 33], [1, 2]] = np.nan
    ok = ~np.isnan(x).any(1)
    boxes, counts, layer = amg_crops_ref.layout(x, 2, amg_crops_ref.OVERLAP_RATIO)
    assert np.array_equal(boxes[0], amg_crops_ref.bounding_box(x[ok])) and counts[0] == ok.sum()
    for lay in (1, 2):
        cover = np.zeros(len(x), bool)
        for t in np.nonzero(layer == lay)[0]:
            cover |= amg_crops_ref.members(x, boxes[t])
        assert np.array_equal(cover, ok)
    allnan = np.full((4, 3), np.nan, F)
    assert amg_crops_ref.bounding_box(allnan).tolist() == [np.inf] * 3 + [-np.inf] * 3


def test_crop_cloud_is_renormalised_in_ascending_order():
    x = _scene(4000, 5)
    rgb = np.random.default_rng(1).uniform(-1, 1, x.shape).astype(F)
    boxes, counts, _ = amg_crops_ref.layout(x, 2, amg_crops_ref.OVERLAP_RATIO)
    ts = [0] + [int(t) for t in np.nonzero(counts > 0)[0][1::6]]
    assert len(ts) > 4
    for t in ts:
        idx, cx, cr, edge = amg_crops_ref.crop_cloud(x, rgb, boxes, t)
        assert len(idx) == counts[t] and np.all(np.diff(idx) > 0)
        assert cx.dtype == np.float32 and np.abs(cx).max() <= 1 and np.isclose(np.linalg.norm(cx, axis=1).max(), 1, atol=1e-6)
        assert np.array_equal(cr, rgb[idx])
        if t == 0:
            assert not edge.any()


@pytest.mark.parametrize("seed", range(3))
def test_edge_flags_match_a_per_point_check(seed):
    x = _scene(1500, 10 + seed)
    boxes, _, layer = amg_crops_ref.layout(x, 2, amg_crops_ref.OVERLAP_RATIO)
    bb = boxes[0]
    for t in range(1, len(boxes)):
        idx, _, _, edge = amg_crops_ref.crop_cloud(x, x, boxes, t)
        box = boxes[t]
        for k, i in enumerate(idx):
            want = False
            for a in range(3):
                m = F(0.02) * F(bb[3 + a] - bb[a])
                if box[a] != bb[a] and F(x[i, a] - box[a]) <= m:
                    want = True
                if box[3 + a] != bb[3 + a] and F(box[3 + a] - x[i, a]) <= m:
                    want = True
            assert edge[k] == want, (t, k)
    # a point exactly on the margin counts as near
    box = np.array([0, 0, 0, 0.5, 1, 1], F)
    bb = np.array([0, 0, 0, 1, 1, 1], F)
    p = np.array([[0.25, 0.5, 0.5], [np.nextafter(np.nextafter(F(0.25), F(0)), F(0)), 0.5, 0.5], [0, 0, 0]], F)
    assert amg_crops_ref.edge_flags(p, box, bb, 0.25).tolist() == [True, False, False]


def test_edge_filter_and_uncrop_equal_a_scatter():
    rng = np.random.default_rng(3)
    N, n, K = 300, 70, 9
    idx = np.sort(rng.choice(N, n, replace=False))
    local = rng.random((K, n)) < 0.3
    local[4] = False
    bits = amg_ref.pack_bits(local)
    want = np.zeros((K, N), bool)
    for k in range(K):
        want[k, idx[local[k]]] = True
    g = amg_crops_ref.uncrop(bits, idx, N)
    assert g.shape == (K, (N + 31) // 32) and np.array_equal(amg_ref.unpack_bits(g, N), want)
    edge = np.zeros(n, bool)
    edge[[5, 60]] = True
    score = rng.uniform(0.5, 1, K).astype(F)
    got = amg_crops_ref.edge_filter(bits, score, amg_ref.pack_bits(edge[None])[0])
    hit = local[:, edge].any(1)
    assert np.array_equal(got == -np.inf, hit) and np.array_equal(got[~hit], score[~hit])


def test_merge_prefers_deeper_layers_and_keeps_slot_order():
    N = 64
    full = np.zeros((3, N), bool)
    full[0, :40] = True   # layer 0, slot 0
    full[1, 40:] = True   # layer 0, slot 1
    full[2, 2:40] = True  # layer 1: overlaps layer-0 mask 0 with IoU 38/40
    c0 = dict(crop=0, layer=0, idx=np.arange(N), bits=amg_ref.pack_bits(full[:2]), area=full[:2].sum(1), score=F([0.9, 0.8]),
              stability=F([1, 1]), keep=np.array([0, 1]), point_index=np.array([7]), slots=2)
    idx = np.arange(32)
    c1 = dict(crop=3, layer=1, idx=idx, bits=amg_ref.pack_bits(full[2:, :32]), area=np.array([30]), score=F([0.5]),
              stability=F([1]), keep=np.array([0]), point_index=np.array([5]), slots=1)
    c1["bits"] = amg_ref.pack_bits(full[2:, :32])
    m = amg_crops_ref.merge([c0, c1], N, 0.7, 16)
    assert m["crop"].tolist() == [0, 0, 3] and m["prompt"].tolist() == [7, 7, 5] and m["mask_slot"].tolist() == [0, 1, 0]
    assert m["keep"].tolist() == [2, 1]  # the layer-1 mask first; layer-0 mask 0 overlaps it (30/40 > 0.7)
    assert not m["overflow"]
    m = amg_crops_ref.merge([c0, c1], N, 0.7, 2)
    assert m["overflow"] and len(m["area"]) == 2


# ------------------------------------------------------------------------------------------------
# generator parameters
# ------------------------------------------------------------------------------------------------
def test_generator_crop_parameters():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    import torch

    defaults = dict(crop_n_layers=0, crop_nms_thresh=0.7, crop_overlap_ratio=512 / 1500, crop_n_points_downscale_factor=1)
    for fn in (PointCloudMaskGenerator.generate_packed, PointCloudMaskGenerator.generate, PointCloudMaskGenerator._enqueue):
        prm = inspect.signature(fn).parameters
        for k, v in defaults.items():
            assert prm[k].kind is inspect.Parameter.KEYWORD_ONLY and prm[k].default == v, (fn, k)
    assert PointCloudMaskGenerator.crop_edge_margin == amg_crops_ref.EDGE_MARGIN
    assert PointCloudMaskGenerator._crop_args(3, 0.5, 0.0, 2) == (3, 0.5, 0.0, 2)
    g = PointCloudMaskGenerator(object())  # the checks come before the model is touched
    for kw in (dict(crop_n_layers=-1), dict(crop_n_layers=4), dict(crop_overlap_ratio=1.0), dict(crop_overlap_ratio=-0.1),
               dict(crop_n_points_downscale_factor=0), dict(crop_nms_thresh=-0.1), dict(crop_nms_thresh=1.5),
               dict(crop_nms_thresh=float("nan"))):
        with pytest.raises(ValueError):
            g.generate_packed(torch.zeros(16, 3), torch.zeros(16, 3), **kw)
        with pytest.raises(ValueError):
            g.generate(torch.zeros(16, 3), torch.zeros(16, 3), **kw)
    g = PointCloudMaskGenerator(object(), points_per_cloud=100)
    assert [g._crop_prompts(4, i, 1000) for i in range(4)] == [100, 25, 6, 1] and g._crop_prompts(4, 1, 7) == 7


# ------------------------------------------------------------------------------------------------
# C ABI: argument validation before any CUDA call
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    for name in ("psam_crop_total", "psam_crop_layout_f32", "psam_crop_gather_f32", "psam_crop_edge_filter", "psam_crop_uncrop"):
        getattr(L, name).restype = ctypes.c_int
    L.psam_crop_gather_workspace_bytes.restype = ctypes.c_size_t
    return L


def test_crop_total_and_workspace(lib):
    from psam_b200 import ops

    assert [lib.psam_crop_total(ctypes.c_int(k)) for k in range(-1, 5)] == [0, 1, 9, 73, 585, 0]
    assert [ops.crop_total(k) for k in range(4)] == [1, 9, 73, 585] and ops.CROP_MAX_LAYERS == 3
    ws = lambda n: lib.psam_crop_gather_workspace_bytes(ctypes.c_int(n))  # noqa: E731
    assert ws(0) == 0 and ws(1) == 24 and ws(1024) == 24 and ws(1025) == 32 and ws(262144) == 256 * 8 + 16


def test_crop_layout_argument_validation_without_gpu(lib):
    i, p, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
    fake = p(0x1000)

    def call(x=fake, N=100, L=1, r=0.3, boxes=fake, counts=fake):
        return lib.psam_crop_layout_f32(x, i(N), i(L), f(r), boxes, counts, None)

    for kw in (dict(x=None), dict(boxes=None), dict(counts=None), dict(N=0), dict(N=-1), dict(L=-1), dict(L=4), dict(r=1.0),
               dict(r=-0.01), dict(r=float("nan"))):
        assert call(**kw) == -1, kw


def test_crop_gather_argument_validation_without_gpu(lib):
    i, p, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
    fake = p(0x1000)

    def call(x=fake, c=fake, N=100, boxes=fake, crop=3, T=9, m=0.02, n=10, idx=fake, xo=fake, co=fake, edge=fake, ws=fake):
        return lib.psam_crop_gather_f32(x, c, i(N), boxes, i(crop), i(T), f(m), i(n), idx, xo, co, edge, ws, None)

    for kw in (dict(x=None), dict(c=None), dict(boxes=None), dict(idx=None), dict(xo=None), dict(co=None), dict(edge=None),
               dict(ws=None), dict(N=0), dict(crop=-1), dict(crop=9), dict(T=0), dict(m=-0.1), dict(m=float("nan")), dict(n=0),
               dict(n=101), dict(ws=p(0x1008))):
        assert call(**kw) == -1, kw


def test_crop_edge_filter_argument_validation_without_gpu(lib):
    i, p = ctypes.c_int, ctypes.c_void_p
    fake = p(0x1000)

    def call(bits=fake, K=10, W=2, edge=fake, score=fake):
        return lib.psam_crop_edge_filter(bits, i(K), i(W), edge, score, None)

    for kw in (dict(bits=None), dict(edge=None), dict(score=None), dict(K=-1), dict(W=0)):
        assert call(**kw) == -1, kw
    assert call(K=0, bits=None, edge=None, score=None) == 0  # nothing to do, nothing launched


def test_crop_uncrop_argument_validation_without_gpu(lib):
    i, p, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
    fake = p(0x1000)
    ptrs = ("bits", "area", "score", "stab", "keep", "cnt", "idx", "prompt", "oin", "oout", "gbits", "garea", "giou", "gstab",
            "gprompt", "gslot", "gcrop", "gscore", "over")

    def call(K=30, W=2, n=40, slots=3, crop=1, N=100, Wg=4, cap=64, **kw):
        a = {k: kw.get(k, fake) for k in ptrs}
        return lib.psam_crop_uncrop(a["bits"], a["area"], a["score"], a["stab"], i(K), i(W), a["keep"], a["cnt"], a["idx"], i(n),
                                    a["prompt"], i(slots), i(crop), f(1.0), i(N), i(Wg), i(cap), a["oin"], a["oout"], a["gbits"],
                                    a["garea"], a["giou"], a["gstab"], a["gprompt"], a["gslot"], a["gcrop"], a["gscore"], a["over"],
                                    None)

    for k in ptrs:
        assert call(**{k: None}) == -1, k
    for kw in (dict(K=0), dict(n=0), dict(n=101), dict(W=1), dict(slots=0), dict(crop=-1), dict(Wg=3), dict(cap=0), dict(cap=16385)):
        assert call(**kw) == -1, kw
