"""CPU tests of dense-scan segmentation: the numpy oracle of the voxel subsample (quantisation at cell edges and at +-1, level
counts that never decrease and the choice of L*, one representative per cell with the smallest (e, index), exactly S
outputs when thinning, seeds that change the selection but not the level, degenerate scans), the C ABI's argument checks
without a device, and the Python API's refusal of CPU tensors."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import scan_ref

F32 = np.float32


def _cloud(P, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (P, 3)).astype(F32)


def test_quantisation_at_cell_edges_and_bounds():
    x = F32([-1.0, -1.5, 1.0, 1.5, 0.0, -0.5, 2.0 ** -20 - 1, np.nextafter(F32(0), F32(-1)), 0.999999])
    xyz = np.stack([x, x, x], 1)
    q, valid = scan_ref.quantize(xyz)
    assert valid.all()
    # the fp32 add rounds first: nextafter(0, -1) + 1 = 1 exactly, so it lands in the cell above 0
    want = [0, 0, 2 ** 21 - 1, 2 ** 21 - 1, 2 ** 20, 2 ** 19, 1, 2 ** 20, int(np.floor((F32(0.999999) + F32(1)) * F32(2 ** 20)))]
    assert q[:, 0].tolist() == want
    # 1 + 2^-21 is exact in fp32 (half a cell above the edge: floor gives the edge's cell), 1 + 2^-25 rounds to 1
    assert scan_ref.quantize(F32([[2.0 ** -21, 2.0 ** -25, -2.0 ** -25]]))[0].tolist() == [[2 ** 20, 2 ** 20, 2 ** 20]]
    # non-finite rows are invalid
    _, valid = scan_ref.quantize(F32([[0, 0, np.nan], [np.inf, 0, 0], [0, 0, 0]]))
    assert valid.tolist() == [False, False, True]


def test_level_counts_never_decrease_and_choose_L_star():
    for xyz in (_cloud(5000, 0), _cloud(3, 1), np.zeros((10, 3), F32)):
        n = scan_ref.level_counts(xyz)
        assert n[0] == 1 and (np.diff(n) >= 0).all()
        for S in (1, 2, 8, 64, 4096, 10 ** 6):
            _, st = scan_ref.subsample(xyz, S)
            above = np.flatnonzero(n >= S)
            assert st[1] == (above[0] if len(above) else 21) and st[2] == n[st[1]]
            assert st[3] == min(S, st[2])


def test_one_representative_per_cell_with_smallest_e_then_index():
    rng = np.random.default_rng(3)
    xyz = _cloud(3000, 2)
    xyz[100:110] = xyz[5]  # duplicates of point 5: the lowest index wins
    idx, st = scan_ref.subsample(xyz, 10 ** 6)  # no thinning: every cell of level 21 (or the last level) is represented
    L = int(st[1])
    q, _ = scan_ref.quantize(xyz)
    keys, e = scan_ref.cell_keys(q, L), scan_ref.centre_dist(q, L)
    kept = idx[idx >= 0]
    assert len(np.unique(keys[kept])) == len(kept) == st[2]
    for j in rng.choice(kept, 50, replace=False):
        same = np.flatnonzero(keys == keys[j])
        best = same[np.lexsort((same, e[same]))[0]]
        assert best == j
    assert 5 in kept and not np.isin(np.arange(100, 110), kept).any()


def test_exactly_S_when_thinning_and_seed_changes_selection_not_level():
    xyz = _cloud(20000, 4)
    S = 500  # n_3 = 512 occupied cells
    a, sa = scan_ref.subsample(xyz, S, seed=0)
    b, sb = scan_ref.subsample(xyz, S, seed=12345)
    assert sa[2] > S and (a >= 0).sum() == S and (b >= 0).sum() == S
    assert (np.diff(a) > 0).all()
    assert sa[1] == sb[1] and sa[2] == sb[2] and not np.array_equal(a, b)


@pytest.mark.parametrize("kind", ["identical", "collinear", "planar", "nan_rows", "all_nan"])
def test_degenerate_scans(kind):
    rng = np.random.default_rng(5)
    P = 4000
    if kind == "identical":
        xyz = np.tile(F32([[0.25, -0.5, 0.1]]), (P, 1))
    elif kind == "collinear":
        t = rng.uniform(-1, 1, P).astype(F32)
        xyz = np.stack([t, t * F32(0.5), np.zeros_like(t)], 1)
    elif kind == "planar":
        xyz = _cloud(P, 6)
        xyz[:, 2] = F32(0.3)
    else:
        xyz = _cloud(P, 7)
        rows = rng.choice(P, P if kind == "all_nan" else 100, replace=False)
        xyz[rows, rng.integers(0, 3, len(rows))] = np.nan
        xyz[rows[: len(rows) // 2], 0] = np.inf
    for S in (1, 64, 1000, 5000):
        idx, st = scan_ref.subsample(xyz, S, seed=1)
        q, valid = scan_ref.quantize(xyz)
        kept = idx[idx >= 0]
        assert st[0] == valid.sum() and valid[kept].all() and len(kept) == st[3]
        if kind == "identical":
            assert st.tolist() == [P, 21 if S > 1 else 0, 1, 1] and kept.tolist() == [0]
        if kind == "all_nan":
            assert st.tolist() == [0, 21, 0, 0] and len(kept) == 0


# ------------------------------------------------------------------------------------------------
# the C ABI and the Python API without a device
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build, native

    build.build()
    return native.lib()


def test_argument_validation_without_gpu(lib):
    p = ctypes.c_void_p(16)  # never dereferenced: every call below is refused before any CUDA call
    ws = ctypes.c_void_p(32)
    assert lib.psam_nn_grid_workspace_bytes(0) == 0
    assert lib.psam_nn_grid_workspace_bytes(1000) >= 1000 * 24
    assert lib.psam_voxel_subsample_workspace_bytes(0) == 0
    assert lib.psam_voxel_subsample_workspace_bytes(1000) >= 1000 * 25 + 2048 * 20
    ok = dict(q=p, n1=5, k=p, n2=7, d=p, i=p, ws=ws)

    def nn(**kw):
        a = dict(ok, **kw)
        return lib.psam_nn_grid_f32(a["q"], a["n1"], a["k"], a["n2"], a["d"], a["i"], a["ws"], None)

    for bad in (dict(q=None), dict(k=None), dict(d=None), dict(ws=None), dict(n1=0), dict(n2=0), dict(n1=-3),
                dict(ws=ctypes.c_void_p(40))):
        assert nn(**bad) == -1, bad
    okv = dict(x=p, P=100, S=10, seed=0, i=p, st=p, ws=ws)

    def vox(**kw):
        a = dict(okv, **kw)
        return lib.psam_voxel_subsample_f32(a["x"], a["P"], a["S"], a["seed"], a["i"], a["st"], a["ws"], None)

    for bad in (dict(x=None), dict(i=None), dict(st=None), dict(ws=None), dict(P=0), dict(S=0), dict(S=-1),
                dict(ws=ctypes.c_void_p(24))):
        assert vox(**bad) == -1, bad


def test_python_api_refuses_cpu_tensors(lib):
    from pc_sam import scan
    from psam_b200 import ops

    x = torch.from_numpy(_cloud(64, 0))
    with pytest.raises(RuntimeError):
        ops.nearest_grid(x, x)
    with pytest.raises(RuntimeError):
        ops.voxel_subsample(x, 8)
    with pytest.raises(RuntimeError):
        scan.voxel_subsample(x, 8)
    with pytest.raises(ValueError):
        scan.voxel_subsample(x, 0)


def test_scan_segmenter_checks_before_the_device():
    from pc_sam.scan import ScanSegmenter

    seg = ScanSegmenter(torch.nn.Linear(1, 1), num_points=64)
    with pytest.raises(RuntimeError):
        seg.predict_masks(np.zeros((1, 3)), np.ones(1))
    with pytest.raises(RuntimeError):
        seg.lift_packed({})
    with pytest.raises(ValueError):
        ScanSegmenter(None, num_points=0)
    with pytest.raises(ValueError):
        seg.set_scan(np.zeros((0, 3), F32))


@pytest.mark.parametrize("names", [("red", "green", "blue"), ("R", "G", "B"), None])
def test_scan_from_ply(tmp_path, names):
    from pc_sam.scan import scan_from_ply

    xyz = _cloud(50, 8)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([(n, "u1") for n in names] if names else [])
    d = np.empty(len(xyz), dtype=fields)
    d["x"], d["y"], d["z"] = xyz.T
    col = (np.arange(150) % 256).astype(np.uint8).reshape(-1, 3)
    head = "ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n" % len(xyz)
    if names:
        for k, n in enumerate(names):
            d[n] = col[:, k]
            head += f"property uchar {n}\n"
    head += "end_header\n"
    path = tmp_path / "s.ply"
    with open(path, "wb") as fh:
        fh.write(head.encode())
        d.tofile(fh)
    got, rgb = scan_from_ply(str(path))
    assert np.array_equal(got, xyz)
    if names:
        assert np.array_equal(rgb, col.astype(F32) / F32(255))
    else:
        assert rgb is None
