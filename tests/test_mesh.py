"""CPU tests of mesh segmentation: the numpy oracle of the mesh kernels (samples on their faces and inside [-1, 1], face
counts that follow area, faces never chosen, the texel rule at the image borders, the hash and mulhi against Python
integers, lifting and label maps on hand-made cases), the C ABI's argument checks without a device, and the Python API's
refusal of CPU tensors."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mesh_ref

F32 = np.float32


def _sphere(n_lat=12, n_lon=24):
    """A closed UV sphere of radius 1 centred on the origin."""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    v = [[0, 0, 1]] + [[np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)] for t in th for p in ph] + [[0, 0, -1]]
    ring = lambda i, j: 1 + i * n_lon + j % n_lon  # noqa: E731
    f = [[0, ring(0, j), ring(0, j + 1)] for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    last = len(v) - 1
    f += [[ring(n_lat - 2, j), last, ring(n_lat - 2, j + 1)] for j in range(n_lon)]
    return np.asarray(v, F32), np.asarray(f, np.int32)


# ------------------------------------------------------------------------------------------------
# the oracle itself
# ------------------------------------------------------------------------------------------------
def test_hash_and_mulhi_match_python_integers():
    rng = np.random.default_rng(0)
    M = 2 ** 64
    seed = int(rng.integers(0, 2 ** 63)) * 2 + 1
    s = np.arange(50, dtype=np.uint64)
    for j in range(3):
        got = mesh_ref.hash_stream(seed, s, j)
        for k in range(50):
            z = (seed + (3 * k + j + 1) * 0x9E3779B97F4A7C15) % M
            z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % M
            z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % M
            assert int(got[k]) == z ^ (z >> 31)
    a = rng.integers(0, 2 ** 63, 200, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    for b in (1, 12345, 2 ** 32 - 1, 2 ** 32 + 7, 2 ** 62 + 3):
        got = mesh_ref.mulhi(a, b)
        assert [int(x) for x in got] == [(int(x) * b) >> 64 for x in a]


def test_samples_lie_on_their_faces_inside_unit_ball():
    v, f = _sphere()
    xyz, rgb, face, stats = mesh_ref.sample(v, f, 4000, seed=3)
    assert stats.tolist()[1:] == [0, 0] and (face >= 0).all()
    assert np.abs(xyz).max() <= 1 and (rgb == F32(0.5)).all()
    a, b, c = (v[f[face, k]].astype(np.float64) for k in range(3))
    # barycentric reconstruction: p - a = s (b - a) + t (c - a) with s, t >= 0, s + t <= 1, and no offset from the plane
    e1, e2, d = b - a, c - a, xyz.astype(np.float64) - a
    n = np.cross(e1, e2)
    assert np.abs((d * n).sum(1)).max() <= 1e-6 * np.linalg.norm(n, axis=1).max()
    g = np.stack([(e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)], 1)
    r = np.stack([(d * e1).sum(1), (d * e2).sum(1)], 1)
    det = g[:, 0] * g[:, 2] - g[:, 1] ** 2
    s_ = (g[:, 2] * r[:, 0] - g[:, 1] * r[:, 1]) / det
    t_ = (g[:, 0] * r[:, 1] - g[:, 1] * r[:, 0]) / det
    tol = 1e-4
    assert (s_ >= -tol).all() and (t_ >= -tol).all() and (s_ + t_ <= 1 + tol).all()
    # the clamp keeps every sample inside the box of its face
    lo, hi = np.minimum(np.minimum(a, b), c), np.maximum(np.maximum(a, b), c)
    assert (xyz >= lo).all() and (xyz <= hi).all()


def test_face_counts_follow_area():
    """Right triangles of areas 1e-6 .. 1 (log-spaced): counts over many samples follow the area."""
    areas = np.logspace(-6, 0, 13)
    v, f = [], []
    for i, A in enumerate(areas):
        s = np.sqrt(2 * A)
        v += [[i * 2.0, 0, 0], [i * 2.0 + s, 0, 0], [i * 2.0, s, 0]]
        f.append([3 * i, 3 * i + 1, 3 * i + 2])
    v, f = np.asarray(v, F32), np.asarray(f, np.int32)
    S = 400000
    _, _, face, _ = mesh_ref.sample(v, f, S, seed=11)
    counts = np.bincount(face, minlength=len(f))
    p = areas / areas.sum()
    expect = S * p
    sd = np.sqrt(S * p * (1 - p))
    assert (np.abs(counts - expect) <= 5 * sd + 1).all(), (counts, expect)


def test_zero_area_and_tiny_faces_are_never_chosen():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 2], [1e-8, 0, 0], [0, 1e-8, 0], [np.nan, 0, 0]], F32)
    f = np.array([[0, 1, 2],      # area 0.5
                  [0, 1, 1],      # degenerate (repeated vertex)
                  [0, 1, 3],      # fine
                  [0, 4, 5],      # 5e-17: below 2^-32 of the largest, weight 0 but not bad
                  [0, 1, 6],      # NaN vertex: bad
                  [0, 1, 7],      # index out of range: bad
                  [0, 0, 0]], np.int32)
    q, cdf, stats = mesh_ref.weights(v, f)
    assert q[1] == 0 and q[3] == 0 and q[4] == 0 and q[5] == 0 and q[6] == 0
    assert q[0] > 0 and q[2] > 0 and max(q) <= 2 ** 32 - 1
    assert stats.tolist() == [int(q.sum()), 4, 1]
    _, _, face, _ = mesh_ref.sample(v, f, 20000, seed=5)
    assert set(np.unique(face).tolist()) == {0, 2}


def test_empty_mesh_gives_minus_one():
    v = np.zeros((3, 3), F32)
    xyz, rgb, face, stats = mesh_ref.sample(v, np.array([[0, 1, 2]], np.int32), 10)
    assert stats.tolist() == [0, 1, 0] and (face == -1).all() and (xyz == 0).all() and (rgb == 0).all()


def test_texel_rule_at_image_borders():
    W = 4
    t = F32([-1.0, 0.0, 0.124, 0.125, 0.375, 0.875, 0.99, 1.0, 2.0, np.nan, np.inf, -np.inf])
    assert mesh_ref.texel(t, W).tolist() == [0, 0, 0, 1, 2, 3, 3, 3, 3, 0, 3, 0]
    # on a one-texel mesh: a face whose uv sits at the corners reads the corner texels (v = 1 - y)
    tex = np.arange(2 * 3 * 4, dtype=np.uint8).reshape(2, 3, 4) * 10
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F32)
    for (u, vv), (y, x) in [((0, 1), (0, 0)), ((1, 1), (0, 2)), ((0, 0), (1, 0)), ((1, 0), (1, 2))]:
        uv = np.tile(F32([[u, vv]]), (3, 1))
        _, rgb, _, _ = mesh_ref.sample(v, np.array([[0, 1, 2]], np.int32), 4, uv=uv, texture=tex)
        assert (rgb == tex[y, x, :3].astype(F32) / F32(255)).all()


def test_lift_hand_made():
    S = 40
    m = np.zeros((3, S), bool)
    m[0, [0, 5, 39]] = True
    m[1, 5:10] = True
    bits = mesh_ref.pack(m)
    for M in (1, 31, 32, 33):
        near = np.arange(M) % S
        near[M - 1] = 5
        if M > 2:
            near[1] = -3  # out of range reads as 0
        if M > 3:
            near[2] = S   # so does S itself
        out, area = mesh_ref.lift(bits, near, S)
        assert out.shape == (3, (M + 31) // 32)
        got = mesh_ref.unpack(out, 32 * out.shape[1])
        assert not got[:, M:].any()
        want = np.zeros((3, M), bool)
        ok = (near >= 0) & (near < S)
        want[:, ok] = m[:, near[ok]]
        assert (got[:, :M] == want).all() and area.tolist() == want.sum(1).tolist()
    out, area = mesh_ref.lift(np.zeros((0, 2), np.uint32), np.zeros(5, np.int64), S)
    assert out.shape == (0, 1) and area.shape == (0,)


def test_label_map_hand_made():
    N = 33
    m = np.zeros((4, N), bool)
    m[0, :20] = True          # area 20
    m[1, 10:15] = True        # area 5
    m[2, 12:17] = True        # area 5: ties with 1 -> lower index wins on 12..14
    m[3, 32] = True           # area 1, the last word's only point
    area = m.sum(1)
    lab = mesh_ref.label_map(mesh_ref.pack(m), area, N)
    want = [0] * 10 + [1] * 5 + [2] * 2 + [0] * 3 + [-1] * 12 + [3]
    assert lab.tolist() == want
    # priority decides, not area: with priorities reversed the biggest mask wins where it overlaps
    assert mesh_ref.label_map(mesh_ref.pack(m), -area, N)[10:20].tolist() == [0] * 10
    assert (mesh_ref.label_map(np.zeros((0, 2), np.uint32), np.zeros(0, np.int32), N) == -1).all()


def test_face_centers():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.5]], F32)
    c = mesh_ref.face_centers(v, np.array([[0, 1, 2], [0, 1, 3]], np.int32))
    assert np.array_equal(c[0], ((v[0] + v[1]) + v[2]) / F32(3)) and np.isnan(c[1]).all()


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
    assert lib.psam_mesh_sample_workspace_bytes(0) == 0
    assert lib.psam_mesh_sample_workspace_bytes(1000) >= 1000 * 12
    ok = dict(vertices=p, V=3, faces=p, F=1, S=8, seed=0, vc=None, uv=None, tex=None, h=0, w=0, c=0, xyz=p, rgb=p, face=p,
              stats=p, ws=ws)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.psam_mesh_sample_f32(a["vertices"], a["V"], a["faces"], a["F"], a["S"], a["seed"], a["vc"], a["uv"], a["tex"],
                                        a["h"], a["w"], a["c"], a["xyz"], a["rgb"], a["face"], a["stats"], a["ws"], None)

    for bad in (dict(vertices=None), dict(V=0), dict(F=0), dict(S=0), dict(stats=None), dict(ws=None), dict(ws=ctypes.c_void_p(40)),
                dict(uv=p), dict(tex=p, uv=None, h=2, w=2, c=3), dict(tex=p, uv=p, h=2, w=2, c=2), dict(tex=p, uv=p, h=0, w=2, c=3),
                dict(tex=p, uv=p, vc=p, h=2, w=2, c=4)):
        assert call(**bad) == -1, bad
    assert lib.psam_mesh_face_centers_f32(p, 0, p, 1, p, None) == -1
    assert lib.psam_mesh_face_centers_f32(p, 3, p, 1, None, None) == -1
    # mask_lift: K < 0, Ws too small for S, Wm too small for M, M = 0; K = 0 is a no-op
    assert lib.psam_mask_lift(p, -1, 1, 32, p, 1, 1, p, p, None) == -1
    assert lib.psam_mask_lift(p, 1, 1, 33, p, 1, 1, p, p, None) == -1
    assert lib.psam_mask_lift(p, 1, 2, 33, p, 33, 1, p, p, None) == -1
    assert lib.psam_mask_lift(p, 1, 1, 32, p, 0, 1, p, p, None) == -1
    assert lib.psam_mask_lift(p, 1, 1, 32, None, 1, 1, p, p, None) == -1
    assert lib.psam_mask_lift(None, 0, 1, 32, p, 1, 1, None, None, None) == 0
    # label map: K < 0, N = 0, W too small, missing priority
    assert lib.psam_mask_label_map(p, -1, 1, p, 1, p, None) == -1
    assert lib.psam_mask_label_map(p, 1, 1, p, 0, p, None) == -1
    assert lib.psam_mask_label_map(p, 1, 1, p, 33, p, None) == -1
    assert lib.psam_mask_label_map(p, 1, 1, None, 1, p, None) == -1
    assert lib.psam_mask_label_map(p, 1, 1, p, 1, None, None) == -1


def test_python_api_refuses_cpu_tensors(lib):
    from pc_sam import mesh

    v, f = _sphere(4, 6)
    vt, ft = torch.from_numpy(v), torch.from_numpy(f)
    with pytest.raises(RuntimeError):
        mesh.sample_surface(vt, ft, 16)
    with pytest.raises(RuntimeError):
        mesh.nearest_samples(vt, vt)
    with pytest.raises(RuntimeError):
        mesh.lift_masks(torch.zeros((2, 1), dtype=torch.int32), torch.zeros(4, dtype=torch.int64), 8)
    with pytest.raises(RuntimeError):
        mesh.mask_labels(torch.zeros((2, 1), dtype=torch.int32), torch.zeros(2, dtype=torch.int32), 8)
    from psam_b200 import ops

    with pytest.raises(RuntimeError):
        ops.mesh_face_centers(vt, ft)


def test_mesh_segmenter_checks_before_the_device():
    from pc_sam.mesh import MeshSegmenter

    seg = MeshSegmenter(torch.nn.Linear(1, 1), num_points=64)
    v, f = _sphere(4, 6)
    bad = v.copy()
    bad[2, 1] = np.inf
    with pytest.raises(ValueError):
        seg.set_mesh(bad, f)
    with pytest.raises(ValueError):
        seg.set_mesh(np.zeros((4, 3), F32), f[:2] % 4)
    with pytest.raises(RuntimeError):
        seg.predict_masks(np.zeros((1, 3)), np.ones(1))
    with pytest.raises(ValueError):
        MeshSegmenter(None, num_points=0)


def test_mesh_from_ply(tmp_path):
    from pc_sam.mesh import mesh_from_ply

    v, f = _sphere(4, 6)
    col = (np.arange(len(v) * 3) % 256).astype(np.uint8).reshape(-1, 3)
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
            "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\n"
            "property list uchar int vertex_indices\nend_header\n" % (len(v), len(f)))
    vd = np.empty(len(v), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vd["x"], vd["y"], vd["z"] = v.T
    vd["red"], vd["green"], vd["blue"] = col.T
    fd = np.empty(len(f), dtype=[("k", "u1"), ("v", "<i4", (3,))])
    fd["k"], fd["v"] = 3, f
    path = tmp_path / "m.ply"
    with open(path, "wb") as fh:
        fh.write(head.encode())
        vd.tofile(fh)
        fd.tofile(fh)
    vv, ff, cc = mesh_from_ply(str(path))
    assert np.array_equal(vv, v) and np.array_equal(ff, f) and ff.dtype == np.int32
    assert np.array_equal(cc, col.astype(F32) / F32(255))
