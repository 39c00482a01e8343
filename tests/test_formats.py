"""CPU tests of the data formats and callers either side of the hot path: PLY readers,
input normalisation, safetensors checkpoints, the hydra-style config instantiation and the demo wire format."""
import json
import os
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "point-sam_b200"))
sys.path.insert(0, ROOT)

from pc_sam.utils import checkpoint, config, ply  # noqa: E402


def _kitti_like(n, seed=0):
    r = np.random.default_rng(seed)
    return {"x": r.normal(size=n).astype(np.float32), "y": r.normal(size=n).astype(np.float32),
            "z": (0.15 * r.normal(size=n)).astype(np.float32), "R": r.integers(0, 256, n).astype(np.uint8),
            "G": r.integers(0, 256, n).astype(np.uint8), "B": r.integers(0, 256, n).astype(np.uint8),
            "label": r.integers(0, 2, n).astype(np.int32)}


@pytest.mark.parametrize("fmt,ext", [("binary_little_endian", "<"), ("binary_big_endian", ">")])
def test_read_binary_ply_hand_built(tmp_path, fmt, ext):
    """File assembled byte by byte here (not with the package's writer): header as KITTI-360 crops carry it."""
    d = _kitti_like(257, 1)
    head = ("ply\nformat %s 1.0\ncomment crop\nelement vertex 257\nproperty float x\nproperty float y\nproperty float z\n"
            "property uchar R\nproperty uchar G\nproperty uchar B\nproperty int label\nend_header\n" % fmt).encode()
    rec = np.empty(257, dtype=[("x", ext + "f4"), ("y", ext + "f4"), ("z", ext + "f4"), ("R", "u1"), ("G", "u1"), ("B", "u1"),
                               ("label", ext + "i4")])
    for k in d:
        rec[k] = d[k]
    p = tmp_path / "crop.ply"
    p.write_bytes(head + rec.tobytes())
    got = ply.read_ply(str(p))
    assert got.dtype.names == ("x", "y", "z", "R", "G", "B", "label")
    for k in d:
        assert np.array_equal(got[k], d[k]), k
    # truncated payload and ASCII input are refused like the reference reader does
    (tmp_path / "bad.ply").write_bytes(head + rec.tobytes()[:-5])
    with pytest.raises(ValueError):
        ply.read_ply(str(tmp_path / "bad.ply"))
    (tmp_path / "notply.ply").write_bytes(b"plx\n")
    with pytest.raises(ValueError):
        ply.read_ply(str(tmp_path / "notply.ply"))


def test_ply_writer_roundtrip_mesh_and_ascii(tmp_path):
    d = _kitti_like(100, 2)
    for fmt in ("binary_little_endian", "binary_big_endian", "ascii"):
        p = str(tmp_path / f"{fmt}.ply")
        ply.write_ply(p, d, fmt)
        if fmt == "ascii":
            with pytest.raises(ValueError):
                ply.read_ply(p)
        got = ply.read_ply(p, allow_ascii=True)
        for k in d:
            assert np.allclose(got[k], d[k], rtol=0, atol=0 if fmt != "ascii" else 1e-6), (fmt, k)
    # triangular mesh: vertex element + uchar/int face lists
    v = np.arange(12, dtype="<f4").reshape(4, 3)
    head = b"ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\n" \
           b"element face 2\nproperty list uchar int vertex_indices\nend_header\n"
    faces = b"".join(struct.pack("<Biii", 3, *f) for f in [(0, 1, 2), (1, 2, 3)])
    (tmp_path / "mesh.ply").write_bytes(head + v.tobytes() + faces)
    vd, fd = ply.read_ply(str(tmp_path / "mesh.ply"), triangular_mesh=True)
    assert np.array_equal(np.stack([vd["x"], vd["y"], vd["z"]], 1), v) and fd.tolist() == [[0, 1, 2], [1, 2, 3]]
    # demo loader: 6 ASCII columns
    body = "\n".join("%f %f %f %d %d %d" % (i, 2 * i, 3 * i, i % 256, 7, 9) for i in range(50))
    (tmp_path / "scene.ply").write_text("ply\nformat ascii 1.0\nelement vertex 50\nproperty float x\nproperty float y\n"
                                        "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
                                        "end_header\n" + body + "\n")
    pts = ply.load_ply(str(tmp_path / "scene.ply"))
    assert pts.shape == (50, 6) and pts[7].tolist() == [7.0, 14.0, 21.0, 7.0, 7.0, 9.0]


def test_normalisation_matches_reference_formulas():
    r = np.random.default_rng(3)
    pts = r.normal(size=(1000, 3)) * [3.0, 1.0, 0.2] + [10.0, -4.0, 2.0]
    n = ply.normalize_points(pts)
    assert abs(np.linalg.norm(n, axis=1).max() - 1.0) < 1e-12 and np.abs(n.mean(0)).max() < 1e-12
    c = ply.normalize_colors(np.array([[0.0, 127.5, 255.0]]))
    assert np.allclose(c, [[-1.0, 0.0, 1.0]])
    assert np.allclose(ply.normalize_colors(np.array([[255.0]]), mean=None, std=None), [[1.0]])


def test_safetensors_reader_writer(tmp_path):
    g = torch.Generator().manual_seed(0)
    tensors = {"a.weight": torch.randn(7, 5, generator=g), "a.bias": torch.randn(5, generator=g),
               "b.idx": torch.arange(11, dtype=torch.int64), "c.half": torch.randn(3, 2, generator=g).to(torch.bfloat16),
               "d.empty": torch.zeros(0, 4)}
    p = str(tmp_path / "m.safetensors")
    checkpoint.save_file(tensors, p, metadata={"format": "pt"})
    got = checkpoint.load_file(p)
    assert set(got) == set(tensors)
    for k in tensors:
        assert got[k].dtype == tensors[k].dtype and torch.equal(got[k], tensors[k]), k
    try:
        from safetensors.torch import load_file as st_load, save_file as st_save
    except ImportError:
        return
    # interoperability with the real library in both directions
    theirs = st_load(p)
    for k in tensors:
        assert torch.equal(theirs[k], tensors[k]), k
    p2 = str(tmp_path / "theirs.safetensors")
    st_save({k: v for k, v in tensors.items()}, p2)
    mine = checkpoint.load_file(p2)
    for k in tensors:
        assert torch.equal(mine[k], tensors[k]), k


def test_config_instantiate_and_checkpoint_keys(tmp_path):
    """A YAML tree with the reference's schema (configs/model/*.yaml) instantiates the mirror modules; the state-dict
    keys equal those of the oracle restatement (which the golden generator pins against the reference's modules), and a
    checkpoint written with those keys loads strictly."""
    from pc_sam.model.eva import EVA_CONFIGS
    from oracle import torch_ref

    name = "eva02_test_tiny"
    assert name in EVA_CONFIGS
    d = tmp_path / "configs"
    (d / "model").mkdir(parents=True)
    cfg = config.model_config("base")
    cfg["pc_encoder"]["transformer"]["model_name"] = name
    cfg["pc_encoder"]["patch_embed"].update(num_patches=16, patch_size=8)
    import yaml

    (d / "model" / "tiny.yaml").write_text(yaml.safe_dump(cfg))
    (d / "tiny.yaml").write_text("defaults:\n  - model: tiny\n  - dataset@train_dataset: partnet\nlr: 3e-4\nrun_name: x\nproject_dir: ./logs/${run_name}\n")
    full = config.compose(str(d), "tiny", ["model.prompt_iters=3", "model.pc_encoder.patch_embed.num_patches=24"])
    assert full["lr"] == 3e-4 and full["model"]["prompt_iters"] == 3
    model = config.instantiate(full["model"])
    assert model.prompt_iters == 3 and model.pc_encoder.patch_embed.grouper.num_groups == 24
    ref = torch_ref.build_model(name, 24, 8, seed=5)
    assert list(model.state_dict().keys()) == list(ref.state_dict().keys())
    p = str(tmp_path / "model.safetensors")
    checkpoint.save_file(ref.state_dict(), p)
    checkpoint.load_model(model, p)
    for k, v in ref.state_dict().items():
        assert torch.equal(model.state_dict()[k], v), k
    bad = dict(ref.state_dict())
    bad.pop(next(iter(bad)))
    bad["extra.weight"] = torch.zeros(1)
    checkpoint.save_file(bad, p)
    with pytest.raises(RuntimeError):
        checkpoint.load_model(model, p)
    assert config.model_config("large")["pc_encoder"]["patch_embed"]["num_patches"] == 1024
    assert config.model_config("giant")["pc_encoder"]["transformer"]["model_name"] == "eva_giant_patch14_560"


def test_eval_helpers_cpu(tmp_path):
    from evaluation import eval_kitti

    d = _kitti_like(300, 4)
    p = str(tmp_path / "car_0001.ply")
    ply.write_ply(p, d)
    crop = eval_kitti.load_crop(p)
    assert crop["xyz"].dtype == np.float32 and crop["xyz"].shape == (300, 3) and crop["mask"].dtype == np.int32
    data = eval_kitti.transform_fn(crop, device="cpu")
    assert data["coords"].shape == (1, 300, 3) and data["gt_masks"].shape == (1, 1, 300) and data["gt_masks"].dtype == torch.bool
    assert abs(float(data["coords"].norm(dim=-1).max()) - 1.0) < 1e-6 and float(data["features"].abs().max()) <= 1.0

    class G:  # grouper stand-in
        num_groups, group_size = 0, 0

    class M:
        class pc_encoder:
            class patch_embed:
                grouper = G()

    for n, want in [(40000, (2048, 256)), (5000, (2048, 256)), (1000, (1000, 256)), (100, (100, 2))]:
        eval_kitti.set_group_shape(M, n)
        g = M.pc_encoder.patch_embed.grouper
        assert (g.num_groups, g.group_size) == want


def test_demo_http_routes_wire_format(tmp_path):
    """The stdlib HTTP front end of the demo: route names, JSON bodies and error mapping of demo/app.py (a stub session
    stands in for the CUDA-backed SegmentSession; the session itself is covered by the GPU tests)."""
    import threading
    import urllib.error
    import urllib.request
    from http.server import ThreadingHTTPServer

    from demo.app import make_handler

    calls = []

    class Stub:
        def segment(self, req):
            calls.append(("segment", req))
            if req.get("prompt_label") == 7:
                raise ValueError("Input coordinates must be normalized to [-1, 1].")
            return {"seg": [True, False, True]}

        def sampled_pointcloud(self, req):
            calls.append(("sampled", sorted(req)))
            return {"response": "success"}

        def pointcloud(self, path):
            calls.append(("pointcloud", os.path.basename(path)))
            return {"xyz": [0.0, 0.0, 0.0], "rgb": [1.0, 1.0, 1.0]}

        def clear(self):
            return {"status": "cleared"}

        def next(self):
            return {"status": "cleared"}

        def save(self):
            return {"status": "saved"}

    static = tmp_path / "static"
    static.mkdir()
    (static / "index.html").write_text("<html>ok</html>")
    srv = ThreadingHTTPServer(("127.0.0.1", 0), make_handler(Stub(), str(static), str(static / "models")))
    port = srv.server_address[1]
    t = threading.Thread(target=srv.serve_forever, daemon=True)
    t.start()
    try:
        def post(route, body):
            req = urllib.request.Request(f"http://127.0.0.1:{port}{route}", data=json.dumps(body).encode(),
                                         headers={"Content-Type": "application/json"})
            return json.loads(urllib.request.urlopen(req, timeout=10).read())

        assert post("/segment", {"prompt_point": [0.1, 0.2, 0.3], "prompt_label": 1}) == {"seg": [True, False, True]}
        assert calls[-1] == ("segment", {"prompt_point": [0.1, 0.2, 0.3], "prompt_label": 1})
        assert post("/sampled_pointcloud", {"points": {"0": 0.0}, "colors": {"0": 1.0}}) == {"response": "success"}
        assert post("/clear", {}) == {"status": "cleared"} and post("/next", {}) == {"status": "cleared"}
        assert post("/save", {}) == {"status": "saved"}
        got = json.loads(urllib.request.urlopen(f"http://127.0.0.1:{port}/pointcloud/scene.ply", timeout=10).read())
        assert got == {"xyz": [0.0, 0.0, 0.0], "rgb": [1.0, 1.0, 1.0]} and calls[-1] == ("pointcloud", "scene.ply")
        assert urllib.request.urlopen(f"http://127.0.0.1:{port}/", timeout=10).read() == b"<html>ok</html>"
        with pytest.raises(urllib.error.HTTPError) as e:
            post("/segment", {"prompt_point": [9, 9, 9], "prompt_label": 7})
        assert e.value.code == 400 and "normalized" in json.loads(e.value.read())["error"]
        with pytest.raises(urllib.error.HTTPError) as e:
            post("/nope", {})
        assert e.value.code == 404
        with pytest.raises(urllib.error.HTTPError) as e:
            urllib.request.urlopen(f"http://127.0.0.1:{port}/static/../../etc/passwd", timeout=10)
        assert e.value.code == 404
    finally:
        srv.shutdown()
        srv.server_close()


def test_eval_driver_rotation_matches_reference_scipy_rotation(tmp_path):
    """ADVICE r1: the reference driver rotates every crop by R.from_euler('xyz', [-90, 180, 0]) (eval_kitti.py:18,347);
    the default of this driver must be that rotation, bit-compatible with scipy's r.apply up to float32 rounding."""
    from scipy.spatial.transform import Rotation as R

    from evaluation import eval_kitti
    from pc_sam.utils import ply

    rng = np.random.default_rng(0)
    xyz = rng.normal(size=(257, 3)).astype(np.float32) * 11
    for deg in ((-90, 180, 0), (10, -20, 33.5)):
        want = R.from_euler("xyz", list(deg), degrees=True)
        np.testing.assert_allclose(eval_kitti.euler_xyz_matrix(deg), want.as_matrix(), atol=1e-12)
    assert eval_kitti.parse_rotation("none") is None
    np.testing.assert_allclose(eval_kitti.parse_rotation(None), eval_kitti.parse_rotation("reference"))
    np.testing.assert_allclose(eval_kitti.parse_rotation("-90,180,0"), eval_kitti.parse_rotation("reference"), atol=1e-15)
    f = str(tmp_path / "car_0000.ply")
    ply.write_ply(f, {"x": xyz[:, 0].copy(), "y": xyz[:, 1].copy(), "z": xyz[:, 2].copy(),
                      "R": np.zeros(257, np.uint8), "G": np.zeros(257, np.uint8), "B": np.zeros(257, np.uint8),
                      "label": np.ones(257, np.int32)})
    got = eval_kitti.load_crop(f, eval_kitti.parse_rotation("reference"))["xyz"]
    want = np.float32(R.from_euler("xyz", [-90, 180, 0], degrees=True).apply(xyz))
    np.testing.assert_allclose(got, want, atol=2e-6, rtol=0)
    assert np.array_equal(eval_kitti.load_crop(f, None)["xyz"], xyz)


def test_forward_in_training_mode_is_refused():
    """ADVICE r1: the inference-only path must not silently run the eval loop when the module is in train() mode."""
    import pytest
    import torch

    from pc_sam.model import build_point_sam

    m = build_point_sam("eva02_test_tiny", 8, 4).train()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 16, 3), torch.zeros(1, 16, 3), torch.zeros(1, 1, 16, dtype=torch.bool))


def test_compose_resolves_group_level_and_string_defaults(tmp_path):
    """configs/model/enc_with_radius.yaml style: a group file with its own `defaults: [default]` list (advisor finding)."""
    from pc_sam.utils.config import compose

    (tmp_path / "model").mkdir()
    (tmp_path / "model" / "default.yaml").write_text("_target_: a.B\npc_encoder:\n  patch_embed:\n    num_patches: 1024\n    radius: null\n")
    (tmp_path / "model" / "with_radius.yaml").write_text("defaults:\n  - default\n\npc_encoder:\n  patch_embed:\n    radius: 0.1\n")
    (tmp_path / "top.yaml").write_text("defaults:\n  - model: with_radius\n  - _self_\nlr: 3e-4\n")
    cfg = compose(str(tmp_path), "top")
    assert cfg["model"]["_target_"] == "a.B"
    assert cfg["model"]["pc_encoder"]["patch_embed"] == {"num_patches": 1024, "radius": 0.1}
    assert cfg["lr"] == 3e-4


def test_demo_static_guard_and_fixed_pointcloud(tmp_path):
    """A sibling directory sharing the static directory's prefix is not served; query strings are ignored; the configured
    point cloud is served whatever name the URL carries (demo/app.py:91-126 always loads args.pointcloud)."""
    import io

    from demo.app import make_handler

    static = tmp_path / "static"
    static.mkdir()
    (static / "index.html").write_text("ok")
    sib = tmp_path / "static_x"
    sib.mkdir()
    (sib / "secret.txt").write_text("no")

    class FakeSession:
        def pointcloud(self, path):
            return {"path": path}

    H = make_handler(FakeSession(), str(static), str(static / "models"), "scene.ply")

    def get(path):
        h = H.__new__(H)
        h.path, h.wfile, h.headers = path, io.BytesIO(), {}
        h.send_response = lambda code: setattr(h, "code", code)
        h.send_header = lambda *a: None
        h.end_headers = lambda: None
        h.do_GET()
        return h.code, h.wfile.getvalue()

    assert get("/?v=3") == (200, b"ok")
    assert get("/../static_x/secret.txt")[0] == 404
    code, body = get("/pointcloud/whatever.ply?x=1")
    assert code == 200 and body.decode().endswith('models/scene.ply"}')
