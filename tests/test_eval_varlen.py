"""CPU tests of the padded evaluation loop: the batch plan of the evaluation driver, the group-shape rule, the PLY header
count, forward_varlen's and the varlen graph predictor's refusals before any device work, the new group-size refusal of
the varlen path, the border sampler's C-ABI refusals, and the driver's file order under any batching (a stub model
stands in for the CUDA path)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "point-sam_b200"))

from evaluation import eval_kitti  # noqa: E402
from pc_sam.utils import ply  # noqa: E402


# ------------------------------------------------------------------------------------------------
# batch plan and group shape
# ------------------------------------------------------------------------------------------------
def _check_plan(plan, sizes, keys, bs, cap):
    flat = [i for b in plan for i in b]
    assert sorted(flat) == list(range(len(sizes)))  # every crop exactly once
    for b in plan:
        assert 1 <= len(b) <= bs
        assert len({keys[i] for i in b}) == 1
        assert [sizes[i] for i in b] == sorted(sizes[i] for i in b)
        assert len(b) == 1 or len(b) * max(sizes[i] for i in b) <= cap


def test_plan_eval_batches_coverage_order_and_cap():
    rng = np.random.default_rng(0)
    sizes = [int(v) for v in np.exp(rng.uniform(np.log(100), np.log(40000), 57))]
    keys = [eval_kitti.group_shape_for(n) for n in sizes]
    for bs in (1, 2, 4, 8, 64):
        for cap in (1, 30000, 100000, 1 << 20):
            plan = eval_kitti.plan_eval_batches(sizes, keys, bs, cap)
            _check_plan(plan, sizes, keys, bs, cap)
    # one key: a group sorted by size, cut greedily
    sizes = [500, 100, 300, 200, 400, 100]
    assert eval_kitti.plan_eval_batches(sizes, [0] * 6, 4, 1 << 20) == [[1, 5, 3, 2], [4, 0]]
    assert eval_kitti.plan_eval_batches(sizes, [0] * 6, 4, 900) == [[1, 5, 3], [2, 4], [0]]
    assert eval_kitti.plan_eval_batches(sizes, [0] * 6, 8, 100) == [[1], [5], [3], [2], [4], [0]]
    # groups in order of first appearance
    assert eval_kitti.plan_eval_batches([5, 3, 4, 1], ["b", "a", "b", "a"], 8, 100) == [[2, 0], [3, 1]]
    # batch size 1: one crop per batch, still every crop once
    plan = eval_kitti.plan_eval_batches(sizes, [0] * 6, 1, 1 << 20)
    assert sorted(i for b in plan for i in b) == list(range(6)) and all(len(b) == 1 for b in plan)
    assert eval_kitti.plan_eval_batches([], [], 4, 100) == []
    for bad in (dict(batch_size=0, max_batch_points=10), dict(batch_size=2, max_batch_points=0)):
        with pytest.raises(ValueError):
            eval_kitti.plan_eval_batches([1], [0], **bad)
    with pytest.raises(ValueError):
        eval_kitti.plan_eval_batches([1, 2], [0], 2, 10)


def test_group_shape_for_branches():
    assert eval_kitti.group_shape_for(255) == (255, 2)
    assert eval_kitti.group_shape_for(256) == (256, 256)
    assert eval_kitti.group_shape_for(2047) == (2047, 256)
    assert eval_kitti.group_shape_for(2048) == (2048, 256)
    assert eval_kitti.group_shape_for(30000) == (2048, 256)
    assert eval_kitti.group_shape_for(30001) == (2048, 256)

    class G:
        num_groups = group_size = 0

    m = type("M", (), {"pc_encoder": type("E", (), {"patch_embed": type("P", (), {"grouper": G()})()})()})()
    for n in (100, 255, 256, 2047, 2048, 30000, 30001):
        eval_kitti.set_group_shape(m, n)
        assert (m.pc_encoder.patch_embed.grouper.num_groups, m.pc_encoder.patch_embed.grouper.group_size) == \
            eval_kitti.group_shape_for(n)


def test_ply_vertex_count_reads_the_header_only(tmp_path):
    f = str(tmp_path / "a.ply")
    ply.write_ply(f, {"x": np.zeros(37, np.float32), "label": np.ones(37, np.int32)})
    assert ply.vertex_count(f) == 37
    with open(f, "r+b") as fh:  # a truncated payload does not matter to the header count
        fh.truncate(os.path.getsize(f) - 40)
    assert ply.vertex_count(f) == 37
    g = str(tmp_path / "b.ply")
    ply.write_ply(g, {"x": np.zeros(5, np.float32)}, fmt="ascii")
    assert ply.vertex_count(g) == 5
    bad = tmp_path / "c.ply"
    bad.write_bytes(b"not a ply\n")
    with pytest.raises(ValueError):
        ply.vertex_count(str(bad))


# ------------------------------------------------------------------------------------------------
# forward_varlen and the graph predictor refuse before the device
# ------------------------------------------------------------------------------------------------
def _model(kind):
    from pc_sam.model import build_point_sam, build_point_sam_hier

    if kind == "base":
        return build_point_sam("eva02_test_tiny", 64, 32).eval()
    return build_point_sam_hier("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3).eval()


def _ragged(sizes, M=2):
    return ([torch.rand(n, 3) * 2 - 1 for n in sizes], [torch.rand(n, 3) for n in sizes],
            [torch.rand(M, n) > 0.5 for n in sizes])


@pytest.mark.parametrize("kind,G", [("base", 64), ("hier", 128)])
def test_forward_varlen_refusals(kind, G):
    """CPU tensors: any device work would fail with a different error than the one expected."""
    model = _model(kind)
    xyz, rgb, gt = _ragged([G + 10, G, 2 * G])
    with pytest.raises(NotImplementedError):
        model.forward_varlen(xyz, rgb, gt, is_eval=False)
    model.train()
    with pytest.raises(NotImplementedError):
        model.forward_varlen(xyz, rgb, gt)
    model.eval()
    for bad in ([gt[0], gt[1]], [gt[0], gt[1][:, :-1], gt[2]], [gt[0], gt[1][:1], gt[2]], [gt[0], gt[1], gt[2][None]],
                [gt[0], gt[1], torch.zeros(0, 2 * G, dtype=torch.bool)]):
        with pytest.raises(ValueError):
            model.forward_varlen(xyz, rgb, bad)
    with pytest.raises(TypeError):
        model.forward_varlen(xyz, rgb, torch.zeros(3, 2, G, dtype=torch.bool))
    with pytest.raises(ValueError):
        model.forward_varlen(xyz, rgb[:2], gt)
    small = _ragged([G + 10, G - 1])
    with pytest.raises(RuntimeError, match="num_samples"):
        model.forward_varlen(*small)


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_varlen_refuses_clouds_below_the_group_size(kind):
    """num_groups <= N_b < group_size: the kNN of that cloud would take padded rows as neighbours."""
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    model = _model(kind)
    pe = model.pc_encoder.patch_embed
    g = pe.grouper if kind == "base" else pe.grouper1
    g.num_groups, g.group_size = 16, 32
    xyz, rgb, gt = _ragged([40, 20, 32])
    with pytest.raises(RuntimeError, match="group size 32"):
        model.varlen_clouds(xyz, rgb)
    with pytest.raises(RuntimeError, match="group size"):
        model.forward_varlen(xyz, rgb, gt)
    with pytest.raises(RuntimeError, match="group size"):
        model.predict_masks_varlen(xyz, rgb, torch.zeros(3, 1, 1, 3), torch.ones(3, 1, 1, dtype=torch.int64))
    gen = PointCloudMaskGenerator(model, points_per_cloud=8, points_per_batch=8)
    for call in (gen.generate_packed_batch, gen.generate_batch):
        with pytest.raises(RuntimeError, match="group size"):
            call(xyz, rgb)
    assert model.varlen_clouds(xyz[::2], rgb[::2]) == [40, 32]  # N_b == group_size is fine


def test_forward_varlen_refuses_the_voronoi_tokenizer():
    from pc_sam.model.pc_encoder import PatchEmbedNN

    model = _model("base")
    model.pc_encoder.patch_embed = PatchEmbedNN(6, 64, 512, 64)
    with pytest.raises(NotImplementedError):
        model.forward_varlen(*_ragged([100, 80]))


def test_sampler_refuses_lengths_outside_evaluation():
    from pc_sam.model import prompt_sampling

    with pytest.raises(NotImplementedError):
        prompt_sampling.sample_prompts_adapter(torch.zeros(1, 4, 3), torch.zeros(1, 1, 4, dtype=torch.bool),
                                               torch.zeros(1, 4), is_eval=False, lengths=torch.ones(1, dtype=torch.int32))


def test_border_prompt_lengths_are_validated():
    from psam_b200 import ops

    for lengths in (torch.ones(2, dtype=torch.int64), torch.ones(3, dtype=torch.int32)):
        with pytest.raises(ValueError, match="lengths"):
            ops.border_prompt(torch.zeros(2, 4, 3), torch.zeros(2, 1, 4, dtype=torch.bool), lengths=lengths)


def test_varlen_graph_predictor_refusals():
    """The host checks of IterativeGraphPredictorVarlen on an instance holding CPU buffers (its constructor needs a GPU
    stream): they run before anything is copied or enqueued."""
    from psam_b200.predictor import IterativeGraphPredictorVarlen

    model = _model("base")
    pred = IterativeGraphPredictorVarlen.__new__(IterativeGraphPredictorVarlen)
    pred.model = model
    B, M, N_max = 3, 2, 300
    pred.xyz, pred.feats = torch.zeros(B, N_max, 3), torch.zeros(B, N_max, 3)
    pred.gt = torch.zeros(B, M, N_max, dtype=torch.bool)
    xyz, rgb, gt = _ragged([100, 300, 64])
    coords, feats, gts, sizes = pred._check(xyz, rgb, gt)
    assert sizes == [100, 300, 64] and [g.shape for g in gts] == [(2, 100), (2, 300), (2, 64)]
    assert pred._check(xyz[:1], rgb[:1], gt[:1])[3] == [100]
    x4, r4, g4 = _ragged([100, 100, 100, 100])
    with pytest.raises(ValueError, match="at most 3"):
        pred._check(x4, r4, g4)
    xb, rb, gb = _ragged([100, 301])
    with pytest.raises(ValueError, match="301"):
        pred._check(xb, rb, gb)
    with pytest.raises(ValueError):
        pred._check(xyz, rgb, [g[:1] for g in gt])  # M = 1 for a predictor of M = 2
    with pytest.raises(ValueError):
        pred._check(xyz, [torch.rand(n, 4) for n in (100, 300, 64)], gt)
    with pytest.raises(RuntimeError, match="num_samples"):
        pred._check(*_ragged([100, 63]))
    with pytest.raises(TypeError):
        pred._check(torch.zeros(3, 100, 3), torch.zeros(3, 100, 3), gt)


# ------------------------------------------------------------------------------------------------
# C ABI refusals
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers must never reach a GPU")
def test_border_prompt_varlen_argument_validation():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    fn = L.psam_border_prompt_varlen_f32
    fn.restype = ctypes.c_int
    i, p = ctypes.c_int, ctypes.c_void_p
    FAKE = p(0x7F0000000000)

    def call(coords=FAKE, lengths=FAKE, gt=FAKE, lg=None, pm=None, B=3, M=2, N=100, mode=0, xyz=FAKE, lab=FAKE, st=FAKE,
             ws=FAKE):
        return fn(coords, lengths, gt, lg, pm, i(B), i(M), i(N), i(mode), xyz, lab, st, ws, None)

    for kw in (dict(coords=None), dict(lengths=None), dict(gt=None), dict(xyz=None), dict(lab=None), dict(st=None),
               dict(ws=None), dict(lg=FAKE, pm=FAKE), dict(B=0), dict(B=-1), dict(M=0), dict(N=0), dict(N=-3),
               dict(ws=p(0x7F0000000002))):
        assert call(**kw) == -1, kw
    assert call(B=20000, M=2) == -2  # B * M * 3 regions past the grid's z extent


# ------------------------------------------------------------------------------------------------
# the driver with a stub model: rows in file order under any batching
# ------------------------------------------------------------------------------------------------
class _Stub(torch.nn.Module):
    """Deterministic per-crop outputs on CPU that depend on the crop's own points only: iteration t predicts the ground
    truth rolled by t + (number of points) % 5.  Records the batches it is given."""

    def __init__(self, varlen=True):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.prompt_iters = 3
        self.pc_encoder = type("E", (), {"patch_embed": type("P", (), {"grouper": type("G", (), {})()})()})()
        self.batches = []
        if varlen:
            self.forward_varlen = self._forward_varlen

    def _one(self, gt):
        gt = gt.float()
        return [{"prompt_masks": torch.roll(gt, t + gt.shape[-1] % 5, dims=-1) * 2 - 1} for t in range(self.prompt_iters)]

    def forward(self, coords, features, gt_masks, is_eval=False):
        return self._one(gt_masks.flatten(0, 1))

    def _forward_varlen(self, coords, features, gt_masks, is_eval=True):
        g = self.pc_encoder.patch_embed.grouper
        self.batches.append(([c.shape[0] for c in coords], (g.num_groups, g.group_size)))
        return [self._one(gt) for gt in gt_masks]


def _crops(tmpdir, sizes):
    files = []
    for i, n in enumerate(sizes):
        r = np.random.default_rng(i)
        files.append(os.path.join(tmpdir, f"c{i:02d}_{i:03d}.ply"))  # one object name per crop: per_object holds its row
        lab = (r.random(n) < 0.4).astype(np.int32)
        lab[:2] = (0, 1)
        ply.write_ply(files[-1], {"x": r.normal(size=n).astype(np.float32), "y": r.normal(size=n).astype(np.float32),
                                  "z": r.normal(size=n).astype(np.float32), "R": r.integers(0, 256, n).astype(np.uint8),
                                  "G": r.integers(0, 256, n).astype(np.uint8), "B": r.integers(0, 256, n).astype(np.uint8),
                                  "label": lab})
    return files


def test_evaluate_keeps_file_order_under_any_batching(tmp_path):
    sizes = [3000, 200, 2500, 40000, 2048, 700, 5000, 2200, 31000]
    files = _crops(str(tmp_path), sizes)
    want = eval_kitti.evaluate(_Stub(varlen=False), files, log=None)  # the reference's forward, one crop at a time
    assert list(want["per_object"]) == [f"c{i:02d}" for i in range(len(files))]
    for bs, cap in ((1, 1 << 20), (2, 1 << 20), (4, 1 << 20), (16, 1 << 20), (16, 10000), (3, 70000)):
        stub = _Stub()
        got = eval_kitti.evaluate(stub, files, log=None, batch_size=bs, max_batch_points=cap)
        assert list(got["per_object"]) == list(want["per_object"])
        for k in want["per_object"]:
            assert np.array_equal(got["per_object"][k], want["per_object"][k]), (bs, cap, k)
        assert np.array_equal(got["total"], want["total"]) and np.array_equal(got["object_mean"], want["object_mean"])
        seen = sorted(n for b, _ in stub.batches for n in b)
        assert seen == sorted(sizes) and all(len(b) <= bs for b, _ in stub.batches)
        for b, shape in stub.batches:  # the group shape set for a batch is every crop's own
            assert all(eval_kitti.group_shape_for(n) == shape for n in b)
            assert len(b) == 1 or len(b) * max(b) <= cap
    assert max(len(b) for b, _ in stub.batches) > 1
    with pytest.raises(TypeError):
        eval_kitti.evaluate(_Stub(varlen=False), files, log=None, batch_size=4)


@pytest.mark.parametrize("value", [0, 1])
def test_evaluate_names_a_crop_without_border(tmp_path, value):
    files = _crops(str(tmp_path), [300, 400])
    r = np.random.default_rng(9)
    bad = str(tmp_path / "flat_000.ply")
    ply.write_ply(bad, {"x": r.normal(size=50).astype(np.float32), "y": r.normal(size=50).astype(np.float32),
                        "z": r.normal(size=50).astype(np.float32), "R": np.zeros(50, np.uint8), "G": np.zeros(50, np.uint8),
                        "B": np.zeros(50, np.uint8), "label": np.full(50, value, np.int32)})
    for bs in (1, 4):
        with pytest.raises(RuntimeError, match="flat_000.ply"):
            eval_kitti.evaluate(_Stub(), files + [bad], log=None, batch_size=bs)
