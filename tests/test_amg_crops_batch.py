"""CPU tests of crop layers on a batch of clouds (generate_packed_batch_crops / generate_batch_crops): argument validation of
the batched crop C ABI before any CUDA call, the binding's layout of psam_crop_run, the signatures and the keyword checks
of the new methods (made before the model or the device is touched), the crop-batch plan, and the Voronoi refusal."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from pc_sam.automatic_mask_generator import DECODE_MAX_ROW_TILES, DECODE_ROW_TILE, PointCloudMaskGenerator


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    for name in ("psam_crop_layout_batched_f32", "psam_crop_gather_batched_f32", "psam_crop_edge_filter_batched",
                 "psam_crop_uncrop_batched"):
        getattr(L, name).restype = ctypes.c_int
    L.psam_crop_gather_batched_workspace_bytes.restype = ctypes.c_size_t
    L.psam_crop_run_bytes.restype = ctypes.c_size_t
    return L


i, f, p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p
FAKE = p(0x1000)  # never dereferenced: validation fails before any CUDA call


def test_layout_batched_argument_validation(lib):
    def call(xyz=FAKE, lengths=FAKE, B=3, N=100, layers=1, r=0.3, boxes=FAKE, counts=FAKE):
        return lib.psam_crop_layout_batched_f32(xyz, lengths, i(B), i(N), i(layers), f(r), boxes, counts, None)

    for kw in (dict(xyz=None), dict(boxes=None), dict(counts=None), dict(B=0), dict(B=65536), dict(N=0), dict(layers=-1),
               dict(layers=4), dict(r=-0.1), dict(r=1.0), dict(r=float("nan"))):
        assert call(**kw) == -1, kw


def test_gather_batched_argument_validation(lib):
    def call(xyz=FAKE, rgb=FAKE, lengths=FAKE, B=3, N=100, boxes=FAKE, n_crops=9, pairs=FAKE, P=4, n_max=50, m=0.02, idx=FAKE,
             xo=FAKE, ro=FAKE, edge=FAKE, ws=FAKE):
        return lib.psam_crop_gather_batched_f32(xyz, rgb, lengths, i(B), i(N), boxes, i(n_crops), pairs, i(P), i(n_max), f(m), idx,
                                                xo, ro, edge, ws, None)

    for kw in (dict(xyz=None), dict(rgb=None), dict(boxes=None), dict(pairs=None), dict(idx=None), dict(xo=None), dict(ro=None),
               dict(edge=None), dict(ws=None), dict(B=0), dict(N=0), dict(n_crops=0), dict(P=0), dict(P=65536), dict(n_max=0),
               dict(n_max=101), dict(m=-0.1), dict(m=float("nan")), dict(ws=p(0x1008))):
        assert call(**kw) == -1, kw
    assert lib.psam_crop_gather_batched_workspace_bytes(0, 100) == 0
    assert lib.psam_crop_gather_batched_workspace_bytes(3, 0) == 0
    # per pair: a count and a maximum per 1024-point chunk, each block rounded up to 16 bytes
    assert lib.psam_crop_gather_batched_workspace_bytes(3, 5000) == 3 * 2 * 32
    assert lib.psam_crop_gather_batched_workspace_bytes(1, 1024) >= lib.psam_crop_gather_workspace_bytes(1024) - 16


def test_edge_filter_batched_argument_validation(lib):
    def call(bits=FAKE, T=2, K=8, W=4, edge=FAKE, score=FAKE):
        return lib.psam_crop_edge_filter_batched(bits, i(T), i(K), i(W), edge, score, None)

    for kw in (dict(bits=None), dict(edge=None), dict(score=None), dict(T=0), dict(T=65536), dict(K=-1), dict(W=0)):
        assert call(**kw) == -1, kw
    assert call(K=0, bits=None, edge=None, score=None) == 0  # nothing to do, nothing launched


def test_uncrop_batched_argument_validation(lib):
    def call(runs=FAKE, R=3, K=96, B=2, N=100, Wg=4, rows=96, **out):
        o = [out.get(k, FAKE) for k in ("gbits", "garea", "giou", "gstab", "gprompt", "gslot", "gcrop", "gscore", "lifted", "over")]
        return lib.psam_crop_uncrop_batched(runs, i(R), i(K), i(B), i(N), i(Wg), i(rows), *o, None)

    for kw in (dict(runs=None), dict(gbits=None), dict(garea=None), dict(giou=None), dict(gstab=None), dict(gprompt=None),
               dict(gslot=None), dict(gcrop=None), dict(gscore=None), dict(lifted=None), dict(over=None), dict(R=0), dict(R=65536),
               dict(K=0), dict(B=0), dict(N=0), dict(Wg=3), dict(rows=0), dict(rows=16385)):
        assert call(**kw) == -1, kw


def test_crop_run_layout_matches_the_header(lib):
    from psam_b200 import ops

    assert lib.psam_crop_run_bytes() == ops.CROP_RUN.itemsize == 8 * 8 + 10 * 4
    assert [ops.CROP_RUN.fields[k][1] for k in ("bits", "prompt_index", "K", "last", "layer_score", "capacity")] == [0, 56, 64, 92,
                                                                                                                   96, 100]


# ------------------------------------------------------------------------------------------------
# the Python layer
# ------------------------------------------------------------------------------------------------
def _model(kind="base"):
    from pc_sam.model import build_point_sam, build_point_sam_hier

    if kind == "base":
        return build_point_sam("eva02_test_tiny", 64, 32).eval()
    return build_point_sam_hier("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3).eval()


def _ragged(sizes):
    return [torch.rand(n, 3) * 2 - 1 for n in sizes], [torch.rand(n, 3) for n in sizes]


def test_batch_crops_interface_signature():
    want = ["self", "xyz", "rgb", "crop_n_layers", "crop_nms_thresh", "crop_overlap_ratio", "crop_n_points_downscale_factor",
            "min_mask_region_area"]
    for name in ("generate_packed_batch_crops", "generate_batch_crops"):
        sig = inspect.signature(getattr(PointCloudMaskGenerator, name))
        assert list(sig.parameters) == want, name
        kw = {k: v.default for k, v in sig.parameters.items() if v.kind is inspect.Parameter.KEYWORD_ONLY}
        assert kw == dict(crop_n_layers=1, crop_nms_thresh=0.7, crop_overlap_ratio=512 / 1500, crop_n_points_downscale_factor=1,
                          min_mask_region_area=0), name


class _Untouchable(torch.nn.Module):
    """A model whose every use fails the test: the keyword checks must come first."""

    def __getattr__(self, name):
        raise AssertionError(f"the model was touched ({name}) before the keywords were checked")


@pytest.mark.parametrize("kw", [dict(crop_n_layers=-1), dict(crop_n_layers=4), dict(crop_overlap_ratio=1.0),
                                dict(crop_overlap_ratio=-0.5), dict(crop_n_points_downscale_factor=0), dict(crop_nms_thresh=1.5),
                                dict(crop_nms_thresh=-0.1), dict(min_mask_region_area=-1)])
def test_batch_crops_keywords_checked_before_the_model(kw):
    gen = PointCloudMaskGenerator(_Untouchable(), points_per_cloud=16)
    xyz, rgb = _ragged([100, 80])
    for fn in (gen.generate_packed_batch_crops, gen.generate_batch_crops):
        with pytest.raises(ValueError):
            fn(xyz, rgb, **kw)
    with pytest.raises(TypeError):  # no positional keywords, and nothing else
        gen.generate_packed_batch_crops(xyz, rgb, 1)
    with pytest.raises(TypeError):
        gen.generate_packed_batch_crops(xyz, rgb, crop_layers=1)


def test_batch_crops_refuse_training_mode_and_bad_clouds_before_the_device():
    model = _model()
    gen = PointCloudMaskGenerator(model, points_per_cloud=16)
    xyz, rgb = _ragged([100, 80])
    model.train()
    with pytest.raises(NotImplementedError):
        gen.generate_packed_batch_crops(xyz, rgb)
    model.eval()
    with pytest.raises(ValueError):
        gen.generate_packed_batch_crops(xyz, rgb[:1])
    with pytest.raises(ValueError):
        gen.generate_packed_batch_crops(xyz, torch.rand(2, 100, 3))
    with pytest.raises(ValueError):
        gen.generate_packed_batch_crops(torch.rand(2, 100, 3), torch.rand(2, 90, 3))
    with pytest.raises(RuntimeError):  # smaller than the first-level num_groups (64)
        gen.generate_packed_batch_crops(*_ragged([100, 40]))
    with pytest.raises(RuntimeError):  # [B, N, 3] tensors take the same padded-batch checks
        gen.generate_packed_batch_crops(torch.rand(2, 40, 3), torch.rand(2, 40, 3))


def test_batch_crops_refuse_the_voronoi_tokenizer():
    from pc_sam.model.pc_encoder import PatchEmbedNN

    model = _model()
    model.pc_encoder.patch_embed = PatchEmbedNN(6, 64, 512, 64)
    gen = PointCloudMaskGenerator(model, points_per_cloud=16)
    xyz, rgb = _ragged([100, 80])
    for a, b in ((xyz, rgb), (torch.rand(2, 100, 3), torch.rand(2, 100, 3))):
        with pytest.raises(NotImplementedError):
            gen.generate_packed_batch_crops(a, b)
        with pytest.raises(NotImplementedError):
            gen.generate_batch_crops(a, b, crop_n_layers=2)


# ------------------------------------------------------------------------------------------------
# the crop-batch plan
# ------------------------------------------------------------------------------------------------
def test_plan_is_shared_with_the_evaluation_driver():
    from evaluation import eval_kitti
    from psam_b200 import parallel

    assert eval_kitti.plan_eval_batches is parallel.plan_eval_batches


@pytest.mark.parametrize("seed", range(6))
def test_crop_batch_plan_covers_each_crop_once_one_layer_per_batch(seed):
    """The generator's use of the plan: crops of every layer >= 1 of several clouds, keyed by layer, batch_size =
    points_per_batch, cap = the decoder's row-tile limit."""
    from psam_b200.parallel import plan_eval_batches

    rng = np.random.default_rng(seed)
    cap = DECODE_MAX_ROW_TILES * DECODE_ROW_TILE
    ppb = int(rng.choice([1, 3, 8, 32, 64]))
    pool = []  # (cloud, layer, points)
    for b in range(int(rng.integers(1, 6))):
        for layer in (1, 2):
            for _ in range(int(rng.integers(0, 8 ** layer))):
                pool.append((b, layer, int(rng.choice([rng.integers(64, 3000), rng.integers(1 << 20, 1 << 22)]))))
    rng.shuffle(pool)
    sizes, keys = [c for _, _, c in pool], [lay for _, lay, _ in pool]
    batches = plan_eval_batches(sizes, keys, ppb, cap)
    flat = [k for bt in batches for k in bt]
    assert sorted(flat) == list(range(len(pool)))  # every crop exactly once
    for bt in batches:
        assert bt and len({keys[k] for k in bt}) == 1  # one layer, so one prompt count per batch
        assert len(bt) <= ppb
        n_max = max(sizes[k] for k in bt)
        assert len(bt) * n_max <= cap or len(bt) == 1  # a crop above the cap runs alone
        assert [sizes[k] for k in bt] == sorted(sizes[k] for k in bt)


def test_crop_batch_plan_keeps_decoder_tiles_in_range():
    from pc_sam.automatic_mask_generator import plan_decode
    from psam_b200.parallel import plan_eval_batches

    sizes = [60000] * 200 + [131072] * 3
    cap = DECODE_MAX_ROW_TILES * DECODE_ROW_TILE
    for bt in plan_eval_batches(sizes, [1] * len(sizes), 64, cap):
        n_max = max(sizes[k] for k in bt)
        plan_decode(len(bt), 1024, n_max, 64)  # raises if one prompt per crop needs too many row tiles
