"""CPU tests of automatic mask generation on a batch of clouds: the decode plan (prompts per cloud and batch, the short
last batch, the decoder's row-tile limit), argument validation of the batched C-ABI entry points before any CUDA call with
their workspace formulas, and the generator's batch interface."""
import ctypes
import inspect
import types

import pytest
import torch

from pc_sam.automatic_mask_generator import DECODE_MAX_ROW_TILES, PointCloudMaskGenerator, plan_decode


# ------------------------------------------------------------------------------------------------
# decode plan
# ------------------------------------------------------------------------------------------------
def test_plan_one_cloud_is_the_single_cloud_batching():
    plan = plan_decode(1, 1024, 32768, 64)
    assert plan.rows == 64 and plan.batches == [(s, s + 64) for s in range(0, 1024, 64)]
    plan = plan_decode(1, 64, 2048, 24)  # short last batch
    assert plan.rows == 24 and plan.batches == [(0, 24), (24, 48), (48, 64)]


def test_plan_keeps_points_per_batch_rows():
    plan = plan_decode(3, 64, 2048, 64)  # B below points_per_batch: 21 prompts of each cloud = 63 rows
    assert plan.rows == 21 and plan.batches == [(0, 21), (21, 42), (42, 63), (63, 64)]
    plan = plan_decode(8, 256, 10000, 64)
    assert plan.rows == 8 and len(plan.batches) == 32 and plan.batches[-1] == (248, 256)
    plan = plan_decode(64, 10, 100, 64)  # B equal to points_per_batch: one prompt of each cloud
    assert plan.rows == 1 and plan.batches == [(s, s + 1) for s in range(10)]
    plan = plan_decode(100, 3, 100, 64)  # B above points_per_batch: still one prompt of each cloud
    assert plan.rows == 1 and plan.batches == [(0, 1), (1, 2), (2, 3)]
    plan = plan_decode(5, 3, 100, 64)  # fewer prompts than one batch holds
    assert plan.rows == 12 and plan.batches == [(0, 3)]


def test_plan_row_tile_limit():
    n = DECODE_MAX_ROW_TILES * 128 // 2  # two clouds with one prompt each fill the grid exactly
    assert plan_decode(2, 4, n, 64).rows == 32  # the limit is checked for one prompt per cloud
    with pytest.raises(ValueError, match="row tiles"):
        plan_decode(2, 4, n + 1, 64)
    with pytest.raises(ValueError, match="row tiles"):
        plan_decode(3, 1, n, 1)
    for bad in ((0, 4, 100, 64), (2, 0, 100, 64), (2, 4, 0, 64), (2, 4, 100, 0)):
        with pytest.raises(ValueError):
            plan_decode(*bad)


# ------------------------------------------------------------------------------------------------
# C ABI: argument validation before any CUDA call, workspace formulas
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    for name in ("psam_mask_candidates_batched_f32", "psam_mask_nms_batched", "psam_mask_regions_batched"):
        getattr(L, name).restype = ctypes.c_int
    for name in ("psam_mask_nms_workspace_bytes", "psam_mask_nms_batched_workspace_bytes", "psam_mask_regions_workspace_bytes",
                 "psam_mask_regions_batched_workspace_bytes"):
        getattr(L, name).restype = ctypes.c_size_t
    return L


i, ll, f, p = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p
FAKE = p(0x1000)  # never dereferenced: validation fails before any CUDA call


def test_candidates_batched_argument_validation(lib):
    def call(lg=FAKE, io=FAKE, B=3, Zc=8, C=3, N=100, base=0, stride=24, W=4, bits=FAKE, area=FAKE, stab=FAKE, score=FAKE):
        return lib.psam_mask_candidates_batched_f32(lg, io, i(B), i(Zc), i(C), i(N), f(0.0), f(1.0), f(0.0), f(0.0), i(0), ll(base),
                                                    ll(stride), i(W), bits, area, stab, score, None)

    for kw in (dict(lg=None), dict(io=None), dict(bits=None), dict(area=None), dict(stab=None), dict(score=None), dict(B=0),
               dict(B=-1), dict(Zc=0), dict(C=0), dict(N=0), dict(base=-1), dict(W=3), dict(stride=23), dict(base=1, stride=24),
               dict(B=1 << 16, Zc=1 << 15, C=3)):
        assert call(**kw) == -1, kw


def test_nms_batched_argument_validation(lib):
    def call(bits=FAKE, area=FAKE, score=FAKE, B=3, K=64, W=4, keep=FAKE, cnt=FAKE, ws=FAKE):
        return lib.psam_mask_nms_batched(bits, area, score, i(B), i(K), i(W), f(0.7), keep, cnt, ws, None)

    for kw in (dict(bits=None), dict(area=None), dict(score=None), dict(keep=None), dict(cnt=None), dict(ws=None), dict(B=0),
               dict(B=-2), dict(B=65536), dict(K=-1), dict(K=16385), dict(W=0), dict(ws=p(0x1008)), dict(K=0, keep=None)):
        assert call(**kw) == -1, kw


def test_regions_batched_argument_validation(lib):
    def call(bits=FAKE, slots=64, B=3, K=64, W=4, N=100, keep=FAKE, cnt=FAKE, nbr=FAKE, k1=9, A=10, bo=FAKE, ao=FAKE, so=FAKE,
             ws=FAKE):
        return lib.psam_mask_regions_batched(bits, ll(slots), i(B), i(K), i(W), i(N), keep, cnt, nbr, i(k1), i(A), bo, ao, so, ws,
                                             None)

    for kw in (dict(bits=None), dict(keep=None), dict(cnt=None), dict(nbr=None), dict(bo=None), dict(ao=None), dict(so=None),
               dict(ws=None), dict(B=0), dict(B=-1), dict(slots=0), dict(slots=-1), dict(K=-1), dict(K=16385), dict(N=0),
               dict(W=3), dict(k1=0), dict(k1=101), dict(A=0), dict(ws=p(0x1008)), dict(K=0, cnt=None)):
        assert call(**kw) == -1, kw
    assert call(K=0, bits=None, keep=None, bo=None, ao=None, so=None) == 0  # nothing to do, nothing launched


def test_nms_batched_workspace_is_b_times_one_cloud(lib):
    for K, W in ((0, 1), (1, 1), (63, 2), (3072, 1024), (16383, 64), (16384, 1)):
        one = lib.psam_mask_nms_workspace_bytes(i(K), i(W))
        assert lib.psam_mask_nms_batched_workspace_bytes(i(1), i(K), i(W)) == one
        for B in (2, 3, 8):
            assert lib.psam_mask_nms_batched_workspace_bytes(i(B), i(K), i(W)) == B * one, (B, K)
    # the suppression matrix dominates: K * ceil(K / 64) * 8 bytes per cloud
    assert lib.psam_mask_nms_batched_workspace_bytes(i(4), i(3072), i(1)) == 4 * (16 + 3072 * 4 + 3072 * 48 * 8)
    assert lib.psam_mask_nms_batched_workspace_bytes(i(0), i(64), i(1)) == 0
    assert lib.psam_mask_nms_batched_workspace_bytes(i(2), i(16385), i(1)) == 0


def test_regions_batched_workspace_does_not_grow_with_b(lib):
    def ws(B, K, N):
        return lib.psam_mask_regions_batched_workspace_bytes(i(B), i(K), i(N))

    for K, N in ((3072, 2047), (3072, 49152), (3072, 131072), (5, 131072), (1, 49153), (16384, 1 << 20)):
        assert ws(1, K, N) == lib.psam_mask_regions_workspace_bytes(i(K), i(N))
    assert ws(8, 3072, 32768) == 16  # shared-memory labels
    for B, K, N in ((3, 3072, 131072), (3, 5, 131072), (4, 1, 49153), (8, 16384, 1 << 20)):
        slices = min(B * K, 132, max(1, (24 << 20) // (4 * N)))  # one label slice pool for the whole launch
        assert ws(B, K, N) == (slices * N * 4 + 15) // 16 * 16, (B, K, N)
    assert ws(0, 8, 100) == ws(2, -1, 100) == ws(2, 16385, 100) == ws(2, 8, 0) == 0


# ------------------------------------------------------------------------------------------------
# generator interface
# ------------------------------------------------------------------------------------------------
def test_batch_interface_signature():
    for fn in (PointCloudMaskGenerator.generate_packed_batch, PointCloudMaskGenerator.generate_batch):
        prm = inspect.signature(fn).parameters
        assert list(prm) == ["self", "xyz", "rgb", "min_mask_region_area"]  # no crop keywords
        assert prm["min_mask_region_area"].kind is inspect.Parameter.KEYWORD_ONLY and prm["min_mask_region_area"].default == 0


def test_batch_arguments_checked_before_the_model_runs():
    g = PointCloudMaskGenerator(object())  # the area check comes before the model is touched
    for fn in (g.generate_packed_batch, g.generate_batch):
        with pytest.raises(ValueError):
            fn(torch.zeros(2, 16, 3), torch.zeros(2, 16, 3), min_mask_region_area=-1)
    g = PointCloudMaskGenerator(types.SimpleNamespace(training=False))  # a model that must never be called
    for xyz, rgb in ((torch.zeros(16, 3), torch.zeros(16, 3)), (torch.zeros(2, 16, 4), torch.zeros(2, 16, 3)),
                     (torch.zeros(2, 16, 3), torch.zeros(2, 15, 3)), (torch.zeros(2, 16, 3), torch.zeros(3, 16, 3)),
                     (torch.zeros(0, 16, 3), torch.zeros(0, 16, 3))):
        with pytest.raises(ValueError):
            g.generate_packed_batch(xyz, rgb)
    g.model.training = True
    with pytest.raises(NotImplementedError):
        g.generate_packed_batch(torch.zeros(2, 16, 3), torch.zeros(2, 16, 3))
