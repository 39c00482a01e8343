"""CPU tests of clouds of different sizes in one batch: the padded-batch C-ABI entry points refuse bad host arguments
before any CUDA call, the padding helper and the decode plan give the right shapes for a ragged list, and the Python layer
refuses mismatched clouds, clouds smaller than the tokenizer's first level and the Voronoi tokenizer before it touches the
device."""
import ctypes

import pytest
import torch

from pc_sam.automatic_mask_generator import PointCloudMaskGenerator, plan_decode


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    for name in ("psam_fps_varlen_f32", "psam_knn_varlen_f32", "psam_mask_candidates_varlen_f32", "psam_mask_regions_varlen"):
        getattr(L, name).restype = ctypes.c_int
    return L


i, ll, f, p = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p
FAKE = p(0x1000)  # never dereferenced: validation fails before any CUDA call


def test_fps_varlen_argument_validation(lib):
    def call(xyz=FAKE, lengths=FAKE, B=3, N=100, G=16, idx=FAKE, centers=FAKE, ws=FAKE):
        return lib.psam_fps_varlen_f32(xyz, lengths, i(B), i(N), i(G), idx, centers, ws, None)

    for kw in (dict(xyz=None), dict(lengths=None), dict(idx=None), dict(centers=None), dict(B=0), dict(B=-1), dict(N=0),
               dict(N=-5), dict(G=0), dict(G=-1)):
        assert call(**kw) == -1, kw


def test_knn_varlen_argument_validation(lib):
    def call(q=FAKE, key=FAKE, lengths=FAKE, B=3, Q=16, N=100, K=9, idx=FAKE, d2=FAKE):
        return lib.psam_knn_varlen_f32(q, key, lengths, i(B), i(Q), i(N), i(K), idx, d2, None)

    for kw in (dict(q=None), dict(key=None), dict(lengths=None), dict(idx=None), dict(B=0), dict(Q=0), dict(N=0), dict(N=-1),
               dict(K=0), dict(K=101), dict(K=10, N=9)):
        assert call(**kw) == -1, kw


def test_candidates_varlen_argument_validation(lib):
    def call(lg=FAKE, io=FAKE, lengths=FAKE, B=3, Zc=8, C=3, N=100, P=8, base=0, stride=24, W=4, bits=FAKE, area=FAKE,
             stab=FAKE, score=FAKE):
        return lib.psam_mask_candidates_varlen_f32(lg, io, lengths, i(B), i(Zc), i(C), i(N), i(P), f(0.0), f(1.0), f(0.0), f(0.0),
                                                   i(0), ll(base), ll(stride), i(W), bits, area, stab, score, None)

    for kw in (dict(lg=None), dict(io=None), dict(lengths=None), dict(bits=None), dict(area=None), dict(stab=None),
               dict(score=None), dict(B=0), dict(B=-1), dict(Zc=0), dict(C=0), dict(N=0), dict(P=-1), dict(base=-1), dict(W=3),
               dict(stride=23), dict(base=1, stride=24), dict(B=1 << 16, Zc=1 << 15, C=3, stride=3 << 15)):
        assert call(**kw) == -1, kw


def test_regions_varlen_argument_validation(lib):
    def call(bits=FAKE, slots=64, lengths=FAKE, B=3, K=64, W=4, N=100, keep=FAKE, cnt=FAKE, nbr=FAKE, k1=9, A=10, bo=FAKE,
             ao=FAKE, so=FAKE, ws=FAKE):
        return lib.psam_mask_regions_varlen(bits, ll(slots), lengths, i(B), i(K), i(W), i(N), keep, cnt, nbr, i(k1), i(A), bo, ao,
                                            so, ws, None)

    for kw in (dict(bits=None), dict(lengths=None), dict(keep=None), dict(cnt=None), dict(nbr=None), dict(bo=None),
               dict(ao=None), dict(so=None), dict(ws=None), dict(B=0), dict(B=-1), dict(slots=0), dict(K=-1), dict(K=16385),
               dict(N=0), dict(N=(1 << 20) + 1, W=1 << 15), dict(W=3), dict(k1=0), dict(k1=101), dict(A=0), dict(ws=p(0x1008))):
        assert call(**kw) == -1, kw
    assert call(K=0, bits=None, keep=None, bo=None, ao=None, so=None) == 0  # nothing to do, nothing launched


# ------------------------------------------------------------------------------------------------
# padding helper and decode plan
# ------------------------------------------------------------------------------------------------
def test_pad_clouds_shapes_and_lengths():
    from psam_b200 import ops

    sizes = [5, 1, 9, 3]
    xyz = [torch.rand(n, 3) * 2 - 1 for n in sizes]
    rgb = [torch.rand(n, 3, dtype=torch.float64) for n in sizes]
    px, pr, lengths = ops.pad_clouds(xyz, rgb)
    assert px.shape == (4, 9, 3) and pr.shape == (4, 9, 3) and px.dtype == pr.dtype == torch.float32
    assert px.is_contiguous() and pr.is_contiguous()
    assert lengths.dtype == torch.int32 and lengths.tolist() == sizes
    for b, n in enumerate(sizes):
        assert torch.equal(px[b, :n], xyz[b]) and torch.equal(pr[b, :n], rgb[b].float())
        assert torch.count_nonzero(px[b, n:]) == 0 and torch.count_nonzero(pr[b, n:]) == 0
    (one, l1) = ops.pad_clouds([xyz[2]])
    assert one.shape == (1, 9, 3) and l1.tolist() == [9]
    with pytest.raises(ValueError):
        ops.pad_clouds([])
    with pytest.raises(ValueError):
        ops.pad_clouds(xyz, rgb[:3])
    with pytest.raises(ValueError):
        ops.pad_clouds(xyz, [torch.rand(n + 1, 3) for n in sizes])


def test_plan_decode_uses_the_largest_cloud():
    sizes = [6000, 14000, 9000]
    plan = plan_decode(len(sizes), 256, max(sizes), 64)
    assert plan.rows == 21 and plan.batches[0] == (0, 21) and plan.batches[-1] == (252, 256)
    assert sum(e - s for s, e in plan.batches) == 256


# ------------------------------------------------------------------------------------------------
# the Python layer refuses bad batches before touching the device
# ------------------------------------------------------------------------------------------------
def _model(kind):
    from pc_sam.model import build_point_sam, build_point_sam_hier

    if kind == "base":
        return build_point_sam("eva02_test_tiny", 64, 32).eval()
    return build_point_sam_hier("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3).eval()


def _ragged(sizes):
    return [torch.rand(n, 3) * 2 - 1 for n in sizes], [torch.rand(n, 3) for n in sizes]


@pytest.mark.parametrize("kind,G", [("base", 64), ("hier", 128)])
def test_varlen_checks_before_the_device(kind, G):
    model = _model(kind)
    xyz, rgb = _ragged([G + 10, G, 3 * G])
    assert model.varlen_clouds(xyz, rgb) == [G + 10, G, 3 * G]
    with pytest.raises(ValueError):
        model.varlen_clouds(xyz, rgb[:2])
    with pytest.raises(ValueError):
        model.varlen_clouds(xyz, [rgb[0], rgb[1][:-1], rgb[2]])
    with pytest.raises(ValueError):
        model.varlen_clouds([xyz[0], xyz[1][:, :2], xyz[2]], rgb)
    with pytest.raises(ValueError):
        model.varlen_clouds([], [])
    with pytest.raises(TypeError):
        model.varlen_clouds(torch.rand(2, G, 3), torch.rand(2, G, 3))
    small_x, small_r = _ragged([G + 10, G - 1])
    with pytest.raises(RuntimeError, match="num_samples"):
        model.varlen_clouds(small_x, small_r)
    # predict_masks_varlen and the generator run the same checks first (CPU tensors: any device work would fail differently)
    pc, pl = torch.zeros(2, 1, 1, 3), torch.ones(2, 1, 1, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="num_samples"):
        model.predict_masks_varlen(small_x, small_r, pc, pl)
    gen = PointCloudMaskGenerator(model, points_per_cloud=16, points_per_batch=8)
    for call in (gen.generate_packed_batch, gen.generate_batch):
        with pytest.raises(RuntimeError, match="num_samples"):
            call(small_x, small_r)
        with pytest.raises(ValueError):
            call(xyz, rgb[:2])
        with pytest.raises(ValueError):
            call(xyz, torch.rand(3, G, 3))


def test_varlen_refuses_the_voronoi_tokenizer():
    from pc_sam.model.pc_encoder import PatchEmbedNN

    model = _model("base")
    model.pc_encoder.patch_embed = PatchEmbedNN(6, 64, 512, 64)
    xyz, rgb = _ragged([100, 80])
    with pytest.raises(NotImplementedError):
        model.varlen_clouds(xyz, rgb)
    with pytest.raises(NotImplementedError):
        model.predict_masks_varlen(xyz, rgb, torch.zeros(2, 1, 1, 3), torch.ones(2, 1, 1, dtype=torch.int64))
    with pytest.raises(NotImplementedError):
        PointCloudMaskGenerator(model, points_per_cloud=16).generate_packed_batch(xyz, rgb)
