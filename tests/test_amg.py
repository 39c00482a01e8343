"""CPU tests of automatic mask generation: the numpy oracle's NMS against a brute-force pairwise loop, the generator's
constructor, argument validation of the new C-ABI entries (before any CUDA call) and the build of the new source."""
import ctypes
import inspect
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import amg_ref

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _brute_nms(masks: np.ndarray, score: np.ndarray, thr: float) -> list:
    """Independent restatement: masks as Python sets, candidates picked one by one by (score desc, index asc)."""
    sets = [set(np.nonzero(m)[0].tolist()) for m in masks]
    alive = [i for i in range(len(score)) if score[i] > -np.inf]
    kept = []
    while alive:
        best = min(alive, key=lambda i: (-float(score[i]), i))
        kept.append(best)
        alive.remove(best)
        nxt = []
        for j in alive:
            inter = len(sets[best] & sets[j])
            union = len(sets[best]) + len(sets[j]) - inter
            if not np.float32(inter) / np.float32(union) > np.float32(thr):
                nxt.append(j)
        alive = nxt
    return kept


def _random_case(seed, K=48, N=70):
    rng = np.random.default_rng(seed)
    masks = rng.random((K, N)) < rng.uniform(0.05, 0.6, size=(K, 1))
    masks[3] = masks[7]                      # duplicate masks (IoU = 1)
    masks[10] = masks[11] | masks[12]
    masks[5] = False                         # an empty mask
    score = rng.choice(np.float32([0.5, 0.7, 0.9, 0.95]), size=K).astype(np.float32)  # many ties
    score[[2, 9]] = -np.inf                  # filtered out
    score[5] = -np.inf                       # empty masks never survive candidate extraction
    return masks, score


@pytest.mark.parametrize("thr", [0.0, 0.3, 0.5, 0.7, 1.0])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_nms_matches_brute_force(seed, thr):
    masks, score = _random_case(seed)
    bits = amg_ref.pack_bits(masks)
    area = masks.sum(1).astype(np.int32)
    got = amg_ref.nms(bits, area, score, thr).tolist()
    assert got == _brute_nms(masks, score, thr)
    if thr == 1.0:  # nothing is suppressed: every valid candidate, in (score desc, index asc) order
        assert got == amg_ref.sort_order(score).tolist()
    assert 7 not in got or 3 not in got or thr >= 1.0  # the duplicate pair never survives together below 1.0


def test_oracle_nms_all_filtered_and_packing():
    masks, score = _random_case(3)
    bits = amg_ref.pack_bits(masks)
    assert amg_ref.nms(bits, masks.sum(1), np.full_like(score, -np.inf), 0.5).tolist() == []
    assert np.array_equal(amg_ref.unpack_bits(bits, masks.shape[1]), masks)
    assert bits.shape == (masks.shape[0], 3) and bits.dtype == np.uint32
    assert np.all(bits[:, 2] >> (70 - 64) == 0)  # tail bits zero


def test_oracle_candidate_rules():
    lg = np.float32([[[2.0, 0.5, -0.5, -2.0], [-2.0, -2.0, -2.0, -2.0], [1.5, 1.5, 0.9, -1.0]]])
    iou = np.float32([[0.9, 0.95, 0.88]])
    c = amg_ref.candidates(lg, iou, 0.0, 1.0, pred_iou_thresh=0.88, stability_thresh=0.5)
    assert c["area"].tolist() == [2, 0, 3]
    # hi = count(> 1), lo = count(> -1): 1/3, 0/0, 2/3
    assert c["stability"][0] == np.float32(1) / np.float32(3) and np.isnan(c["stability"][1])
    # row 0 fails stability (0.33 < 0.5), row 1 is empty, row 2 fails iou > 0.88 (equal is not greater)
    assert np.all(c["score"] == -np.inf)
    c = amg_ref.candidates(lg, iou, 0.0, 1.0, pred_iou_thresh=0.0, stability_thresh=np.float32(2) / np.float32(3))
    assert c["score"].tolist() == [-np.inf, -np.inf, np.float32(0.88)]  # stability == thresh survives (>=)


def test_generator_constructor_and_defaults():
    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator

    sig = inspect.signature(PointCloudMaskGenerator.__init__)
    want = dict(points_per_cloud=1024, points_per_batch=64, pred_iou_thresh=0.88, stability_score_thresh=0.95,
                stability_score_offset=1.0, mask_nms_thresh=0.7, min_mask_area=0)
    assert list(sig.parameters)[1:] == ["model"] + list(want)
    assert {k: sig.parameters[k].default for k in want} == want
    g = PointCloudMaskGenerator(object())
    assert (g.points_per_cloud, g.points_per_batch, g.mask_nms_thresh, g.min_mask_area) == (1024, 64, 0.7, 0)
    with pytest.raises(ValueError):
        PointCloudMaskGenerator(object(), points_per_cloud=6000)  # 18000 candidates > 16384
    with pytest.raises(ValueError):
        PointCloudMaskGenerator(object(), points_per_batch=0)


def test_generator_refuses_training_mode():
    import torch

    from pc_sam.automatic_mask_generator import PointCloudMaskGenerator
    from pc_sam.model import build_point_sam

    m = build_point_sam("eva02_test_tiny", 8, 4).train()
    with pytest.raises(NotImplementedError):
        PointCloudMaskGenerator(m).generate_packed(torch.zeros(16, 3), torch.zeros(16, 3))


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    L = ctypes.CDLL(build.build())
    L.psam_mask_candidates_f32.restype = ctypes.c_int
    L.psam_mask_nms.restype = ctypes.c_int
    L.psam_mask_nms_workspace_bytes.restype = ctypes.c_size_t
    return L


def test_mask_gen_source_is_built(lib):
    from psam_b200 import build

    assert "mask_gen.cu" in build.SOURCES
    assert os.path.exists(os.path.join(build.LIBDIR, "mask_gen.o"))
    if shutil.which("cuobjdump"):
        elf = subprocess.run(["cuobjdump", "-lelf", os.path.join(build.LIBDIR, "mask_gen.o")], capture_output=True, text=True).stdout
        assert "sm_90a" in elf


def test_mask_gen_argument_validation_without_gpu(lib):
    f, i, ll, p = ctypes.c_float, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p
    fake = p(0x1000)  # never dereferenced: validation fails before any CUDA call

    def cand(logits=fake, iou=fake, Z=2, C=3, N=100, base=0, W=4, bits=fake, area=fake, stab=fake, score=fake):
        return lib.psam_mask_candidates_f32(logits, iou, i(Z), i(C), i(N), f(0.0), f(1.0), f(0.88), f(0.95), i(0), ll(base),
                                            i(W), bits, area, stab, score, None)

    for kw in (dict(logits=None), dict(iou=None), dict(bits=None), dict(area=None), dict(stab=None), dict(score=None),
               dict(Z=0), dict(C=0), dict(N=0), dict(base=-1), dict(W=3), dict(N=33, W=1)):
        assert cand(**kw) == -1, kw

    def nms(bits=fake, area=fake, score=fake, K=64, W=4, keep=fake, cnt=fake, ws=fake):
        return lib.psam_mask_nms(bits, area, score, i(K), i(W), f(0.7), keep, cnt, ws, None)

    for kw in (dict(bits=None), dict(area=None), dict(score=None), dict(keep=None), dict(cnt=None), dict(ws=None),
               dict(K=16385), dict(K=-1), dict(W=0), dict(ws=p(0x1004))):
        assert nms(**kw) == -1, kw
    assert lib.psam_mask_nms_workspace_bytes(i(3072), i(1024)) == 16 + 3072 * 4 + 3072 * 48 * 8
    assert lib.psam_mask_nms_workspace_bytes(i(0), i(1)) == 16


def test_generator_does_not_import_oracle():
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import pc_sam.automatic_mask_generator; "
            "assert not any(k.startswith('oracle') for k in sys.modules)") % (os.path.join(REPO, "point-sam_b200"), REPO)
    subprocess.check_call([sys.executable, "-c", code])
