"""Argument checks of the geometry entry points (FPS, kNN, the Voronoi features, the border-prompt sampler, the group
gather and the 3-NN weights), called through the C ABI with fake, never dereferenced device pointers.  Every refusal the
header states must come back as PSAM_ERR_ARG or PSAM_ERR_UNSUPPORTED before any CUDA call.

This runs only where no CUDA device is visible: there, a refusal that regressed reaches at most the CUDA runtime's own
error for the missing device, never a kernel.  The accepted controls only assert that the argument checks let them
through (whatever the runtime then says about the missing device)."""
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers must never reach a GPU")

ERR_ARG, ERR_UNSUPPORTED = -1, -2
FAKE = 0x7F0000000000  # 16-byte aligned, never dereferenced


def _p(i):
    """The i-th fake buffer: distinct, 64 KB apart."""
    return FAKE + i * 0x10000


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build, native

    build.build()
    return native.lib()


def _fps(lib, B=1, N=1000, G=64, ws=_p(9)):
    return lib.psam_fps_f32(_p(0), B, N, G, _p(1), _p(2), ws, None)


def _fps_varlen(lib, B=1, N=1000, G=64, ws=_p(9)):
    return lib.psam_fps_varlen_f32(_p(0), _p(3), B, N, G, _p(1), _p(2), ws, None)


@pytest.mark.parametrize("entry", [_fps, _fps_varlen], ids=["psam_fps_f32", "psam_fps_varlen_f32"])
def test_fps_refuses(lib, entry):
    assert entry(lib, G=0) == ERR_ARG
    assert entry(lib, G=-3) == ERR_ARG
    assert entry(lib, N=0) == ERR_ARG
    assert entry(lib, B=0) == ERR_ARG
    # beyond the 8-CTA register capacity the streaming plan needs its workspace
    assert lib.psam_fps_workspace_bytes(1, 200000, 64) > 0
    assert entry(lib, N=200000, ws=None) == ERR_ARG


def test_fps_refuses_more_samples_than_points(lib):
    assert _fps(lib, N=63, G=64) == ERR_ARG
    assert _fps_varlen(lib, N=63, G=64) != ERR_ARG  # a padded batch repeats sample 0 past a cloud's length


def test_fps_accepts_null_workspace_when_none_is_needed(lib):
    assert lib.psam_fps_workspace_bytes(2, 65536, 64) == 0
    assert _fps(lib, B=2, N=65536, ws=None) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert _fps(lib, N=200000, ws=_p(9)) not in (ERR_ARG, ERR_UNSUPPORTED)


def _knn(lib, B=2, Q=100, N=2000, K=9, d2=_p(4)):
    return lib.psam_knn_f32(_p(0), _p(1), B, Q, N, K, _p(2), d2, None)


def _knn_varlen(lib, B=2, Q=100, N=2000, K=9, d2=_p(4)):
    return lib.psam_knn_varlen_f32(_p(0), _p(1), _p(3), B, Q, N, K, _p(2), d2, None)


@pytest.mark.parametrize("entry", [_knn, _knn_varlen], ids=["psam_knn_f32", "psam_knn_varlen_f32"])
def test_knn_refuses(lib, entry):
    assert entry(lib, K=2001) == ERR_ARG
    assert entry(lib, K=0) == ERR_ARG
    assert entry(lib, Q=0) == ERR_ARG
    assert entry(lib, K=1025) == ERR_UNSUPPORTED
    assert entry(lib, B=65536) == ERR_UNSUPPORTED  # the clouds are the grid's y extent
    assert entry(lib, K=1024) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert entry(lib, K=1000, N=1000) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert entry(lib, B=65535, d2=None) not in (ERR_ARG, ERR_UNSUPPORTED)


def test_knn3_interp_refuses_too_many_clouds(lib):
    assert lib.psam_knn3_interp_f32(_p(0), _p(1), 65536, 100, 64, _p(2), _p(3), None) == ERR_UNSUPPORTED
    assert lib.psam_knn3_interp_f32(_p(0), _p(1), 65535, 100, 64, _p(2), _p(3), None) not in (ERR_ARG, ERR_UNSUPPORTED)


def _voronoi(lib, C=3, out=_p(5), y_hi=_p(6), pitch=64):
    return lib.psam_voronoi_features_f32(_p(0), _p(1), _p(2), _p(3), 2, 1, 1000, 64, C, out, y_hi, 1000 * pitch, pitch, None)


def test_voronoi_refuses(lib):
    assert _voronoi(lib, C=3, pitch=6) == ERR_ARG
    assert _voronoi(lib, C=60, pitch=63) == ERR_ARG
    assert _voronoi(lib, out=None, y_hi=None) == ERR_ARG
    assert _voronoi(lib, C=-1) == ERR_ARG
    assert _voronoi(lib, C=60, pitch=64) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert _voronoi(lib, y_hi=None, pitch=0) not in (ERR_ARG, ERR_UNSUPPORTED)  # no split output: pitch is unused


def _border(lib, B=2, M=3, N=500, logits=None, masks=None, ws=_p(9)):
    return lib.psam_border_prompt_f32(_p(0), _p(1), logits, masks, B, M, N, 0, _p(4), _p(5), _p(6), ws, None)


def test_border_prompt_refuses(lib):
    assert _border(lib, logits=_p(2), masks=_p(3)) == ERR_ARG
    assert _border(lib, ws=_p(9) + 2) == ERR_ARG
    assert _border(lib, ws=None) == ERR_ARG
    assert _border(lib, B=1, M=21846) == ERR_UNSUPPORTED  # B * M * 3 = 65538
    assert _border(lib, B=2, M=10923) == ERR_UNSUPPORTED
    assert _border(lib, B=1, M=21845) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert _border(lib, logits=_p(2)) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert _border(lib, masks=_p(3)) not in (ERR_ARG, ERR_UNSUPPORTED)


def _gather(lib, ptrs=None, B=2, rep=1, N=500, G=32, K=8, C=3, center=_p(4)):
    p = ptrs or [_p(0), _p(1), _p(2), _p(3)]
    return lib.psam_group_gather_f32(p[0], p[1], p[2], p[3], center, B, rep, N, G, K, C, 0.1, _p(5), None)


@pytest.mark.parametrize("missing", range(4), ids=["xyz", "feats", "centers", "knn_idx"])
def test_group_gather_refuses_null(lib, missing):
    p = [_p(0), _p(1), _p(2), _p(3)]
    p[missing] = None
    assert _gather(lib, ptrs=p) == ERR_ARG


@pytest.mark.parametrize("field", ["rep", "C", "N", "G", "K", "B"])
def test_group_gather_refuses_sizes(lib, field):
    assert _gather(lib, **{field: -1}) == ERR_ARG
    if field != "C":
        assert _gather(lib, **{field: 0}) == ERR_ARG


def test_group_gather_accepts(lib):
    assert _gather(lib, C=0) not in (ERR_ARG, ERR_UNSUPPORTED)
    assert _gather(lib, center=None, rep=4, K=1) not in (ERR_ARG, ERR_UNSUPPORTED)
