"""Argument checks of the tensor-core entry points (psam_gemm_bf16x3, psam_attention_bf16x3 and its two-pass form), called
through the C ABI with fake, never dereferenced device pointers.  Every combination here that the kernels would
mis-compute must come back as PSAM_ERR_ARG before any CUDA call.

This runs only where no CUDA device is visible: there, a refusal that regressed reaches at most the CUDA runtime's own
error for the missing device, never a kernel.  The accepted controls only assert that the argument checks let them
through (whatever the runtime then says about the missing device)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers must never reach a GPU")

ERR_ARG = -1
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
FAKE = 0x7F0000000000  # 16-byte aligned, never dereferenced


def _p(i):
    """The i-th fake buffer: distinct, 64 KB apart, so aliasing is explicit."""
    return FAKE + i * 0x10000


@pytest.fixture(scope="module")
def nv():
    from psam_b200 import build, native

    build.build()
    return native


def _operand(nv, i, rows, k, pitch=None, nb1=0, nb2=0, b1=0, b2=0):
    pitch = pitch or (k + 63) // 64 * 64
    return nv.Operand(_p(i), rows * pitch * max(nb1, 1) * max(nb2, 1), rows, k, pitch, nb1, nb2, b1, b2)


def _gemm(nv, M=256, N=128, K=64, split_k=1, passes=3, **fields):
    a, w = _operand(nv, 0, M, K), _operand(nv, 1, N, K)
    o = nv.GemmOut()
    o.alpha = 1.0
    for name, v in fields.items():
        setattr(o, name, v)
    return nv.lib().psam_gemm_bf16x3(ctypes.byref(a), ctypes.byref(w), ctypes.byref(o), passes, split_k, None)


_F32 = dict(out_f32=_p(2), ldo=128)
_SPLIT = dict(out_hi=_p(3), out_plane=256 * 128, ldo_s=128)

_GEMM_REFUSED = {
    "accumulate_without_out_f32": dict(accumulate=1),
    "accumulate_split_k_without_out_f32": dict(accumulate=1, _split_k=2),
    "accumulate_with_split_output": dict(accumulate=1, **_F32, **_SPLIT),
    "accumulate_split_output_only": dict(accumulate=1, **_SPLIT),
    "accumulate_with_gelu": dict(accumulate=1, act=ACT_GELU, **_F32),
    "accumulate_with_relu": dict(accumulate=1, act=ACT_RELU, **_F32),
    "accumulate_with_other_resid": dict(accumulate=1, resid=_p(4), **_F32),
    "accumulate_split_k_with_gelu": dict(accumulate=1, act=ACT_GELU, _split_k=3, **_F32),
    "accumulate_split_k_with_other_resid": dict(accumulate=1, resid=_p(4), _split_k=3, **_F32),
    "split_k_without_accumulate": dict(_split_k=2, **_F32),
    "rowdot_rows_not_multiple_of_32": dict(rd_w=_p(5), rd_out=_p(6), rd_rows=100, rd_c=2),
    "rowdot_nine_vectors": dict(rd_w=_p(5), rd_out=_p(6), rd_rows=128, rd_c=9),
    "gmax_with_resid": dict(gmax=_p(7), ld_gmax=128, group_rows=32, resid=_p(4), **_F32),
    "gmax_with_act": dict(gmax=_p(7), ld_gmax=128, group_rows=32, act=ACT_RELU),
    "swiglu_odd_n": dict(swiglu=1, ldo=64, out_f32=_p(2), _N=127),
    "stats_out_with_split_k": dict(stats_out=_p(8), accumulate=1, _split_k=2, **_F32),
    "no_output": dict(),
}


@pytest.mark.parametrize("case", list(_GEMM_REFUSED))
def test_gemm_refuses(nv, case):
    f = dict(_GEMM_REFUSED[case])
    split_k, N = f.pop("_split_k", 1), f.pop("_N", 128)
    assert _gemm(nv, N=N, split_k=split_k, **f) == ERR_ARG, case


_GEMM_ACCEPTED = {
    "accumulate": dict(accumulate=1, **_F32),
    "accumulate_resid_is_out_f32": dict(accumulate=1, resid=_p(2), **_F32),
    "accumulate_split_k": dict(accumulate=1, _split_k=7, bias=_p(9), **_F32),
    "accumulate_split_k_ln_fold": dict(accumulate=1, _split_k=3, ln_stats=_p(10), ln_c=_p(11), ln_h=64, ln_eps=1e-6, **_F32),
    "ln_fold_without_bias_alpha_half": dict(ln_stats=_p(10), ln_c=_p(11), ln_h=64, ln_eps=1e-6, alpha=0.5, **_SPLIT),
    "split_output_odd_column": dict(out_hi=_p(3) + 2, out_plane=256 * 130, ldo_s=130),
}


@pytest.mark.parametrize("case", list(_GEMM_ACCEPTED))
def test_gemm_accepts(nv, case):
    """Controls: the engine's accumulate forms, and the ones the header allows, pass the argument checks."""
    f = dict(_GEMM_ACCEPTED[case])
    split_k = f.pop("_split_k", 1)
    assert _gemm(nv, split_k=split_k, **f) != ERR_ARG, case


def _attention(nv, entry, scale=0.125, dh=64, L=200, q_nb=(3, 2), k_nb=(3, 2), v_nb=(3, 2)):
    pitch = 3 * 3 * dh
    mk = lambda i, nb: nv.Operand(_p(i), 2 * L * pitch, L, dh, pitch, nb[0], nb[1], dh, L * pitch)
    q, k, v = mk(0, q_nb), mk(1, k_nb), mk(2, v_nb)
    ldo = 3 * 64 * 2
    return getattr(nv.lib(), entry)(ctypes.byref(q), ctypes.byref(k), ctypes.byref(v), _p(3), 2 * L * ldo, ldo, 64,
                                    L * ldo, scale, None)


_ATT_REFUSED = {
    "k_fewer_heads": dict(k_nb=(2, 2)),
    "v_fewer_heads": dict(v_nb=(1, 2)),
    "k_fewer_clouds": dict(k_nb=(3, 1)),
    "v_more_clouds": dict(v_nb=(3, 3)),
    "v_unbatched": dict(v_nb=(0, 0)),
    "scale_zero": dict(scale=0.0),
    "scale_negative_zero": dict(scale=-0.0),
    "scale_negative": dict(scale=-0.125),
    "scale_nan": dict(scale=float("nan")),
    "scale_inf": dict(scale=float("inf")),
    "scale_negative_inf": dict(scale=float("-inf")),
}


@pytest.mark.parametrize("entry", ["psam_attention_bf16x3", "psam_attention_bf16x3_twopass"])
@pytest.mark.parametrize("case", list(_ATT_REFUSED))
def test_attention_refuses(nv, entry, case):
    assert _attention(nv, entry, **_ATT_REFUSED[case]) == ERR_ARG


@pytest.mark.parametrize("entry", ["psam_attention_bf16x3", "psam_attention_bf16x3_twopass"])
def test_attention_accepts(nv, entry):
    """Controls: equal batch extents (0 and 1 both mean none) and a small positive scale pass the argument checks."""
    assert _attention(nv, entry) != ERR_ARG
    assert _attention(nv, entry, scale=1e-30) != ERR_ARG
    assert _attention(nv, entry, q_nb=(1, 0), k_nb=(0, 1), v_nb=(0, 0)) != ERR_ARG
