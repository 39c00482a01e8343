"""CPU tests of encoder fine-tuning: which parameters training mode accepts and refuses (before any device work), and the
C-ABI argument validation of the encoder backward entry points."""
import ctypes

import pytest
import torch


def _tiny(enc="eva02_test_tiny"):
    from pc_sam.model import build_point_sam

    m = build_point_sam(enc, 8, 4).train()
    m.requires_grad_(False)
    return m


def _inputs():
    return torch.zeros(1, 16, 3), torch.zeros(1, 16, 3), torch.zeros(1, 1, 16, dtype=torch.bool)


def _reaches_the_device(m):
    m._check_trainable()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(*_inputs())


def test_legal_encoder_sets_pass_the_refusals():
    m = _tiny()
    m.mask_decoder.requires_grad_(True)
    m.pc_encoder.transformer.blocks[-1].requires_grad_(True)
    _reaches_the_device(m)
    m.pc_encoder.transformer.fc_norm.requires_grad_(True)
    m.pc_encoder.out_proj.requires_grad_(True)
    _reaches_the_device(m)
    m = _tiny("eva_test_tiny_fused")  # the encoder alone, decoder frozen, with patch_proj and pos_embed
    m.pc_encoder.transformer.blocks.requires_grad_(True)
    m.pc_encoder.patch_proj.requires_grad_(True)
    m.pc_encoder.pos_embed.requires_grad_(True)
    _reaches_the_device(m)


@pytest.mark.parametrize("part", ["pc_encoder.patch_embed.patch_encoder", "point_encoder", "mask_encoder",
                                  "pc_encoder.transformer.head", "pc_encoder.transformer.cls_token"])
def test_tokenizer_prompt_encoders_and_unused_parameters_are_refused_by_name(part):
    m = _tiny()
    m.mask_decoder.requires_grad_(True)
    m.pc_encoder.transformer.blocks.requires_grad_(True)
    target = m.get_submodule(part) if not part.endswith("cls_token") else None
    if target is None:
        m.pc_encoder.transformer.cls_token.requires_grad_(True)
    else:
        target.requires_grad_(True)
    first = next(n for n, p in m.named_parameters() if p.requires_grad and n.startswith(part))
    with pytest.raises(NotImplementedError, match=rf"'{first}' has requires_grad=True.*model.requires_grad_\(False\).*"
                                                  r"model.mask_decoder.requires_grad_\(True\)"):
        m(*_inputs())


def test_hier_keeps_refusing_an_encoder_block():
    from pc_sam.model import build_point_sam_hier

    h = build_point_sam_hier("eva02_test_tiny").train()
    h.requires_grad_(False)
    h.pc_encoder.transformer.blocks[-1].requires_grad_(True)
    with pytest.raises(NotImplementedError, match="PointCloudSAMHier"):
        h(*_inputs())


def test_trainable_block_without_a_backward_is_refused_before_device_work():
    from pc_sam.model.eva import EvaBlock

    m = _tiny()
    # a width of 128 with 16 heads (dh = 8) is supported; 20 heads do not divide it and dh = 4 has no aligned operand
    for heads, ok in ((16, True), (32, False)):
        m.pc_encoder.transformer.blocks[-1] = EvaBlock(128, heads, 344, False, True)
        m.requires_grad_(False)
        m.pc_encoder.transformer.blocks[-1].requires_grad_(True)
        if ok:
            _reaches_the_device(m)
        else:
            with pytest.raises(NotImplementedError, match=r"width and head dim are multiples of 8, got width 128 with 32 heads"):
                m(*_inputs())
    # the same block frozen is not refused (inference needs no backward)
    m.requires_grad_(False)
    m.mask_decoder.requires_grad_(True)
    m._check_trainable()


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    return ctypes.CDLL(build.build())


def test_encoder_backward_entry_points_validate_arguments_without_gpu(lib):
    """Bad arguments are rejected before any CUDA call (PSAM_ERR_ARG = -1)."""
    P = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    f = ctypes.c_float(1e-6)
    L = ctypes.c_longlong
    for fn in ("psam_layernorm_backward", "psam_swiglu_ln_backward", "psam_gelu_backward", "psam_softmax_backward"):
        getattr(lib, fn).restype = ctypes.c_int
    ln = lambda x=P, ldx=128, M=4, D=128, dy=P, g=P, eps=f, dres=None, dx=P, hi=None, part=P, rb=256: lib.psam_layernorm_backward(
        x, L(ldx), M, D, dy, L(D), g, eps, dres, L(D), dx, L(D), hi, L(0), L(D), part, rb, None)
    assert ln(x=None) == -1 and ln(dy=None) == -1 and ln(g=None) == -1 and ln(dx=None) == -1 and ln(part=None) == -1
    assert ln(M=0) == -1 and ln(D=0) == -1 and ln(ldx=100) == -1 and ln(rb=0) == -1 and ln(rb=1025) == -1
    assert ln(eps=ctypes.c_float(-1.0)) == -1 and ln(eps=ctypes.c_float(float("nan"))) == -1
    sw = lambda a=P, lda=768, M=4, Hd=344, Hp=384, dhn=P, beta=P, da=P, ldo=768, part=P, rb=256: lib.psam_swiglu_ln_backward(
        a, L(lda), M, Hd, Hp, dhn, L(Hp), P, beta, f, da, L(ldo), None, L(0), L(0), None, L(0), L(0), part, rb, None)
    assert sw(a=None) == -1 and sw(beta=None) == -1 and sw(da=None) == -1 and sw(part=None) == -1
    assert sw(Hp=300) == -1 and sw(lda=700) == -1 and sw(lda=769) == -1 and sw(ldo=767) == -1 and sw(M=-1) == -1 and sw(rb=2048) == -1
    ge = lambda a=P, M=4, n=64, dh=P, da=P: lib.psam_gelu_backward(a, L(n), M, n, dh, L(n), da, L(n), None, L(0), L(0), None, L(0), L(0), None)
    assert ge(a=None) == -1 and ge(dh=None) == -1 and ge(da=None) == -1 and ge(M=0) == -1 and ge(n=0) == -1
    sm = lambda s=P, dp=P, rows=8, Ls=64, ds=P, ld=64: lib.psam_softmax_backward(s, L(Ls), dp, L(Ls), L(rows), Ls, f, ds, L(0), L(ld), None)
    assert sm(s=None) == -1 and sm(dp=None) == -1 and sm(ds=None) == -1 and sm(rows=0) == -1 and sm(Ls=0) == -1 and sm(ld=32) == -1
