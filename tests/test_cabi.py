"""CPU tests of the drop-in boundary: the C-ABI library builds, loads, and exports every symbol that
include/psam_b200.h declares; the host-side API mirrors the reference's module tree (no compute calls)."""
import ctypes
import os
import re

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    from psam_b200 import build

    return build.build()


def test_header_symbols_exported(lib_path):
    hdr = open(os.path.join(REPO, "include", "psam_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(psam_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 20
    lib = ctypes.CDLL(lib_path)
    missing = [n for n in declared if not hasattr(lib, n)]
    assert not missing, missing
    from psam_b200 import native

    assert sorted(native.EXPORTS) == declared
    lib.psam_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.psam_version()


def test_argument_validation_without_gpu(lib_path):
    """Bad arguments are rejected before any CUDA call (PSAM_ERR_ARG = -1)."""
    lib = ctypes.CDLL(lib_path)
    lib.psam_fps_f32.restype = ctypes.c_int
    assert lib.psam_fps_f32(None, 1, 10, 4, None, None, None, None) == -1
    lib.psam_fps_workspace_bytes.restype = ctypes.c_size_t
    assert lib.psam_fps_workspace_bytes(1, 32768, 512) == 0            # register-resident plan
    assert lib.psam_fps_workspace_bytes(2, 200000, 512) == 2 * 200000 * 4  # streaming plan
    # round-2 entry points: rejected before any CUDA call as well
    lib.psam_voronoi_features_f32.restype = ctypes.c_int
    assert lib.psam_voronoi_features_f32(None, None, None, None, 1, 1, 8, 4, 3, None, None, 0, 0, None) == -1
    lib.psam_scatter_amax_f32.restype = ctypes.c_int
    assert lib.psam_scatter_amax_f32(None, None, 1, 8, 4, 6, None, None) == -1
    lib.psam_gemm_rowln_bf16x3.restype = ctypes.c_int
    assert lib.psam_gemm_rowln_bf16x3(None, None, None, 0, 0, None, None, ctypes.c_float(1e-5), 1, None, 0, 0, 3, None) == -1
    lib.psam_group_gather_f32.restype = ctypes.c_int
    assert lib.psam_group_gather_f32(None, None, None, None, None, 1, 1, 8, 4, 2, 3, ctypes.c_float(0.0), None, None) == -1


def test_state_dict_contract_and_api_surface():
    from oracle import torch_ref
    from pc_sam.model import PointCloudSAM, PointSAM, build_point_sam
    from pc_sam.model.loss import compute_iou
    from pc_sam.utils.torch_utils import replace_with_fused_layernorm

    assert PointSAM is PointCloudSAM
    for enc in ("eva02_test_tiny", "eva_test_tiny_fused", "eva02_base_patch14_448"):
        m = build_point_sam(enc, 32, 16)
        o = torch_ref.build_model(enc, 32, 16)
        assert list(m.state_dict().keys()) == list(o.state_dict().keys())
        m.load_state_dict(o.state_dict(), strict=True)
        m.apply(replace_with_fused_layernorm)
    keys = set(m.state_dict().keys())
    for k in ["pc_encoder.patch_embed.patch_encoder.conv1.0.weight", "pc_encoder.patch_proj.weight", "pc_encoder.pos_embed.2.bias",
              "pc_encoder.transformer.blocks.0.attn.q_proj.bias", "pc_encoder.transformer.blocks.0.mlp.fc1_g.weight",
              "pc_encoder.transformer.fc_norm.weight", "pc_encoder.transformer.cls_token", "pc_encoder.out_proj.weight",
              "point_encoder.pe_layer.positional_encoding_gaussian_matrix", "point_encoder.point_embeddings.1.weight",
              "mask_encoder.no_mask_embed.weight", "mask_decoder.iou_token.weight",
              "mask_decoder.transformer.layers.1.cross_attn_image_to_token.out_proj.weight",
              "mask_decoder.transformer.final_attn_token_to_image.q_proj.weight", "mask_decoder.transformer.norm_final_attn.bias",
              "mask_decoder.output_hypernetworks_mlps.3.layers.2.weight", "mask_decoder.output_upscaling.3.bias",
              "mask_decoder.iou_prediction_head.layers.0.weight"]:
        assert k in keys, k
    assert "pc_encoder.transformer.blocks.0.attn.k_proj.bias" not in keys
    g = m.pc_encoder.patch_embed.grouper
    g.num_groups, g.group_size = 2048, 256  # runtime-mutable like eval_kitti.py:352-362
    assert m.prompt_iters == 5
    iou = compute_iou(torch.tensor([[1.0, -1.0, 2.0]]), torch.tensor([[True, True, False]]))
    assert abs(float(iou) - 1 / 3) < 1e-6


def test_product_path_has_no_cpu_fallback():
    from oracle import synth
    from pc_sam.model import build_point_sam

    m = build_point_sam("eva02_test_tiny", 8, 4)
    xyz, feats = synth.make_batch(1, 64, 0)
    pc, pl = synth.make_prompts(xyz, 1, 0)
    with pytest.raises(RuntimeError):
        m.predict_masks(xyz, feats, pc, pl)
    # the product package never imports the oracle
    import subprocess
    import sys

    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import pc_sam.model, psam_b200.engine; "
            "assert not any(k.startswith('oracle') for k in sys.modules)") % (os.path.join(REPO, "point-sam_b200"), REPO)
    subprocess.check_call([sys.executable, "-c", code])
