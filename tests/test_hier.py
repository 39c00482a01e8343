"""CPU tests of the hierarchical model (PointCloudSAMHier, pc_sam.py:377-496): the fp32 oracle reproduces the fixture minted
by the reference's own modules, the configuration mirrors configs/model/hier.yaml, and the decoder's new C-ABI entry
validates its arguments."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import hier_ref
from oracle.make_golden import state_checksum


def _golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "hier.npz"))
    B, M, N, G1, G2, K1, K2, R, seed = [int(v) for v in g["meta"]]
    return g, dict(B=B, M=M, N=N, G=(G1, G2), K=(K1, K2), R=R, seed=seed, radius=tuple(float(r) for r in g["radius"]))


def test_oracle_reproduces_reference_hier_forward(golden_dir):
    g, m = _golden(golden_dir)
    oracle = hier_ref.build_hier_model(str(g["encoder"]), m["G"], m["K"], m["radius"], prompt_iters=m["R"], seed=1234 + m["seed"])
    assert state_checksum(oracle.state_dict()) == str(g["weights_checksum"])
    xyz, feats = torch.from_numpy(g["xyz"]), torch.from_numpy(g["feats"])
    seq_c = [torch.from_numpy(g[f"prompt_coords{t}"]) for t in range(m["R"])]
    seq_l = [torch.from_numpy(g[f"prompt_labels{t}"]) for t in range(m["R"])]
    with torch.no_grad():
        emb, (p1, p2) = oracle.pc_encoder(xyz, feats)
        outs = oracle.predict_iterative(xyz, feats, seq_c, seq_l)
    np.testing.assert_allclose(p1["embeddings"].numpy(), g["emb1"], atol=1e-5)
    np.testing.assert_allclose(p2["embeddings"].numpy(), g["emb2"], atol=1e-5)
    np.testing.assert_allclose(emb.numpy(), g["pc_embeddings"], atol=1e-5)
    assert [tuple(o["masks"].shape) for o in outs] == [(4, 3, m["N"]), (4, 1, m["N"]), (4, 1, m["N"])]
    for t, o in enumerate(outs):
        np.testing.assert_allclose(o["masks"].numpy(), g[f"masks{t}"], atol=1e-5)
        np.testing.assert_allclose(o["iou_preds"].numpy(), g[f"iou{t}"], atol=1e-5)
        np.testing.assert_allclose(o["prompt_masks"].numpy(), g[f"prompt_masks{t}"], atol=1e-5)
    # the one-round form equals round 0 of the loop
    with torch.no_grad():
        masks, iou = oracle.predict_masks(xyz, feats, seq_c[0], seq_l[0], None, True)
    np.testing.assert_allclose(masks.numpy(), g["masks0"], atol=1e-5)


def test_hier_config_mirrors_hier_yaml_and_state_dict_keys():
    from pc_sam.model import PointCloudSAMHier, build_point_sam_hier
    from pc_sam.model.mask_decoder import MaskDecoderHier
    from pc_sam.model.pc_encoder import PatchEmbedHier
    from pc_sam.model.prompt_encoder import MaskEncoderHier
    from pc_sam.utils import config

    cfg = config.model_config("hier")
    assert cfg["_target_"] == "pc_sam.model.pc_sam.PointCloudSAMHier" and cfg["prompt_iters"] == 8
    pe = cfg["pc_encoder"]["patch_embed"]
    assert (pe["num_patches"], pe["patch_size"], pe["radius"], pe["out_channels"]) == ([2048, 512], [32, 32], [0.05, 0.1], 512)
    assert cfg["pc_encoder"]["transformer"]["model_name"] == "eva02_large_patch14_448"
    assert cfg["mask_encoder"] == {"_target_": "pc_sam.model.prompt_encoder.MaskEncoderHier", "embed_dim": 256,
                                   "radius": [0.05, 0.1]}
    cfg["pc_encoder"]["transformer"]["model_name"] = "eva02_test_tiny"  # same module tree, small enough for a CPU test
    model = config.instantiate(cfg)
    assert isinstance(model, PointCloudSAMHier) and model.prompt_iters == 8
    assert isinstance(model.pc_encoder.patch_embed, PatchEmbedHier)
    assert isinstance(model.mask_encoder, MaskEncoderHier) and model.mask_encoder.radius == [0.05, 0.1]
    assert isinstance(model.mask_decoder, MaskDecoderHier)
    g1, g2 = model.pc_encoder.patch_embed.grouper1, model.pc_encoder.patch_embed.grouper2
    assert (g1.num_groups, g1.group_size, g1.radius, g2.num_groups, g2.group_size, g2.radius) == (2048, 32, 0.05, 512, 32, 0.1)
    ref = hier_ref.build_hier_model("eva02_test_tiny", seed=5)
    assert list(model.state_dict().keys()) == list(ref.state_dict().keys())
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    model.load_state_dict(ref.state_dict(), strict=True)
    built = build_point_sam_hier("eva02_test_tiny")
    assert list(built.state_dict().keys()) == list(ref.state_dict().keys())
    with pytest.raises(NotImplementedError):
        built.train()(torch.zeros(1, 16, 3), torch.zeros(1, 16, 3), torch.zeros(1, 1, 16, dtype=torch.bool))


def test_set_group_shape_leaves_hierarchical_tokenizer():
    from evaluation import eval_kitti
    from pc_sam.model import build_point_sam_hier

    m = build_point_sam_hier("eva02_test_tiny", (64, 16), (16, 8), (0.2, 0.4))
    eval_kitti.set_group_shape(m, 40000)
    pe = m.pc_encoder.patch_embed
    assert (pe.grouper1.num_groups, pe.grouper1.group_size, pe.grouper2.num_groups, pe.grouper2.group_size) == (64, 16, 16, 8)


def test_interp_add_ln_gelu_argument_validation_without_gpu():
    from psam_b200 import build

    lib = ctypes.CDLL(build.build())
    fn = lib.psam_interp_add_ln_gelu
    fn.restype = ctypes.c_int
    p = ctypes.c_void_p(16)  # never dereferenced: the arguments are rejected before any CUDA call
    eps = ctypes.c_float(1e-5)
    ll = ctypes.c_longlong

    def call(f=p, addend=p, D=256, Z=4, rep=2):
        return fn(f, Z, rep, 32, D, p, p, 100, addend, p, p, eps, p, ll(100 * 256), ll(256), None)

    assert call(f=None) == -1
    assert call(addend=None) == -1
    assert call(Z=0) == -1
    assert call(rep=0) == -1
    assert call(D=96) == -2
    assert call(D=2048) == -2
    assert call(D=384) == -2
