"""CPU tests of mask_decoder fine-tuning: the training-mode refusals (before any device work), the C-ABI argument validation
of the fine-tuning entry points, the fp64 oracle restatement (oracle/train_ref.py) against the reference's own code
(tests/golden/train.npz), and Criterion through the config reader."""
import ctypes
import os

import numpy as np
import pytest
import torch


def _tiny():
    from pc_sam.model import build_point_sam

    return build_point_sam("eva02_test_tiny", 8, 4)


def _inputs():
    return torch.zeros(1, 16, 3), torch.zeros(1, 16, 3), torch.zeros(1, 1, 16, dtype=torch.bool)


def test_training_refuses_a_trainable_parameter_outside_the_decoder_and_names_it():
    m = _tiny().train()
    with pytest.raises(NotImplementedError, match=r"pc_encoder\..*requires_grad=True.*model.requires_grad_\(False\).*"
                                                  r"model.mask_decoder.requires_grad_\(True\)"):
        m(*_inputs())
    m.requires_grad_(False)
    m.mask_decoder.requires_grad_(True)
    m.point_encoder.point_embeddings[0].weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match=r"'point_encoder.point_embeddings.0.weight'"):
        m(*_inputs())


def test_partly_frozen_decoder_passes_the_refusals():
    """Only mask_decoder parameters train, some of them frozen: the checks pass and the call reaches the device (which a
    CPU model does not have: the engine's CUDA-only error, not a refusal)."""
    m = _tiny().train()
    m.requires_grad_(False)
    m.mask_decoder.output_hypernetworks_mlps.requires_grad_(True)
    m._check_trainable()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(*_inputs())


def test_hier_varlen_and_generators_keep_refusing_training():
    from pc_sam.model import build_point_sam_hier

    h = build_point_sam_hier("eva02_test_tiny").train()
    h.requires_grad_(False)
    h.mask_decoder.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="PointCloudSAMHier"):
        h(*_inputs())
    m = _tiny().train()
    m.requires_grad_(False)
    m.mask_decoder.requires_grad_(True)
    with pytest.raises(NotImplementedError):
        m.forward_varlen([torch.zeros(16, 3)], [torch.zeros(16, 3)], [torch.zeros(1, 16, dtype=torch.bool)])


def test_training_refuses_an_active_drop_path():
    m = _tiny().train()
    m.requires_grad_(False)
    m.mask_decoder.requires_grad_(True)
    blk = m.pc_encoder.transformer.blocks[0]
    blk.drop_path1 = torch.nn.Dropout(0.1)
    with pytest.raises(NotImplementedError, match="drop_path1"):
        m(*_inputs())


@pytest.fixture(scope="module")
def lib():
    from psam_b200 import build

    return ctypes.CDLL(build.build())


def test_finetune_entry_points_validate_arguments_without_gpu(lib):
    """Bad arguments are rejected before any CUDA call (PSAM_ERR_ARG = -1)."""
    P = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    f = ctypes.c_float(1e-5)
    for fn in ("psam_mask_loss_stats", "psam_mask_loss_grad", "psam_interp_inverse", "psam_head_dp", "psam_interp_ln_gelu_backward",
               "psam_interp_backward", "psam_sum_partials"):
        getattr(lib, fn).restype = ctypes.c_int
    assert lib.psam_mask_loss_stats(None, P, 1, 1, 8, P, P, None) == -1
    assert lib.psam_mask_loss_stats(P, P, 1, 0, 8, P, P, None) == -1
    assert lib.psam_mask_loss_grad(P, P, 1, 1, 8, P, None, P, None) == -1
    assert lib.psam_mask_loss_grad(P, P, 256, 256, 8, P, P, P, None) == -1  # Z * C > 65535
    assert lib.psam_interp_inverse(P, 1, 8, 0, P, P, None) == -1
    assert lib.psam_interp_inverse(P, 1, 8, 8193, P, P, None) == -1
    assert lib.psam_head_dp(P, P, P, 1, 9, 8, 256, P, ctypes.c_longlong(0), ctypes.c_longlong(256), P, P, None) == -1  # C > 8
    assert lib.psam_head_dp(P, P, P, 1, 3, 8, 250, P, ctypes.c_longlong(0), ctypes.c_longlong(256), P, P, None) == -1  # D % 32
    assert lib.psam_interp_ln_gelu_backward(P, 1, 1, 4, 256, P, P, 8, P, P, f, None, P, 256, None) == -1
    assert lib.psam_interp_ln_gelu_backward(P, 1, 1, 4, 1024, P, P, 8, P, P, f, P, P, 256, None) == -2  # D > 512
    assert lib.psam_interp_backward(P, 1, 1, 4, 256, None, P, P, 8, P, None) == -1
    assert lib.psam_interp_backward(P, 1, 1, 4, 200, P, P, P, 8, P, None) == -2
    assert lib.psam_sum_partials(P, 1, 0, ctypes.c_longlong(4), P, None) == -1
    lib.psam_head_dp_chunks.restype = ctypes.c_int
    assert lib.psam_head_dp_chunks(32768) == 256 and lib.psam_head_dp_chunks(1) == 1


def test_oracle_restatement_matches_reference_golden(golden_dir):
    """oracle/train_ref.py (decoder loop over torch_ref.MaskDecoder, restated focal / dice / Criterion) in fp64 against the
    reference's own MaskDecoder and Criterion (tests/golden/train.npz): masks, loss, aux and every parameter gradient."""
    from oracle import torch_ref, train_ref

    g = np.load(os.path.join(golden_dir, "train.npz"), allow_pickle=False)
    D, MLP, B, M, G, N = [int(v) for v in g["dims"]]
    md = torch_ref.MaskDecoder(D, torch_ref.TwoWayTransformer(2, D, 8, MLP)).double()
    train_ref.fill_params(md, int(g["seed"]))
    t = lambda k: torch.from_numpy(g[k])
    aux = torch_ref.AuxInputs(coords=None, features=None, centers=None, interp_index=t("interp_index"),
                              interp_weight=t("interp_weight"))
    outs = train_ref.decoder_loop(md, t("pc_embeddings"), t("pc_pe"), [(t("sparse0"), t("dense0")), (t("sparse1"), t("dense1"))], aux)
    loss, aux_out = train_ref.criterion(outs, t("gt"))
    loss.backward()
    for i, o in enumerate(outs):
        np.testing.assert_allclose(o["masks"].detach().numpy(), g[f"masks{i}"], rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(o["iou_preds"].detach().numpy(), g[f"iou_preds{i}"], rtol=1e-10, atol=1e-12)
        assert np.array_equal(aux_out[i]["iou"].numpy(), g[f"aux{i}_iou"])
        for k in ("best_masks", "loss_mask", "loss_iou"):
            np.testing.assert_allclose(aux_out[i][k].detach().numpy(), g[f"aux{i}_{k}"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(float(loss.detach()), float(g["loss"]), rtol=1e-12)
    names = [str(n) for n in g["grad_names"]]
    assert names == [n for n, _ in md.named_parameters()]
    for n, p, want in zip(names, md.parameters(), g["grad_probes"]):
        np.testing.assert_allclose(train_ref.grad_probe(n, p.grad), want, rtol=1e-8, atol=1e-12, err_msg=n)


def test_criterion_reachable_through_the_config_target(tmp_path):
    from pc_sam.model.loss import Criterion
    from pc_sam.utils import config

    (tmp_path / "loss").mkdir()
    (tmp_path / "loss" / "default.yaml").write_text("_target_: pc_sam.model.loss.Criterion\n")
    (tmp_path / "top.yaml").write_text("defaults:\n  - loss: default\n  - _self_\n")
    crit = config.instantiate(config.compose(str(tmp_path), "top")["loss"])
    assert isinstance(crit, Criterion) and crit.use_soft_iou is False
    assert config.instantiate({"_target_": "pc_sam.model.loss.Criterion", "use_soft_iou": True}).use_soft_iou is True
