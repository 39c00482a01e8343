"""ORACLE (test infrastructure, NOT product code).

Trained-like parameters for the seeded oracle models, and their fp64 reference outputs.

Default initialisation gives every LayerNorm gamma = 1 and beta = 0, zero q / v biases on fused-qkv attention and one eps
per kind of LayerNorm.  Under those values a dropped or misrouted LayerNorm or bias term in the engine's weight packing
computes exactly the right answer.  ``perturb`` draws them the way a trained checkpoint has them, with large distinct eps so
that eps routing is observable; ``copy_to`` moves the perturbed weights (and each LayerNorm's eps, which the state dict
does not carry) into a CUDA-path model before its first call.

``reference`` runs the oracle in fp64.  Neighbour selection stays the fp32 one: ``fp32_neighbours`` chooses the k nearest
by fp32 distance and returns the fp64 distances of those neighbours, so near-ties at the k-th neighbour cannot make the fp64
run group or interpolate differently from the fp32 oracle (and the CUDA path).  FPS already runs in fp32.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Sequence, Tuple, Union

import torch
import torch.nn as nn

from . import torch_ref

EPS_SET = (1.0, 2.0, 4.0, 8.0)
QV = ("q_bias", "v_bias")


def layernorms(model: nn.Module) -> List[Tuple[str, nn.LayerNorm]]:
    return [(n, m) for n, m in model.named_modules() if isinstance(m, nn.LayerNorm)]


def qv_biases(model: nn.Module) -> List[Tuple[str, nn.Parameter]]:
    return [(f"{n}.{a}", getattr(m, a)) for n, m in model.named_modules() for a in QV
            if isinstance(getattr(m, a, None), nn.Parameter)]


# LayerNorms whose output reaches the compared outputs only weakly (the mask encoders feed the dense prompt embedding,
# one addend of the decoder's keys) get a larger draw, so that reverting any one of them still moves the outputs
SCALE = {"": (0.5, 0.3), "mask_encoder.": (3.0, 2.0)}


def _scale(name: str):
    return SCALE[max((p for p in SCALE if name.startswith(p)), key=len)]


def perturb(model: nn.Module, seed: int, eps: Union[float, Sequence[float]] = EPS_SET, calibrate=None) -> Dict[str, list]:
    """In place: every LayerNorm gets gamma = 1 + a N(0,1) and beta = b N(0,1), (a, b) = (0.5, 0.3) (larger in the mask
    encoders, SCALE), and an eps; every q_bias / v_bias gets 0.3 N(0,1).  k_bias stays the zero buffer timm defines.
    eps: one value for all, or a set used in rotation (the i-th LayerNorm in named_modules order takes eps[i % len(eps)]).
    With `calibrate` (a function that runs the model once) the set is relative: eps_i = eps[i % len(eps)] times the mean
    row variance of the LayerNorm's input in that run.  EPS_SET then scales every LayerNorm's output by 0.71 to 0.33,
    whatever the scale of its input; smaller eps were not observable behind the next LayerNorm, which undoes most of such a
    scale.  Returns the names touched, and asserts that they are every LayerNorm and q / v bias the module tree has."""
    g = torch.Generator().manual_seed(seed)
    eps = (float(eps),) if isinstance(eps, (int, float)) else tuple(eps)
    lns, qv = layernorms(model), qv_biases(model)
    with torch.no_grad():
        for i, (n, m) in enumerate(lns):
            assert m.weight is not None and m.bias is not None, f"{n}: LayerNorm without affine parameters"
            a, b = _scale(n)
            m.weight.copy_(1 + a * torch.randn(m.weight.shape, generator=g, dtype=torch.float64))
            m.bias.copy_(b * torch.randn(m.bias.shape, generator=g, dtype=torch.float64))
            m.eps = eps[i % len(eps)]
        for n, p in qv:
            p.copy_(0.3 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    if calibrate is not None:
        var = {n: [] for n, _ in lns}
        hooks = [m.register_forward_pre_hook(
            lambda mod, x, n=n: var[n].append(float(x[0].double().var(-1, unbiased=False).mean()))) for n, m in lns]
        try:
            calibrate(model)
        finally:
            for h in hooks:
                h.remove()
        for i, (n, m) in enumerate(lns):
            assert var[n], f"{n}: the calibration run does not reach this LayerNorm"
            m.eps = eps[i % len(eps)] * sum(var[n]) / len(var[n])
    # a normalisation this helper does not perturb (RMSNorm, GroupNorm, any module carrying an eps) or a bias parameter
    # that is neither a Linear or convolution bias nor q_bias / v_bias would leave its plumbing untested: refuse the model
    other_norms = [n for n, m in model.named_modules()
                   if not isinstance(m, nn.LayerNorm) and ("Norm" in type(m).__name__ or hasattr(m, "eps"))]
    assert not other_norms, f"normalisation modules perturb() does not handle: {other_norms}"
    plain = (nn.Linear, nn.LayerNorm, nn.modules.conv._ConvNd)
    linear_biases = {f"{n}.bias" for n, m in model.named_modules() if isinstance(m, plain)}
    other_biases = [n for n, _ in model.named_parameters() if "bias" in n.rsplit(".", 1)[-1]
                    and n not in linear_biases and n.rsplit(".", 1)[-1] not in QV]
    assert not other_biases, f"bias parameters perturb() does not handle: {other_biases}"
    assert sorted(n for n, _ in model.named_parameters() if n.rsplit(".", 1)[-1] in QV) == sorted(n for n, _ in qv)
    for n, m in lns:
        assert not torch.all(m.weight == 1) and not torch.all(m.bias == 0), n
    return dict(layernorms=[n for n, _ in lns], qv=[n for n, _ in qv])


def copy_to(src: nn.Module, dst: nn.Module) -> None:
    """dst <- src: load_state_dict(strict=True) plus every LayerNorm's eps.  Call it before dst's first CUDA call (the
    engine's packed-weight cache does not see eps)."""
    dst.load_state_dict(src.state_dict(), strict=True)
    a, b = dict(layernorms(src)), dict(layernorms(dst))
    assert a.keys() == b.keys(), sorted(set(a) ^ set(b))
    for n, m in b.items():
        m.eps = a[n].eps


@contextlib.contextmanager
def fp32_neighbours():
    """torch_ref.knn_points choosing neighbours by fp32 distance and returning their distances in the query's dtype."""
    orig = torch_ref.knn_points

    def knn(query, key, k, sorted=False):
        _, idx = orig(query.float(), key.float(), k, sorted)
        d = torch.cdist(query, key, compute_mode="donot_use_mm_for_euclid_dist")
        return torch.gather(d, 2, idx), idx

    torch_ref.knn_points = knn
    try:
        yield
    finally:
        torch_ref.knn_points = orig


def reference(oracle: nn.Module, xyz, feats, pc, pl, pm=None) -> Dict[str, torch.Tensor]:
    """fp64 outputs of a (perturbed) PointCloudSAM / PointCloudSAMHier oracle, on the device of its parameters:
    patch embeddings of every tokenizer level, pc_embeddings, the multimask pass without a prompt mask (masks, iou), the mask
    encoder's outputs for prompt mask pm (mask_embeddings, every level), and a single-mask pass with prompt mask pm
    (masks2, iou2; default: mask 1 of the multimask pass, rounded to fp32).  Also the fp32-selected fps / knn indices.
    The oracle is converted to fp64 in place."""
    oracle.double()
    dev = next(oracle.parameters()).device
    x, f, c = (t.to(dev, torch.float64) for t in (xyz, feats, pc))
    l = pl.to(dev)
    out = {}
    with torch.no_grad(), fp32_neighbours():
        emb, patches = oracle.pc_encoder(x, f)
        levels = patches if isinstance(patches, list) else [patches]
        for i, p in enumerate(levels):
            out[f"patch_embeddings{i}"] = p["embeddings"]
            out[f"fps_idx{i}"] = p["fps_idx"]
            out[f"knn_idx{i}"] = torch.sort(p["knn_idx"], -1).values
        out["pc_embeddings"] = emb
        out["masks"], out["iou"] = oracle.predict_masks(x, f, c, l, None, True)
        pm = out["masks"][:, 1].float() if pm is None else pm.to(dev)
        out["pm"] = pm
        for i, e in enumerate(mask_embeddings(oracle.mask_encoder, pm.double(), x, patches)):
            out[f"mask_embeddings{i}"] = e
        out["masks2"], out["iou2"] = oracle.predict_masks(x, f, c, l, pm.double(), False)
    return out


def mask_embeddings(mask_encoder, pm, x, patches) -> list:
    """The mask encoder's outputs for prompt mask pm: [dense] (MaskEncoder) or [level 1, level 2] (MaskEncoderHier)."""
    if isinstance(patches, list):
        p1, p2 = patches
        return mask_encoder(pm, x, p1["centers"], p1["knn_idx"], p2["centers"], p2["knn_idx"])
    return [mask_encoder(pm, x, patches["centers"], patches["knn_idx"])]


# output family -> (atol, rtol): encoder outputs at the tokenizer / ViT bound, decoder outputs at the north-star bound
BOUNDS = {"patch_embeddings": (2e-4, 1e-3), "pc_embeddings": (2e-4, 1e-3), "mask_embeddings": (2e-4, 1e-3),
          "masks": (1e-3, 1e-2), "iou": (1e-3, 1e-2)}


def family(key: str) -> str:
    return key.rstrip("0123456789")


def ratio(got: torch.Tensor, want: torch.Tensor, key: str) -> float:
    """max |got - want| / (atol + rtol |want|) for the output family of `key`: <= 1 is within the bound."""
    atol, rtol = BOUNDS[family(key)]
    g, w = got.detach().to(want.device, torch.float64), want.detach().double()
    assert g.shape == w.shape, (key, tuple(g.shape), tuple(w.shape))
    return float(((g - w).abs() / (atol + rtol * w.abs())).max())


COMPARED = ("patch_embeddings", "pc_embeddings", "mask_embeddings", "masks", "iou")


def compared(out: Dict[str, torch.Tensor]) -> List[str]:
    return [k for k in out if family(k) in COMPARED]


# ------------------------------------------------------------------------------------------------
# model configurations
# ------------------------------------------------------------------------------------------------
# encoder shapes used only by the tests (not timm models), registered for the duration of a build:
#   dh64: two 64-wide heads (the fused attention kernel's main form), SwiGLU 688 wide (fc2 with split-K 2 at 128 rows)
#   gelu_d352: fused qkv with q / v bias, four 88-wide heads, GELU MLP 512 wide: the LayerNorm-free block with a GELU MLP
TEST_EVA = {
    "psam_test_dh64": (128, 2, 2, 688, False, True, 28, 14),
    "psam_test_gelu_d352": (352, 2, 4, 512, True, False, 28, 14),
}


@contextlib.contextmanager
def eva_configs(*tables):
    """TEST_EVA added to each EVA_CONFIGS dict in `tables` for the duration of the block."""
    added = [(t, k) for t in tables for k in TEST_EVA if k not in t]
    for t, k in added:
        t[k] = TEST_EVA[k]
    try:
        yield
    finally:
        for t, k in added:
            del t[k]


def spec(kind="base", enc="eva02_test_tiny", G=64, K=32, N=2048, seed=101, tail="fc_norm", dec_act="relu",
         centralize=False, radius=None, eps=EPS_SET) -> dict:
    """One model configuration.  kind: "base" (PointCloudSAM) or "hier" (PointCloudSAMHier, G / K / radius per level).
    tail: the LayerNorms after the blocks - "fc_norm" (timm's), "both" (norm and fc_norm) or "none".
    dec_act: the two-way transformer's MLP activation.  centralize: the tokenizer's KNNGrouper with radius 0.3 and
    centralize_features (9 input channels)."""
    return dict(kind=kind, enc=enc, G=G, K=K, N=N, seed=seed, tail=tail, dec_act=dec_act, centralize=centralize,
                radius=radius, eps=eps)


def restructure(model: nn.Module, s: dict, ns) -> nn.Module:
    """Apply the structural options of spec `s` to a freshly built model whose module classes live in namespace `ns`
    (LayerNorm, Identity, TwoWayTransformer, PatchEmbed): the oracle's and the CUDA path's trees come out the same."""
    tr = model.pc_encoder.transformer
    D = model.pc_encoder.transformer_dim
    if s["tail"] == "both":
        tr.norm = nn.LayerNorm(D, eps=1e-6)
    elif s["tail"] == "none":
        tr.fc_norm = nn.Identity()
    if s["dec_act"] == "gelu":
        model.mask_decoder.transformer = ns.TwoWayTransformer(2, 256, 8, 2048, activation=nn.GELU)
    if s["centralize"]:
        model.pc_encoder.patch_embed = ns.PatchEmbed(9, 512, s["G"], s["K"], radius=0.3, centralize_features=True)
    return model.eval()


def build_oracle(s: dict) -> nn.Module:
    """The fp32 oracle of spec `s`, seeded, restructured and perturbed."""
    from . import hier_ref

    with eva_configs(torch_ref.EVA_CONFIGS):
        if s["kind"] == "hier":
            m = hier_ref.build_hier_model(s["enc"], s["G"], s["K"], s["radius"], prompt_iters=1, seed=s["seed"])
        else:
            m = torch_ref.build_model(s["enc"], s["G"], s["K"], seed=s["seed"])
    restructure(m, s, torch_ref)
    calibrate = None
    if not isinstance(s["eps"], float):  # an eps set is relative to the input variance seen on the spec's own inputs
        x, f, c, l = inputs(s)

        def calibrate(model):
            with torch.no_grad():
                masks, _ = model.predict_masks(x, f, c, l, None, True)
                model.predict_masks(x, f, c, l, masks[:, 1], False)
    perturb(m, s["seed"] + 1, s["eps"], calibrate)
    return m


# the model configurations of tests/test_gpu_model_params.py (tests/test_model_params.py checks each on the CPU)
GPU_CONFIGS = {
    "tiny": spec(),                                                    # D 128, 4 x 32 heads, SwiGLU 344, K 32, N 2048
    "tiny_k24_n2000": spec(K=24, N=2000),                              # group max kernel, mask dot kernel
    "dh64": spec(enc="psam_test_dh64", G=128),                         # L 128, fc2 split-K 2
    "dh64_long": spec(enc="psam_test_dh64", G=640, K=16, N=4096),      # L 640 > 512
    "dh88": spec(enc="eva_test_tiny_fused"),                           # D 176, 2 x 88 heads, q / v bias, GELU 256
    "gelu_d352": spec(enc="psam_test_gelu_d352"),                      # D 352, 4 x 88 heads, q / v bias, GELU 512
    "tail_both": spec(tail="both"),
    "tail_none": spec(tail="none"),
    "decoder_gelu": spec(dec_act="gelu"),
    "centralize": spec(centralize=True),
    "hier": spec(kind="hier", G=(128, 32), K=(32, 16), radius=(0.2, 0.4)),
}


def inputs(s: dict, B: int = 2, M: int = 2, P: int = 2):
    """B clouds of N points, B*M prompt sets of P points each (prompt sets b*M .. b*M+M-1 belong to cloud b)."""
    from . import synth

    xyz, feats = synth.make_batch(B, s["N"], s["seed"])
    pc, pl = synth.make_prompts(xyz, M * P, s["seed"] + 2)
    return xyz, feats, pc.reshape(B * M, P, 3), pl.reshape(B * M, P)
