"""Minimal stand-in for the two hydra calls the reference's entry points make (evaluation/inference.py:29-41):
``compose`` a YAML config with a ``defaults: [- model: X]`` list and ``instantiate`` a tree of ``_target_`` nodes.
Works on the reference's own ``configs/`` directory when it is present; hydra/omegaconf are not required."""
from __future__ import annotations

import importlib
import os
from typing import Any, Dict

import re

import yaml


class _Loader(yaml.SafeLoader):
    """YAML 1.1 reads ``3e-4`` as a string; OmegaConf (and the reference's configs: ``lr: 3e-4``) mean a float."""


_Loader.add_implicit_resolver("tag:yaml.org,2002:float",
                              re.compile(r"^[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)$"), list("-+0123456789."))


def _load(text):
    return yaml.load(text, Loader=_Loader)


def _import_target(path: str):
    mod, _, name = path.rpartition(".")
    if mod == "timm" and name == "create_model":
        try:
            return getattr(importlib.import_module("timm"), "create_model")
        except ImportError:  # offline image: the mirror builds the same module tree / state-dict keys
            from pc_sam.model.eva import create_model

            return create_model
    return getattr(importlib.import_module(mod), name)


def instantiate(node: Any):
    """Depth-first ``hydra.utils.instantiate``: dicts with ``_target_`` become calls, everything else is passed through."""
    if isinstance(node, dict):
        built = {k: instantiate(v) for k, v in node.items() if k != "_target_"}
        if "_target_" in node:
            return _import_target(node["_target_"])(**built)
        return built
    if isinstance(node, list):
        return [instantiate(v) for v in node]
    return node


def _merge(dst: Dict, src: Dict) -> Dict:
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = v
    return dst


def _load_group_file(directory: str, name: str) -> Dict:
    """One YAML file with its own (group-level) defaults list resolved inside its directory, e.g.
    configs/model/enc_with_radius.yaml: ``defaults: [default]`` then its own keys on top."""
    with open(os.path.join(directory, name.lstrip("/") + ".yaml")) as f:
        node = _load(f) or {}
    out: Dict = {}
    for d in node.pop("defaults", []) if isinstance(node, dict) else []:
        if d == "_self_":
            continue
        if isinstance(d, str):
            _merge(out, _load_group_file(directory, d))
        else:
            (group, option), = d.items()
            sub = os.path.join(directory, group.partition("@")[0])
            if os.path.exists(os.path.join(sub, str(option) + ".yaml")):
                out[group.partition("@")[2] or group.partition("@")[0]] = _load_group_file(sub, str(option))
    return _merge(out, node)


def compose(config_dir: str, config_name: str, overrides=()) -> Dict:
    """``hydra.compose`` for the subset the reference uses: the defaults list (``group: option`` and
    ``group@dest: option``), ``_self_`` ordering, and ``a.b.c=value`` overrides.  ``${...}`` interpolations are left as
    text (only logging paths use them)."""
    root = _load_group_file(config_dir, config_name)
    defaults = root.pop("defaults", [])
    cfg: Dict = {}
    for d in defaults:
        if d == "_self_":
            continue
        if isinstance(d, str):  # `- other` : another file of the same directory merged at the root
            _merge(cfg, _load_group_file(config_dir, d))
            continue
        (group, option), = d.items()
        group, _, dest = group.partition("@")
        if not os.path.exists(os.path.join(config_dir, group, str(option) + ".yaml")):
            continue  # dataset/loss groups are not needed for inference
        cfg[dest or group] = _load_group_file(os.path.join(config_dir, group), str(option))
    _merge(cfg, root)
    for ov in overrides:
        key, _, val = ov.partition("=")
        cur = cfg
        parts = key.split(".")
        for p in parts[:-1]:
            cur = cur.setdefault(p, {})
        cur[parts[-1]] = _load(val)
    return cfg


# The shipped model configurations (configs/model/{base,default,giant,hier}.yaml) as a function of the encoder name,
# for hosts without the reference's configs directory.
def model_config(name: str = "large") -> Dict:
    if name == "hier":
        return _hier_config()
    enc = {"base": "eva02_base_patch14_448", "large": "eva02_large_patch14_448", "default": "eva02_large_patch14_448",
           "giant": "eva_giant_patch14_560"}[name]
    G, K, iters = (1024, 256, 5) if name in ("large", "default") else (512, 64, 10)  # as shipped in configs/model/*.yaml
    return {"_target_": "pc_sam.model.pc_sam.PointCloudSAM",
            "pc_encoder": {"_target_": "pc_sam.model.pc_encoder.PointCloudEncoder",
                           "patch_embed": {"_target_": "pc_sam.model.pc_encoder.PatchEmbed", "in_channels": 6, "out_channels": 512,
                                           "num_patches": G, "patch_size": K},
                           "transformer": {"_target_": "timm.create_model", "model_name": enc, "pretrained": False},
                           "embed_dim": 256},
            "mask_encoder": {"_target_": "pc_sam.model.prompt_encoder.MaskEncoder", "embed_dim": 256},
            "mask_decoder": {"_target_": "pc_sam.model.mask_decoder.MaskDecoder", "transformer_dim": 256,
                             "transformer": {"_target_": "pc_sam.model.transformer.TwoWayTransformer", "depth": 2,
                                             "embedding_dim": 256, "num_heads": 8, "mlp_dim": 2048}},
            "prompt_iters": iters}


def _hier_config() -> Dict:
    """configs/model/hier.yaml: PointCloudSAMHier with the two-level tokenizer, mask encoder and upscaling decoder."""
    radius = [0.05, 0.1]
    return {"_target_": "pc_sam.model.pc_sam.PointCloudSAMHier",
            "pc_encoder": {"_target_": "pc_sam.model.pc_encoder.PointCloudEncoder",
                           "patch_embed": {"_target_": "pc_sam.model.pc_encoder.PatchEmbedHier", "in_channels": 6,
                                           "out_channels": 512, "num_patches": [2048, 512], "patch_size": [32, 32],
                                           "radius": list(radius)},
                           "transformer": {"_target_": "timm.create_model", "model_name": "eva02_large_patch14_448",
                                           "pretrained": False},
                           "embed_dim": 256},
            "mask_encoder": {"_target_": "pc_sam.model.prompt_encoder.MaskEncoderHier", "embed_dim": 256, "radius": list(radius)},
            "mask_decoder": {"_target_": "pc_sam.model.mask_decoder.MaskDecoderHier", "transformer_dim": 256,
                             "transformer": {"_target_": "pc_sam.model.transformer.TwoWayTransformer", "depth": 2,
                                             "embedding_dim": 256, "num_heads": 8, "mlp_dim": 2048}},
            "prompt_iters": 8}
