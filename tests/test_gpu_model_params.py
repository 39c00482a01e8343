"""The whole model against the fp64 oracle with trained-like parameters, engine path by engine path.

Every other model test runs default-initialised weights: LayerNorm gamma = 1 and beta = 0, zero q / v biases and one eps per
kind of LayerNorm.  Under those values a dropped W beta term, swapped biases or a LayerNorm's parameters routed to another
one compute exactly the right answer.  Here the oracle's LayerNorms and q / v biases are drawn like a trained checkpoint's
(oracle/params_ref.py: gamma = 1 + 0.5 N, beta = 0.3 N, q / v bias 0.3 N, each eps 1 to 8 times its LayerNorm's input
variance; tests/test_model_params.py checks on the CPU that reverting any one of them moves the compared outputs by at
least 10x their tolerance, 3x for eps), copied into the CUDA model, and every engine branch is compared with the oracle
run in fp64 (neighbours chosen by fp32 distance, like the CUDA path).  Each case builds a fresh model (the engine reads its
switches when it packs a module) and its id names the branch it reaches; test_routing_guard checks under torch.profiler
that a representative of each branch launched its kernel.

Bounds: patch, point-cloud and mask-encoder embeddings 2e-4 abs + 1e-3 rel; masks and IoU 1e-3 abs + 1e-2 rel (the
north-star bound)."""
import os
import re
import subprocess
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import params_ref as pr  # noqa: E402
from oracle import torch_ref  # noqa: E402

# every engine switch, set for each case (a case overrides some)
SWITCHES = dict(FUSED_ATTENTION=True, FUSED_ATTENTION_LONG=True, ATTENTION_TWOPASS=False, FUSED_ATTENTION_DH88=True,
                FUSED_INNER_LN=True, FUSED_BLOCK_LN=True, BLOCK_LN_POLICY="never", FUSED_ROW_LN=True, DECODER_TC=True,
                FUSED_MASK_DOT=True)

CONFIGS = pr.GPU_CONFIGS

# Case ids are "-"-joined tokens; every token names a branch or a switch setting, and test_routing_guard checks each token of
# each id (_token_checks, _check_attn).
CASES = [
    # attention x block forms
    ("attn_unfused_dh32-block_ln-swiglu_inner_fold-splitk1-decoder_tc-rowdot", "tiny", {}),
    ("attn_unfused_dh32-block_ln-swiglu_inner_ln", "tiny", dict(FUSED_INNER_LN=False)),
    ("attn_unfused_dh32-block_folded-swiglu_inner_fold", "tiny", dict(BLOCK_LN_POLICY="always")),
    ("attn_fused_dh64_L128-block_ln-swiglu_inner_fold-splitk2", "dh64", {}),
    ("attn_fused_dh64_L128-block_ln-swiglu_inner_ln-splitk2", "dh64", dict(FUSED_INNER_LN=False)),
    ("attn_fused_dh64_L128-block_folded-swiglu_inner_fold", "dh64", dict(BLOCK_LN_POLICY="always")),
    ("attn_twopass_dh64_L128-twopass_on", "dh64", dict(ATTENTION_TWOPASS=True)),
    ("attn_fused_dh64_L640", "dh64_long", {}),
    ("attn_twopass_dh64_L640-twopass_on", "dh64_long", dict(ATTENTION_TWOPASS=True)),
    ("attn_unfused_dh64_L640-long_off", "dh64_long", dict(FUSED_ATTENTION_LONG=False)),
    ("attn_fused_dh88-qv_bias-block_ln-gelu_mlp", "dh88", {}),
    ("attn_fused_dh88-qv_bias-block_ln-gelu_mlp-policy_always", "dh88", dict(BLOCK_LN_POLICY="always")),
    ("attn_unfused_dh88-qv_bias-dh88_off", "dh88", dict(FUSED_ATTENTION_DH88=False)),
    ("attn_unfused_dh88-qv_bias-twopass_on", "dh88", dict(ATTENTION_TWOPASS=True)),
    ("attn_fused_dh88-qv_bias-block_ln-gelu_mlp-splitk2", "gelu_d352", {}),
    ("attn_fused_dh88-qv_bias-block_folded-gelu_mlp", "gelu_d352", dict(BLOCK_LN_POLICY="always")),
    # transformer tail
    ("tail_two_ln-block_ln", "tail_both", {}),
    ("tail_two_ln-block_ln-policy_always", "tail_both", dict(BLOCK_LN_POLICY="always")),
    ("tail_none-block_ln", "tail_none", {}),
    ("tail_none-block_ln-policy_always", "tail_none", dict(BLOCK_LN_POLICY="always")),
    # tokenizers
    ("gmax_epilogue-rowln_off", "tiny", dict(FUSED_ROW_LN=False)),
    ("group_max-rowln-mask_dot_kernel", "tiny_k24_n2000", {}),
    ("group_max-rowln_off-mask_dot_kernel-decoder_simt", "tiny_k24_n2000", dict(FUSED_ROW_LN=False, DECODER_TC=False)),
    ("centralize_radius-gmax_epilogue", "centralize", {}),
    # mask decoder
    ("decoder_simt-rowdot", "tiny", dict(DECODER_TC=False)),
    ("decoder_gelu-decoder_tc", "decoder_gelu", {}),
    ("decoder_gelu-decoder_simt", "decoder_gelu", dict(DECODER_TC=False)),
    # hierarchical model: level 2's mini-PointNet has Cin = 131 (conv1 on the tensor cores, LayerNorm after it)
    ("hier-wide_cin131-rowln-decoder_tc", "hier", {}),
    ("hier-wide_cin131-rowln_off-decoder_simt", "hier", dict(DECODER_TC=False, FUSED_ROW_LN=False)),
    ("hier-block_folded", "hier", dict(BLOCK_LN_POLICY="always")),
]


def _set_switches(setter, overrides):
    from psam_b200 import engine

    for k, v in dict(SWITCHES, **overrides).items():
        setter(engine, k, v)


def _build(s):
    """(CUDA model, fp32 oracle) of spec s: the oracle seeded, restructured and perturbed, its state and every eps copied
    into the CUDA model before the model's first call."""
    from pc_sam.model import build_point_sam, build_point_sam_hier, eva
    from pc_sam.model.pc_encoder import PatchEmbed
    from pc_sam.model.transformer import TwoWayTransformer

    with pr.eva_configs(eva.EVA_CONFIGS, torch_ref.EVA_CONFIGS):
        oracle = pr.build_oracle(s)
        if s["kind"] == "hier":
            model = build_point_sam_hier(s["enc"], s["G"], s["K"], s["radius"], 1)
        else:
            model = build_point_sam(s["enc"], s["G"], s["K"])
    pr.restructure(model, s, types.SimpleNamespace(TwoWayTransformer=TwoWayTransformer, PatchEmbed=PatchEmbed))
    pr.copy_to(oracle, model)
    return model.cuda().eval(), oracle


def _run(model, s, pm):
    """The CUDA path's outputs under the keys of pr.reference."""
    d = torch.device("cuda:0")
    x, f, c, l = (t.to(d) for t in pr.inputs(s))
    out = {}
    with torch.no_grad():
        emb, patches = model.pc_encoder(x, f)
        for i, p in enumerate(patches if isinstance(patches, list) else [patches]):
            out[f"patch_embeddings{i}"] = p["embeddings"]
            out[f"fps_idx{i}"] = p["fps_idx"]
            out[f"knn_idx{i}"] = torch.sort(p["knn_idx"], -1).values
        out["pc_embeddings"] = emb
        out["masks"], out["iou"] = model.predict_masks(x, f, c, l, None, True)
        for i, e in enumerate(pr.mask_embeddings(model.mask_encoder, pm.to(d), x, patches)):
            out[f"mask_embeddings{i}"] = e
        out["masks2"], out["iou2"] = model.predict_masks(x, f, c, l, pm.to(d), False)
    return out


def _compare(name, got, want):
    for k in want:
        if k.startswith(("fps_idx", "knn_idx")):
            assert torch.equal(got[k].cpu(), want[k].cpu()), f"{name}: {k} differs from the fp32 oracle's"
    ratios = {k: pr.ratio(got[k], want[k], k) for k in pr.compared(want)}
    print(f"[params] {name}: worst err/bound " + " ".join(f"{k}={v:.3f}" for k, v in ratios.items()))
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f"{name}: outside the bound (err/bound): {bad}"


@pytest.fixture(scope="module")
def reference():
    """fp64 oracle outputs, computed once per model configuration (they do not depend on the engine's switches)."""
    cache = {}

    def get(name):
        if name not in cache:
            s = CONFIGS[name]
            with pr.eva_configs(torch_ref.EVA_CONFIGS):
                cache[name] = pr.reference(pr.build_oracle(s), *pr.inputs(s))
        return cache[name]

    return get


@pytest.mark.parametrize("case,cfg,overrides", CASES, ids=[c[0] for c in CASES])
def test_model_vs_fp64(case, cfg, overrides, reference, monkeypatch):
    """B = 2 clouds x 2 prompt sets of 2 points: multimask pass without a prompt mask (the no-mask embedding broadcast),
    single-mask pass with one prompt mask per prompt set."""
    _set_switches(monkeypatch.setattr, overrides)
    want = reference(cfg)
    model, _ = _build(CONFIGS[cfg])
    _compare(case, _run(model, CONFIGS[cfg], want["pm"]), want)


@pytest.mark.parametrize("tc", [True, False], ids=["decoder_tc", "decoder_simt"])
def test_decoder_one_dense_map_for_all_prompt_sets(tc, monkeypatch):
    """The third dense-embedding form run_mask_decoder takes: one [1, G, D] map added to every prompt set.  The decoder alone,
    on the CUDA encoder's outputs, against the fp64 oracle decoder on the same inputs."""
    from psam_b200 import engine

    _set_switches(monkeypatch.setattr, dict(DECODER_TC=tc))
    s = CONFIGS["tiny"]
    model, oracle = _build(s)
    d = torch.device("cuda:0")
    x, f, c, l = (t.to(d) for t in pr.inputs(s))
    dense = torch.randn((1, s["G"], 256), generator=torch.Generator().manual_seed(5)).to(d)
    with torch.no_grad():
        enc = model._encode(x, f)
        sparse = engine.run_point_encoder(model.point_encoder, c, l)
        got = model.mask_decoder(enc["pc_embeddings"], enc["pc_pe"], sparse, dense, aux_inputs=enc["aux"], multimask_output=True)
        oracle.double()
        aux = torch_ref.AuxInputs(coords=x.cpu().double(), features=f.cpu().double(), centers=enc["aux"].centers.cpu().double())
        with pr.fp32_neighbours():
            want = oracle.mask_decoder(enc["pc_embeddings"].cpu().double(), enc["pc_pe"].cpu().double(), sparse.cpu().double(),
                                       dense.cpu().double(), aux, True)
    _compare(f"one dense map tc={tc}", {"masks": got[0], "iou": got[1]}, {"masks": want[0], "iou": want[1]})


def test_voronoi_patch_embed_nn_vs_fp64():
    """PatchEmbedNN at module level with its 13 LayerNorms perturbed: per-point residual blocks, maximum per Voronoi cell,
    per-cell blocks, final LayerNorm."""
    from oracle import synth
    from pc_sam.model.pc_encoder import PatchEmbedNN

    torch.manual_seed(4323)
    oracle = torch_ref.PatchEmbedNN(7, 64, 96, 32).eval()
    assert len(pr.perturb(oracle, 4324)["layernorms"]) == 13
    m = PatchEmbedNN(7, 64, 96, 32)
    pr.copy_to(oracle, m)
    m = m.cuda().eval()
    xyz, feats = synth.make_batch(2, 2048, 17)
    with torch.no_grad():
        got = m(xyz.cuda(), feats.cuda())
        with pr.fp32_neighbours():
            want = oracle.double()(xyz.double(), feats.double())
    assert torch.equal(got["nn_idx"].cpu(), want["nn_idx"])
    _compare("voronoi PatchEmbedNN", {"patch_embeddings": got["embeddings"]}, {"patch_embeddings": want["embeddings"]})


@pytest.fixture(scope="module")
def reference_vitl():
    s = pr.spec(enc="eva02_large_patch14_448", G=512, K=64, N=32768, seed=131, eps=1e-6)
    oracle = pr.build_oracle(s).cuda()
    return s, pr.reference(oracle, *pr.inputs(s))


@pytest.mark.parametrize("ln_policy", ["never", "always"])
def test_full_size_vitl_c2_vs_fp64(ln_policy, reference_vitl, monkeypatch):
    """ViT-L at the c2 shape (N = 32768, G = 512, K = 64), perturbed with timm's eps (1e-6), B = 2 x 2 prompt sets, with the
    LayerNorm kernels and the LayerNorm-free blocks, against the fp64 oracle run on the GPU."""
    _set_switches(monkeypatch.setattr, dict(BLOCK_LN_POLICY=ln_policy))
    s, want = reference_vitl
    model, _ = _build(s)
    _compare(f"ViT-L c2 policy={ln_policy}", _run(model, s, want["pm"]), want)


# ------------------------------------------------------------------------------------------------
# the packed-weight cache
# ------------------------------------------------------------------------------------------------
def _plain(s):
    """The spec's model with default initialisation (not perturbed)."""
    from pc_sam.model import build_point_sam

    oracle = torch_ref.build_model(s["enc"], s["G"], s["K"], seed=s["seed"])
    model = build_point_sam(s["enc"], s["G"], s["K"])
    pr.copy_to(oracle, model)
    return model


@pytest.mark.parametrize("how", ["load_state_dict", "inplace_no_grad", "cpu_cuda_round_trip"])
def test_packed_cache_follows_weight_changes(how, reference, monkeypatch):
    """One call packs the default-initialised weights; the perturbed ones then arrive by load_state_dict, by in-place copies
    under torch.no_grad(), or by load_state_dict while the model is on the CPU followed by .cuda().  The next call must
    match the oracle with the new weights.  Each LayerNorm's eps is assigned with the new weights, before that call."""
    _set_switches(monkeypatch.setattr, {})
    s = CONFIGS["dh88"]  # fused qkv: the q / v biases go through the cache too
    want = reference("dh88")
    model = _plain(s).cuda().eval()
    _run(model, s, want["pm"])
    perturbed, _ = _build(s)
    if how == "load_state_dict":
        pr.copy_to(perturbed, model)
    elif how == "inplace_no_grad":
        new = dict(perturbed.named_parameters())
        with torch.no_grad():
            for n, p in model.named_parameters():
                p.copy_(new[n])
        eps = {n: m.eps for n, m in pr.layernorms(perturbed)}
        for n, m in pr.layernorms(model):
            m.eps = eps[n]
    else:
        model.cpu()
        pr.copy_to(perturbed.cpu(), model)
        model.cuda()
    _compare(f"cache after {how}", _run(model, s, want["pm"]), want)


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def test_routing_guard():
    """Every case of test_model_vs_fp64 runs once more under the profiler, and every token of its id is checked against the
    kernels it launched and the engine's calls into ops (GUARD_TOKENS).  It runs in a fresh interpreter: after other work
    in one process the profiler has been seen to record no CUDA activity, and what the guard sees must not depend on what
    ran before it."""
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_model_params as t; t._routing_guard()" % (
        here, repo, os.path.join(repo, "point-sam_b200"))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def _count(ks, sub):
    return sum(sub in k for k in ks)


def _calls(r, name):
    return [(a, k) for n, a, k in r["log"] if n == name]


def _ln_rows(r, shape):
    return [a for a, k in _calls(r, "layernorm") if tuple(a[0].shape) == shape]


def _block_fold_gemms(r):
    return [k for a, k in _calls(r, "gemm") if k.get("ln_fold") is not None and k["ln_fold"][2] == r["D"]]


def _check_attn(r, tok):
    kind, dh, L = re.fullmatch(r"attn_(fused|unfused|twopass)_dh(\d+)(?:_L(\d+))?", tok).groups()
    assert int(dh) == r["dh"] and (L is None or int(L) == r["L"]), (r["dh"], r["L"])
    ks, depth = r["ks"], r["depth"]
    fused, twopass = f"attention_wgmma_kernel<{dh}, false>", f"attention_wgmma_kernel<{dh}, true>"
    if kind == "fused":
        return _count(ks, fused) == depth and not _count(ks, "softmax_split_kernel")
    if kind == "twopass":
        return _count(ks, twopass) == depth and not _count(ks, fused)
    return (_count(ks, "softmax_split_kernel") == depth and _count(ks, "transpose_split_kernel") == depth
            and not _count(ks, "attention_wgmma"))


def _packed_decoder_acts(r):
    return {l["act"] for l in r["model"].mask_decoder.__dict__["_psam_packed"][1].layers}


def _token_checks():
    from psam_b200 import ops

    gemm = lambda r: [k for _, k in _calls(r, "gemm")]
    md = lambda r: (r["M"], r["D"])
    return {
        "block_ln": lambda r: len(_ln_rows(r, md(r))) == 2 * r["depth"] + r["ntail"] and not _block_fold_gemms(r),
        "block_folded": lambda r: not _ln_rows(r, md(r)) and len(_block_fold_gemms(r)) == 2 * r["depth"] + 1,
        "swiglu_inner_fold": lambda r: (sum(k.get("swiglu", False) and k.get("stats_out") is not None for k in gemm(r))
                                        == r["depth"] and not any(k.get("padded") for _, k in _calls(r, "layernorm"))),
        "swiglu_inner_ln": lambda r: (sum(bool(k.get("padded")) for _, k in _calls(r, "layernorm")) == r["depth"]
                                      and sum(k.get("swiglu", False) for k in gemm(r)) == r["depth"]),
        "gelu_mlp": lambda r: not any(k.get("swiglu") for k in gemm(r)),
        "splitk1": lambda r: max(k.get("split_k", 1) for k in gemm(r)) == 1,
        "splitk2": lambda r: max(k.get("split_k", 1) for k in gemm(r)) == 2,
        "qv_bias": lambda r: all(b.attn.q_bias is not None and b.attn.v_bias is not None
                                 for b in r["model"].pc_encoder.transformer.blocks),
        "policy_always": lambda r: r["sw"]["BLOCK_LN_POLICY"] == "always",
        "twopass_on": lambda r: r["sw"]["ATTENTION_TWOPASS"],
        "dh88_off": lambda r: not r["sw"]["FUSED_ATTENTION_DH88"],
        "long_off": lambda r: not r["sw"]["FUSED_ATTENTION_LONG"] and r["L"] > 512,
        "tail_two_ln": lambda r: r["ntail"] == 2 and len(_ln_rows(r, md(r))) == 2 * r["depth"] + 2,
        "tail_none": lambda r: r["ntail"] == 0 and len(_ln_rows(r, md(r))) == 2 * r["depth"],
        "gmax_epilogue": lambda r: (any(k.get("gmax") is not None for k in gemm(r))
                                    and not _count(r["ks"], "group_max_kernel")),
        "group_max": lambda r: (_count(r["ks"], "group_max_kernel") == 2
                                and not any(k.get("gmax") is not None for k in gemm(r))),
        "rowln": lambda r: _count(r["ks"], "gemm_rowln_kernel") >= 1,
        "rowln_off": lambda r: (not _count(r["ks"], "gemm_rowln_kernel")
                                and any(k.get("gbias") is not None for _, k in _calls(r, "layernorm"))),
        "centralize_radius": lambda r: any(len(a) > 4 and a[4] is not None and k.get("center_idx") is not None
                                           for a, k in _calls(r, "group_gather")),
        # the patch-row projections of the two-way transformer (k / q, v per layer, k and v of the final attention,
        # output_upscaling[0]) write [Z*G, .] fp32 outputs from the tensor-core GEMM
        "decoder_tc": lambda r: sum(k.get("out_f32") is not None and k["out_f32"].shape[0] == r["ZG"] for k in gemm(r))
        == 2 * r["ndec"] + 3,
        "decoder_simt": lambda r: not any(k.get("out_f32") is not None and k["out_f32"].shape[0] == r["ZG"] for k in gemm(r)),
        "rowdot": lambda r: any(k.get("rowdot") is not None for k in gemm(r)) and not _count(r["ks"], "mask_dot_kernel"),
        "mask_dot_kernel": lambda r: (_count(r["ks"], "mask_dot_kernel") == 1
                                      and not any(k.get("rowdot") is not None for k in gemm(r))),
        "decoder_gelu": lambda r: _packed_decoder_acts(r) == {ops.ACT_GELU},
        "hier": lambda r: r["hier"],
        # level 2 (Cin = 131): conv1 on the tensor cores, then a LayerNorm over its B*G2*K2 rows; no small-input kernel
        "wide_cin131": lambda r: (any(isinstance(a[0], ops.Split) and a[0].cols == 131 for a, _ in _calls(r, "gemm"))
                                  and len(_ln_rows(r, (r["R2"], 128))) == 1
                                  and not any(a[0].shape[-1] == 131 for a, _ in _calls(r, "small_in_linear"))),
    }


def _routing_guard():
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from psam_b200 import engine, ops

    log = []
    for name in ("gemm", "layernorm", "small_in_linear", "group_gather"):
        def wrapped(*a, _f=getattr(ops, name), _n=name, **k):
            log.append((_n, a, k))
            return _f(*a, **k)
        setattr(ops, name, wrapped)

    d = torch.device("cuda:0")
    runs = []
    for case, cfg, overrides in CASES:  # build and pack everything before the profiled session
        _set_switches(setattr, overrides)
        s = CONFIGS[cfg]
        model, _ = _build(s)
        x, f, c, l = (t.to(d) for t in pr.inputs(s))
        with torch.no_grad():
            model.predict_masks(x, f, c, l, None, True)
        tr = model.pc_encoder.transformer
        hier = s["kind"] == "hier"
        G, K = (s["G"][-1], s["K"][-1]) if hier else (s["G"], s["K"])
        runs.append(dict(case=case, sw=dict(SWITCHES, **overrides), model=model, args=(x, f, c, l), hier=hier,
                         M=x.shape[0] * G, L=G, D=model.pc_encoder.transformer_dim, depth=len(tr.blocks),
                         dh=model.pc_encoder.transformer_dim // tr.blocks[0].attn.num_heads,
                         ntail=len(engine.validate_transformer(tr)), ZG=c.shape[0] * G,
                         ndec=len(model.mask_decoder.transformer.layers), R2=x.shape[0] * G * K))
    torch.cuda.synchronize()
    # one profiler session; a spin kernel (launched by nothing else) separates the runs
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for r in runs:
            torch.cuda._sleep(1000)
            _set_switches(setattr, {k: v for k, v in r["sw"].items()})
            n0 = len(log)
            with torch.no_grad():
                r["model"].predict_masks(*r["args"], None, True)
            torch.cuda.synchronize()
            r["log"] = log[n0:]
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "_kernel" in e.name),
                key=lambda e: e.time_range.start)
    segs, cur = [], None
    for e in ev:
        if "spin_kernel" in e.name:
            if cur is not None:
                segs.append(cur)
            cur = []
        elif cur is not None:
            cur.append(e.name)
    assert len(segs) == len(runs), f"{len(runs)} runs, {len(segs)} marker-separated kernel segments"
    checks = _token_checks()
    attn = re.compile(r"attn_(fused|unfused|twopass)_dh\d+(_L\d+)?")
    n = 0
    for r, ks in zip(runs, segs):
        r["ks"] = ks
        assert ks, f"{r['case']}: the profiler recorded no kernel"
        for tok in r["case"].split("-"):
            chk = (lambda r, tok=tok: _check_attn(r, tok)) if attn.fullmatch(tok) else checks.get(tok)
            assert chk is not None, f"{r['case']}: no guard check for '{tok}'"
            assert chk(r), f"{r['case']}: '{tok}' not reached; kernels {sorted(set(ks))}"
            n += 1
    print(f"[params] routing guard: {len(runs)} cases, {n} id tokens, each reached the branch it names")
