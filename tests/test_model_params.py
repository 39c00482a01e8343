"""The perturbed parameters of oracle/params_ref.py can see every LayerNorm and q / v bias (CPU, oracle only).

tests/test_gpu_model_params.py compares the CUDA path with the fp64 oracle on models whose LayerNorms and q / v biases
are drawn like trained ones.  That only pins the engine's routing of a parameter if the parameter moves the compared
outputs: here each one is reverted alone (gamma -> 1, beta -> 0, eps -> 1e-6, q_bias / v_bias -> 0) in the fp64 oracle,
and some compared output must move by a fixed multiple of its tolerance - 10x for gamma, beta and biases, 3x for eps."""
import copy

import pytest
import torch

from oracle import params_ref as pr
from oracle import torch_ref

MIN_MULT = {"gamma": 10.0, "beta": 10.0, "bias": 10.0, "eps": 3.0}

# the model classes and encoder forms of the GPU file (pr.GPU_CONFIGS), at CPU-sized shapes
MODELS = {
    "base_swiglu": pr.spec(N=1024, G=32),
    "base_gelu_fused_qkv_both_tail_gelu_decoder": pr.spec(enc="eva_test_tiny_fused", tail="both", dec_act="gelu", N=1024,
                                                          G=32),
    "base_dh64_no_tail": pr.spec(enc="psam_test_dh64", tail="none", N=1024, G=32, K=24),
    "base_gelu_d352_centralize": pr.spec(enc="psam_test_gelu_d352", centralize=True, N=1024, G=32),
    "hier": pr.spec(kind="hier", G=(64, 16), K=(32, 16), radius=(0.2, 0.4), N=1024),
}


def _groups(model):
    """(kind, name of the LayerNorm or bias parameter) for every perturbed group."""
    for n, _ in pr.layernorms(model):
        yield from (("gamma", n), ("beta", n), ("eps", n))
    for n, _ in pr.qv_biases(model):
        yield "bias", n


def _moves(out, base):
    """Largest move of any compared output, in multiples of its tolerance."""
    return max(pr.ratio(out[k], base[k], k) for k in pr.compared(base))


@pytest.mark.parametrize("name", list(MODELS))
def test_every_perturbed_group_moves_the_outputs(name):
    s = MODELS[name]
    with pr.eva_configs(torch_ref.EVA_CONFIGS):
        oracle = pr.build_oracle(s)
    inp = pr.inputs(s)
    ref = copy.deepcopy(oracle)
    base = pr.reference(ref, *inp)
    with torch.no_grad(), pr.fp32_neighbours():  # fp64 encoder outputs, reused where a group cannot change them
        enc = ref.pc_encoder(inp[0].double(), inp[1].double())
    worst = {}
    short = []
    for kind, n in _groups(oracle):
        m = copy.deepcopy(oracle)
        _revert(kind, dict(m.named_modules())[n.rsplit(".", 1)[0] if kind == "bias" else n], n)
        if not n.startswith("pc_encoder."):
            m.pc_encoder.forward = lambda *a: enc
        mult = _moves(pr.reference(m, *inp, pm=base["pm"]), base)
        if kind not in worst or mult < worst[kind][0]:
            worst[kind] = (mult, n)
        if mult < MIN_MULT[kind]:
            short.append(f"{kind} of {n}: {mult:.2f}x")
    print(f"[params] {name}: smallest move per group kind " +
          ", ".join(f"{k} {v[0]:.1f}x ({v[1]})" for k, v in sorted(worst.items())))
    assert not short, "reverting these moves no compared output enough: " + "; ".join(short)
    assert set(worst) >= {"gamma", "beta", "eps"}


def _revert(kind, target, name):
    with torch.no_grad():
        if kind == "gamma":
            target.weight.fill_(1.0)
        elif kind == "beta":
            target.bias.zero_()
        elif kind == "eps":
            target.eps = 1e-6
        else:
            getattr(target, name.rsplit(".", 1)[1]).zero_()


def test_voronoi_patch_embed_every_layernorm_moves_the_embeddings():
    """PatchEmbedNN (13 LayerNorms: two per residual block, six blocks, and the final one) at module level."""
    from oracle import synth

    torch.manual_seed(4323)
    m = torch_ref.PatchEmbedNN(7, 64, 96, 32).eval()
    names = pr.perturb(m, 4324)["layernorms"]
    assert len(names) == 13
    xyz, feats = synth.make_batch(2, 1024, 17)

    def run(mod):
        mod = copy.deepcopy(mod).double()
        with torch.no_grad(), pr.fp32_neighbours():
            return {"patch_embeddings": mod(xyz.double(), feats.double())["embeddings"]}

    base = run(m)
    worst = {}
    short = []
    for n in names:
        for kind in ("gamma", "beta", "eps"):
            c = copy.deepcopy(m)
            _revert(kind, dict(c.named_modules())[n], n)
            mult = _moves(run(c), base)
            if kind not in worst or mult < worst[kind][0]:
                worst[kind] = (mult, n)
            if mult < MIN_MULT[kind]:
                short.append(f"{kind} of {n}: {mult:.2f}x")
    print("[params] voronoi: smallest move per group kind " +
          ", ".join(f"{k} {v[0]:.1f}x ({v[1]})" for k, v in sorted(worst.items())))
    assert not short, "; ".join(short)


def test_perturb_touches_every_group_and_copy_to_carries_eps():
    """perturb touches every LayerNorm and q / v bias; copy_to carries each eps, which the state dict does not."""
    s = pr.spec(enc="eva_test_tiny_fused", tail="both", dec_act="gelu", N=1024, G=32)
    oracle = pr.build_oracle(s)
    lns, qv = pr.layernorms(oracle), pr.qv_biases(oracle)
    assert len(qv) == 4 and all(float(p.detach().abs().max()) > 0 for _, p in qv)
    assert len({m.eps for _, m in lns}) == len(lns)  # calibrated to each LayerNorm's input: all distinct
    other = pr.build_oracle(dict(s, seed=s["seed"] + 50))
    pr.copy_to(oracle, other)
    for (n, a), (_, b) in zip(lns, pr.layernorms(other)):
        assert a.eps == b.eps and torch.equal(a.weight, b.weight) and torch.equal(a.bias, b.bias), n
    # k_bias stays timm's zero buffer
    for n, m in oracle.named_modules():
        if getattr(m, "k_bias", None) is not None:
            assert float(m.k_bias.abs().max()) == 0.0, n
