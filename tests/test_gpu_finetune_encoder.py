"""GPU tests of encoder fine-tuning: the row-wise backward kernels at every width the released and test encoders use, one
EvaBlock's backward and the whole ViT-L chain against fp64 (oracle/torch_ref with perturbed LayerNorms and q / v biases),
a whole teacher-forced training step, partial unfreezing, determinism, what the blocks save, the per-block weight cache
after an optimizer step, and the README loop with the last two blocks trainable."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import params_ref, torch_ref, train_ref  # noqa: E402

DEV = torch.device("cuda:0")


def _nrel(got, want):
    got, want = got.detach().double(), want.detach().double().to(got.device)
    return float((got - want).norm() / want.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 176, 768, 1024, 1408])
@pytest.mark.parametrize("M", [1, 257, 1000])
def test_layernorm_backward_against_fp64(D, M):
    from psam_b200 import train

    g = torch.Generator().manual_seed(D * 7 + M)
    x = (torch.randn(M, D, generator=g, dtype=torch.float64) * 2 + 3)
    dy = torch.randn(M, D, generator=g, dtype=torch.float64)
    dres = torch.randn(M, D, generator=g, dtype=torch.float64)
    w = 1 + 0.5 * torch.randn(D, generator=g, dtype=torch.float64)
    b = 0.3 * torch.randn(D, generator=g, dtype=torch.float64)
    xd, wd, bd = (t.clone().requires_grad_(True) for t in (x, w, b))
    F.layer_norm(xd, (D,), wd, bd, 1e-6).backward(dy)
    f = lambda t: t.float().to(DEV).contiguous()
    dx, part = train._ln_backward(f(x), f(dy), f(w), 1e-6, dres=f(dres))
    dg, db = train._ln_params(part)
    assert _nrel(dx, xd.grad + dres) < 1e-5 and _nrel(dg, wd.grad) < 1e-5 and _nrel(db, bd.grad) < 1e-5


@pytest.mark.parametrize("Hd", [344, 2048, 2730])
def test_swiglu_layernorm_backward_against_fp64(Hd):
    from psam_b200 import engine, native as nv, ops, train

    Hp, M = engine.swiglu_hidden_pad(Hd), 300
    g = torch.Generator().manual_seed(Hd)
    gx = torch.randn(M, 2, Hd, generator=g, dtype=torch.float64) * 2
    dhn = torch.randn(M, Hd, generator=g, dtype=torch.float64)
    w = 1 + 0.5 * torch.randn(Hd, generator=g, dtype=torch.float64)
    b = 0.3 * torch.randn(Hd, generator=g, dtype=torch.float64)
    gd, wd, bd = (t.clone().requires_grad_(True) for t in (gx, w, b))
    hn = F.layer_norm(F.silu(gd[:, 0]) * gd[:, 1], (Hd,), wd, bd, 1e-6)
    hn.backward(dhn)
    a = torch.zeros(M, 2 * Hp, dtype=torch.float32, device=DEV)
    a[:, 0:2 * Hd:2], a[:, 1:2 * Hd:2] = gx[:, 0].float().to(DEV), gx[:, 1].float().to(DEV)
    dh = torch.zeros(M, Hp, dtype=torch.float32, device=DEV)
    dh[:, :Hd] = dhn.float().to(DEV)
    gp, bp = torch.zeros(Hp, device=DEV), torch.zeros(Hp, device=DEV)
    gp[:Hd], bp[:Hd] = w.float().to(DEV), b.float().to(DEV)
    da = torch.full((M, 2 * Hp), float("nan"), device=DEV)
    das, hns = ops.Split(M, 2 * Hp, DEV), ops.Split(M, Hp, DEV, pitch=Hp)
    part = torch.empty(((M + 255) // 256, 2, Hd), device=DEV)
    nv.check(nv.lib().psam_swiglu_ln_backward(nv.ptr(a), 2 * Hp, M, Hd, Hp, nv.ptr(dh), Hp, nv.ptr(gp), nv.ptr(bp), 1e-6, nv.ptr(da),
                                              2 * Hp, das.ptr(), das.plane, das.pitch, hns.ptr(), hns.plane, hns.pitch, nv.ptr(part), 256,
                                              nv.stream()), "swiglu_ln_backward")
    dg, db = train._ln_params(part)
    assert _nrel(da[:, 0:2 * Hd:2], gd.grad[:, 0]) < 1e-5 and _nrel(da[:, 1:2 * Hd:2], gd.grad[:, 1]) < 1e-5
    assert torch.equal(da[:, 2 * Hd:], torch.zeros_like(da[:, 2 * Hd:]))
    assert _nrel(das.float(), da) < 1e-5  # hi + lo of two bf16 carry 16 significand bits: 2^-17 relative per element
    assert _nrel(hns.float()[:, :Hd], hn) < 1e-5 and not hns.float()[:, Hd:].any()
    assert _nrel(dg, wd.grad) < 1e-5 and _nrel(db, bd.grad) < 1e-5


@pytest.mark.parametrize("n", [256, 6144])
def test_gelu_backward_against_fp64(n):
    from psam_b200 import native as nv, ops

    M = 77
    g = torch.Generator().manual_seed(n)
    a = torch.randn(M, n, generator=g, dtype=torch.float64) * 3
    dh = torch.randn(M, n, generator=g, dtype=torch.float64)
    ad = a.clone().requires_grad_(True)
    h = F.gelu(ad)
    h.backward(dh)
    af, dhf = a.float().to(DEV), dh.float().to(DEV)
    da = torch.empty_like(af)
    das, hs = ops.Split(M, n, DEV), ops.Split(M, n, DEV)
    nv.check(nv.lib().psam_gelu_backward(nv.ptr(af), n, M, n, nv.ptr(dhf), n, nv.ptr(da), n, das.ptr(), das.plane, das.pitch, hs.ptr(),
                                         hs.plane, hs.pitch, nv.stream()), "gelu_backward")
    assert _nrel(da, ad.grad) < 1e-6 and _nrel(das.float(), ad.grad) < 1e-5 and _nrel(hs.float(), h) < 1e-5


@pytest.mark.parametrize("L", [100, 512])
def test_softmax_backward_against_fp64(L):
    from psam_b200 import native as nv, ops

    rows, scale = 3 * L + 5, 0.125
    g = torch.Generator().manual_seed(L)
    s = torch.randn(rows, L, generator=g, dtype=torch.float64) * 8
    dp = torch.randn(rows, L, generator=g, dtype=torch.float64)
    sd = s.clone().requires_grad_(True)
    torch.softmax(sd * scale, -1).backward(dp)
    ds = ops.Split(rows, L, DEV, pitch=ops._round_up(L, 64))
    sf, dpf = s.float().to(DEV), dp.float().to(DEV)
    nv.check(nv.lib().psam_softmax_backward(nv.ptr(sf), L, nv.ptr(dpf), L, rows, L, scale, ds.ptr(), ds.plane, ds.pitch, nv.stream()),
             "softmax_backward")
    assert _nrel(ds.float(), sd.grad) < 1e-5


# ------------------------------------------------------------------------------------------------
# one block, and the ViT-L chain
# ------------------------------------------------------------------------------------------------
def _blocks(name, n, seed):
    """n oracle EvaBlocks (fp64, perturbed LayerNorms and q / v biases, eps 1e-6) and the same weights as pc_sam modules."""
    from pc_sam.model.eva import EVA_CONFIGS, EvaBlock

    D, _, H, hid, fused, swiglu = EVA_CONFIGS[name][:6]
    torch.manual_seed(seed)
    ref = torch.nn.Sequential(*[torch_ref.EvaBlock(D, H, hid, fused, swiglu) for _ in range(n)]).double()
    params_ref.perturb(ref, seed, eps=1e-6)
    ours = torch.nn.Sequential(*[EvaBlock(D, H, hid, fused, swiglu) for _ in range(n)])
    ours.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    return ref.to(DEV), ours.to(DEV), D


def _apply(blocks, x, B, L):
    from psam_b200 import engine, train

    for blk in blocks:
        x = train.EvaBlockFn.apply(x, blk, engine.block_pack(blk, x.shape[1]), B, L, *blk.parameters())
    return x


@pytest.mark.parametrize("name,B,L", [("eva02_test_tiny", 2, 64), ("eva_test_tiny_fused", 2, 64), ("eva02_test_tiny", 1, 200),
                                      ("eva02_base_patch14_448", 1, 512), ("eva02_large_patch14_448", 2, 512),
                                      ("eva_giant_patch14_560", 1, 512), ("eva_giant_patch14_560", 2, 512)])
def test_block_backward_against_fp64(name, B, L):
    ref, ours, D = _blocks(name, 1, seed=31 * len(name) + B)
    g = torch.Generator().manual_seed(L + B)
    x = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    dy = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    xd = x.to(DEV).requires_grad_(True)
    ref(xd).backward(dy.to(DEV))
    xf = x.float().to(DEV).reshape(B * L, D).requires_grad_(True)
    y = _apply(ours, xf, B, L)
    y.backward(dy.float().to(DEV).reshape(B * L, D))
    assert _nrel(xf.grad.reshape(B, L, D), xd.grad) <= 1e-4
    for (n, p), (_, q) in zip(ours.named_parameters(), ref.named_parameters()):
        assert _nrel(p.grad, q.grad) <= 1e-4, n


def test_vit_large_chain_against_fp64():
    """All 24 ViT-L blocks, fc_norm and out_proj trainable, B = 2 clouds of 512 patches."""
    B, L = 2, 512
    ref, ours, D = _blocks("eva02_large_patch14_448", 24, seed=11)
    torch.manual_seed(12)
    norm, proj = torch.nn.LayerNorm(D, eps=1e-6).double(), torch.nn.Linear(D, 256).double()
    with torch.no_grad():
        norm.weight.copy_(1 + 0.5 * torch.randn(D, dtype=torch.float64))
        norm.bias.copy_(0.3 * torch.randn(D, dtype=torch.float64))
    norm, proj = norm.to(DEV), proj.to(DEV)
    norm32, proj32 = [torch.nn.Module.float(type(m)(*a).to(DEV)) for m, a in ((norm, (D, 1e-6)), (proj, (D, 256)))]
    norm32.load_state_dict({k: v.float() for k, v in norm.state_dict().items()})
    proj32.load_state_dict({k: v.float() for k, v in proj.state_dict().items()})
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, L, D, generator=g, dtype=torch.float64)
    dout = torch.randn(B, L, 256, generator=g, dtype=torch.float64)
    xd = x.to(DEV).requires_grad_(True)
    proj(norm(ref(xd))).backward(dout.to(DEV))
    xf = x.float().to(DEV).reshape(B * L, D).requires_grad_(True)
    out = proj32(norm32(_apply(ours, xf, B, L)))
    out.backward(dout.float().to(DEV).reshape(B * L, 256))
    worst = {"x": _nrel(xf.grad.reshape(B, L, D), xd.grad)}
    for (n, p), (_, q) in zip(ours.named_parameters(), ref.named_parameters()):
        worst[n] = _nrel(p.grad, q.grad)
    for m32, m64 in ((norm32, norm), (proj32, proj)):
        for (n, p), (_, q) in zip(m32.named_parameters(), m64.named_parameters()):
            worst[n] = _nrel(p.grad, q.grad)
    top = max(worst, key=worst.get)
    print(f"[vit-l chain] worst {top}: {worst[top]:.3e}")
    assert worst[top] <= 1e-3, (top, worst[top])


# ------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------
def _model(prompt_iters=5, seed=7, G=64, K=32):
    from pc_sam.model import build_point_sam

    oracle = torch_ref.build_model("eva02_test_tiny", G, K, prompt_iters=prompt_iters, seed=seed)
    params_ref.perturb(oracle.pc_encoder.transformer, seed, eps=1e-6)
    m = build_point_sam("eva02_test_tiny", G, K, prompt_iters=prompt_iters)
    m.load_state_dict(oracle.state_dict())
    m = m.to(DEV)
    m.requires_grad_(False)
    return m.train()


def _batch(B, M, N, seed=0):
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    rgb = torch.rand(B, N, 3, generator=g)
    gt = torch.zeros(B, M, N, dtype=torch.bool)
    for b in range(B):
        for m in range(M):
            c = xyz[b, torch.randint(0, N, (1,), generator=g)]
            r = 0.4 + 0.4 * torch.rand(1, generator=g)
            gt[b, m] = (xyz[b] - c).norm(dim=-1) < r
    return xyz.to(DEV), rgb.to(DEV), gt.to(DEV)


def _enc_trainable(m, blocks=None):
    enc = m.pc_encoder
    (enc.transformer.blocks if blocks is None else enc.transformer.blocks[blocks]).requires_grad_(True)
    if blocks is None:
        for mod in (enc.transformer.fc_norm, enc.out_proj, enc.patch_proj, enc.pos_embed):
            mod.requires_grad_(True)


def test_whole_step_against_teacher_forced_fp64_oracle(monkeypatch):
    from pc_sam.model.loss import Criterion
    from psam_b200 import train

    m = _model(prompt_iters=5)
    m.mask_decoder.requires_grad_(True)
    _enc_trainable(m)
    xyz, rgb, gt = _batch(2, 4, 4096, seed=1)
    fed, toks = [], []
    real_dec, real_enc = train.run_mask_decoder_train, train.run_pc_encoder_train

    def record_enc(enc, coords, features):
        out, patches = real_enc(enc, coords, features)
        toks.append((patches["embeddings"].detach().clone(), patches["centers"].detach().clone()))
        return out, patches

    def record_dec(md, pc_emb, pc_pe, sparse, dense, aux, multimask_output):
        fed.append((pc_pe, sparse.detach().clone(), dense.detach().clone(), aux))
        return real_dec(md, pc_emb, pc_pe, sparse, dense, aux, multimask_output)

    monkeypatch.setattr(train, "run_pc_encoder_train", record_enc)
    monkeypatch.setattr(train, "run_mask_decoder_train", record_dec)
    torch.manual_seed(123)
    outs = m(xyz, rgb, gt)
    loss, aux_out = Criterion()(outs, gt.flatten(0, 1))
    loss.backward()
    assert len(toks) == 1 and len(fed) == 5
    # oracle: encoder after the tokenizer and decoder in fp64, teacher-forced with the CUDA path's tokenizer outputs,
    # prompts and fed-back masks
    oe = torch_ref.build_model("eva02_test_tiny", 64, 32, prompt_iters=5, seed=7).pc_encoder
    oe.load_state_dict({k: v.detach().cpu() for k, v in m.pc_encoder.state_dict().items()})
    for (n, a), (_, b) in zip(m.pc_encoder.named_modules(), oe.named_modules()):
        if isinstance(a, torch.nn.LayerNorm):
            b.eps = a.eps
    oe = oe.double()
    od = torch_ref.MaskDecoder(256, torch_ref.TwoWayTransformer(2, 256, 8, 2048))
    od.load_state_dict({k: v.detach().cpu() for k, v in m.mask_decoder.state_dict().items()})
    od = od.double()
    emb, centers = (t.double().cpu() for t in toks[0])
    x = oe.patch_proj(emb) + oe.pos_embed(centers)
    for blk in oe.transformer.blocks:
        x = blk(x)
    pc_emb = oe.out_proj(oe.transformer.fc_norm(oe.transformer.norm(x)))
    a = fed[0][3]
    oaux = torch_ref.AuxInputs(coords=None, features=None, centers=None, interp_index=a.interp_index.cpu(),
                               interp_weight=a.interp_weight.double().cpu())
    steps = [(s.double().cpu(), d.double().cpu()) for _, s, d, _ in fed]
    oouts = train_ref.decoder_loop(od, pc_emb, fed[0][0].double().cpu(), steps, oaux)
    wl, _ = train_ref.criterion(oouts, gt.flatten(0, 1).cpu(), hard_iou=[x["iou"].double().cpu() for x in aux_out])
    wl.backward()
    assert abs(float(loss) - float(wl)) <= 1e-4 * abs(float(wl))
    total = float(torch.sqrt(sum(q.grad.double().square().sum() for q in od.parameters())))
    for (n, p), (_, q) in zip(m.mask_decoder.named_parameters(), od.named_parameters()):
        if n.endswith("k_proj.bias"):
            assert float(p.grad.double().norm()) < 1e-6 * total, n
        else:
            assert _nrel(p.grad, q.grad) < 1e-4, n
    checked = 0
    for (n, p), (_, q) in zip(m.pc_encoder.named_parameters(), oe.named_parameters()):
        if p.requires_grad:
            assert _nrel(p.grad, q.grad) < 1e-4, n
            checked += 1
        else:
            assert p.grad is None, n
    assert checked == sum(1 for p in m.pc_encoder.parameters() if p.requires_grad) > 30


def test_partial_unfreezing_and_determinism():
    """Last block only: frozen parameters get no gradient, and the trainable block's gradients are those of a run with
    both blocks trainable on the same saved input and upstream gradient, bit for bit; two autograd.grad calls on one graph
    agree bit for bit."""
    from psam_b200 import engine, train

    B, L = 2, 64
    _, ours, D = _blocks("eva02_test_tiny", 2, seed=3)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B * L, D, generator=g).to(DEV)
    dy = torch.randn(B * L, D, generator=g).to(DEV)
    last = ours[1]
    saved = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
        y = _apply(ours, x.clone().requires_grad_(True), B, L)
    params = list(last.parameters())
    full = torch.autograd.grad(y, params, dy, retain_graph=True)
    again = torch.autograd.grad(y, params, dy)
    assert all(torch.equal(a, b) for a, b in zip(full, again))
    x1 = saved[-1].detach()
    ours.requires_grad_(False)
    last.requires_grad_(True)
    y1 = train.EvaBlockFn.apply(x1, last, engine.block_pack(last, D), B, L, *last.parameters())
    y1.backward(dy)
    assert all(p.grad is None for p in ours[0].parameters())
    assert all(torch.equal(p.grad, f) for p, f in zip(params, full))


def test_blocks_save_only_their_input():
    m = _model()
    m.pc_encoder.transformer.blocks.requires_grad_(True)
    xyz, rgb, gt = _batch(2, 2, 4096)
    outs = m(xyz, rgb, gt)
    nodes, seen, todo = [], set(), [outs[0]["masks"].grad_fn]
    while todo:
        n = todo.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        if "EvaBlockFn" in n.name():
            nodes.append(n)
        todo.extend(f for f, _ in n.next_functions)
    B, L, D = 2, 64, 128
    # one B*L*D input per block, so nothing of B*H*L*L elements (the attention probabilities) is kept
    assert len(nodes) == 2 and all([t.numel() for t in n.saved_tensors] == [B * L * D] for n in nodes)


def test_encoder_only_training_and_eval_after_a_step():
    """Decoder frozen, the last block trainable: non-zero encoder gradients; after an AdamW step the eval path (which
    repacks only the changed block) matches the training forward."""
    from pc_sam.model.loss import Criterion

    m = _model(prompt_iters=3)
    _enc_trainable(m, slice(-1, None))
    xyz, rgb, gt = _batch(1, 2, 4096, seed=2)
    blk = m.pc_encoder.transformer.blocks[-1]
    m.eval()
    with torch.no_grad():
        m.predict_masks(xyz, rgb, xyz[:, :2].reshape(2, 1, 3), torch.ones(2, 1, dtype=torch.bool, device=DEV))  # packs the weights
    frozen_pack = engine_pack(m.pc_encoder.transformer.blocks[0])
    m.train()
    loss, _ = Criterion()(m(xyz, rgb, gt), gt.flatten(0, 1))
    loss.backward()
    assert all(p.grad is not None and p.grad.abs().sum() > 0 for p in blk.parameters())
    assert all(p.grad is None for p in m.mask_decoder.parameters())
    opt = torch.optim.AdamW(blk.parameters(), lr=1e-3, weight_decay=0.1)
    opt.step()
    opt.zero_grad()
    with torch.no_grad():
        outs = m(xyz, rgb, gt)
    m.eval()
    seq_c, seq_l, prev = [], [], 0
    for o in outs:
        seq_c.append(o["prompt_coords"][:, prev:])
        seq_l.append(o["prompt_labels"][:, prev:])
        prev = o["prompt_coords"].shape[1]
    with torch.no_grad():
        ev = m.predict_iterative(xyz, rgb, seq_c, seq_l)
    assert engine_pack(m.pc_encoder.transformer.blocks[0]) is frozen_pack
    for a, b in zip(outs, ev):
        np.testing.assert_allclose(a["masks"].cpu().numpy(), b["masks"].cpu().numpy(), atol=1e-3, rtol=1e-2)
        np.testing.assert_allclose(a["iou_preds"].cpu().numpy(), b["iou_preds"].cpu().numpy(), atol=1e-3, rtol=1e-2)


def engine_pack(blk):
    return blk.__dict__["_psam_packed"][1]


def test_readme_loop_with_the_last_two_blocks_lowers_the_loss():
    from pc_sam.model.loss import Criterion

    torch.manual_seed(0)
    model = _model()
    model.mask_decoder.requires_grad_(True)
    model.pc_encoder.transformer.blocks[-2:].requires_grad_(True)
    model.pc_encoder.transformer.fc_norm.requires_grad_(True)
    model.pc_encoder.out_proj.requires_grad_(True)
    xyz, rgb, gt = _batch(2, 4, 4096, seed=4)
    criterion = Criterion()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=3e-4, weight_decay=0.1)
    hist = []
    for _ in range(50):
        outputs = model(xyz, rgb, gt)
        loss, aux = criterion(outputs, gt.flatten(0, 1))
        loss.backward()
        opt.step()
        opt.zero_grad()
        hist.append((float(loss), float(aux[-1]["iou"].nanmean())))
    print("[finetune encoder] first", hist[0], "last", hist[-1])
    assert hist[-1][0] < hist[0][0]
    assert hist[-1][1] > hist[0][1]
