"""GPU tests of mask_decoder fine-tuning: the loss kernels and the per-point head's backward against the fp64 oracle
(oracle/train_ref.py, pinned to the reference by tests/golden/train.npz), determinism, what the forward saves, a whole
training step against the teacher-forced oracle loop, the weight cache after opt.step(), and the README loop."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import torch_ref, train_ref  # noqa: E402

DEV = torch.device("cuda:0")


def _nrel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).norm() / want.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------
# loss kernels
# ------------------------------------------------------------------------------------------------
def _loss_case(C, N, seed):
    g = torch.Generator().manual_seed(seed)
    Z = 6
    x = torch.randn(Z, C, N, generator=g) * 4
    big = torch.rand(Z, C, N, generator=g) < 0.05
    x[big] = torch.where(torch.rand(int(big.sum()), generator=g) < 0.5, -100.0, 100.0)  # large magnitudes
    x[1] = -torch.rand(C, N, generator=g) - 0.5  # an all-negative prediction
    if C == 3:
        x[2, 2] = x[2, 0]  # a tie between masks 0 and 2
    gt = torch.rand(Z, N, generator=g) < 0.4
    gt[0] = False  # an empty ground truth (with a non-empty prediction)
    return x, gt


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("N", [1, 31, 4097, 32768])
def test_mask_loss_kernels_against_fp64_oracle(C, N):
    from pc_sam.model.loss import Criterion
    from psam_b200.train import mask_loss

    x, gt = _loss_case(C, N, seed=C * 100003 + N)
    xd = x.double().requires_grad_(True)
    want = train_ref.compute_mask_loss(xd, gt)
    up = torch.randn(want.shape, generator=torch.Generator().manual_seed(N), dtype=torch.float64)
    (want * up).sum().backward()
    xc = x.to(DEV).requires_grad_(True)
    got, stats, counts = mask_loss(xc, gt.to(DEV))
    (got * up.float().to(DEV)).sum().backward()
    rel = ((got.detach().double().cpu() - want.detach()).abs() / want.detach().abs().clamp_min(1e-30)).max()
    assert float(rel) < 1e-5, float(rel)
    assert _nrel(xc.grad, xd.grad) < 1e-5
    # hard IoU: integer counts, then one fp32 division - bit for bit the reference's compute_iou on the same logits
    iou = counts[..., 0].float() / counts[..., 1].float()
    want_iou = train_ref.compute_iou(x, gt.unsqueeze(1).expand_as(x))
    assert want_iou.dtype == torch.float32
    assert torch.equal(torch.isnan(iou.cpu()), torch.isnan(want_iou))
    assert torch.equal(torch.nan_to_num(iou.cpu(), nan=-1.0), torch.nan_to_num(want_iou, nan=-1.0))
    # the whole Criterion over two iterations (selection with ties, MSE, means)
    ipd = torch.rand(x.shape[0], C, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    x1 = x[:, :1] * 0.5
    outs_d = [dict(masks=x.double(), iou_preds=ipd), dict(masks=x1.double(), iou_preds=ipd[:, :1])]
    wl, wa = train_ref.criterion(outs_d, gt)
    outs_c = [dict(masks=x.to(DEV), iou_preds=ipd.float().to(DEV)), dict(masks=x1.to(DEV), iou_preds=ipd[:, :1].float().to(DEV))]
    gl, ga = Criterion()(outs_c, gt.to(DEV))
    assert abs(float(gl) - float(wl)) <= 1e-5 * abs(float(wl)) or np.isnan(float(wl))
    for a, b in zip(ga, wa):
        assert torch.equal(torch.nan_to_num(a["iou"].cpu(), nan=-1.0), torch.nan_to_num(b["iou"].float(), nan=-1.0))
        assert torch.equal(a["best_masks"].cpu(), b["best_masks"].float())  # same mask selected (ties: lowest index)


def test_mask_loss_is_deterministic():
    from psam_b200.train import mask_loss

    x, gt = _loss_case(3, 32768, seed=5)
    runs = []
    for _ in range(2):
        xc = x.to(DEV).requires_grad_(True)
        l, s, c = mask_loss(xc, gt.to(DEV))
        l.sum().backward()
        runs.append((l.detach(), s, c, xc.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# the per-point head
# ------------------------------------------------------------------------------------------------
def _decoder(seed=3):
    from pc_sam.model.mask_decoder import MaskDecoder
    from pc_sam.model.transformer import TwoWayTransformer

    md = MaskDecoder(256, TwoWayTransformer(2, 256, 8, 2048))
    return train_ref.fill_params(md, seed).to(DEV)


def _head_case(Z, rep, N, C, G=64, seed=0):
    from pc_sam.model.mask_decoder import AuxInputs
    from psam_b200 import train

    g = torch.Generator().manual_seed(seed)
    B = Z // rep
    coords = (torch.rand(B, N, 3, generator=g) * 2 - 1).to(DEV)
    centers = (torch.rand(B, G, 3, generator=g) * 2 - 1).to(DEV)
    aux = AuxInputs(coords=coords, features=None, centers=centers)
    md = _decoder(seed + 1)
    geo = train.head_geometry(aux, G, rep, md.output_upscaling[1].eps)
    f0 = torch.randn(Z * G, 256, generator=g).to(DEV)
    hyper = (torch.randn(Z, C, 256, generator=g) / 16).to(DEV)
    dm = torch.randn(Z, C, N, generator=g).to(DEV)
    return md, aux, geo, f0, hyper, dm


HEAD_CASES = [(1, 1, 4096, 3), (1, 1, 1000, 1), (16, 8, 1000, 3), (16, 16, 2048, 1), (4, 2, 4097, 3), (16, 8, 32768, 3)]


@pytest.mark.parametrize("Z,rep,N,C", HEAD_CASES)
def test_head_function_against_fp64_autograd(Z, rep, N, C):
    from psam_b200 import engine, train

    md, aux, geo, f0, hyper, dm = _head_case(Z, rep, N, C, seed=Z + N + C)
    up = md.output_upscaling
    f0r, hr = f0.clone().requires_grad_(True), hyper.clone().requires_grad_(True)
    masks = train.MaskHead.apply(f0r, hr, up[1].weight, up[1].bias, up[3].weight, up[3].bias, geo)
    # forward: the eval-mode decoder's per-point code on the same f0 / hyper
    pk = engine._cached(md, engine._PackedDecoder)
    u1 = engine.upscale_ln_gelu(f0, Z, rep, 64, 256, aux.interp_index, aux.interp_weight, N, pk.up1)
    ref = engine.mask_product(u1, pk.up3w, pk.up3b, hyper, Z, C, N)
    if N % 32:
        assert torch.equal(masks.detach(), ref)  # psam_mask_dot: one writer per logit
    else:  # the fused row-dot adds the 32-column chunks of a point with float atomics: equal up to their order
        assert float((masks.detach() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    masks.backward(dm)
    # fp64 autograd of the restated head
    p64 = {n: p.detach().double().cpu().requires_grad_(True) for n, p in
           (("g", up[1].weight), ("b", up[1].bias), ("w3", up[3].weight), ("b3", up[3].bias))}
    f64, h64 = f0.double().cpu().view(Z, 64, 256).requires_grad_(True), hyper.double().cpu().requires_grad_(True)
    want = train_ref.mask_head(f64, h64, p64["g"], p64["b"], up[1].eps, p64["w3"], p64["b3"], aux.interp_index.cpu(),
                               aux.interp_weight.double().cpu(), rep)
    assert _nrel(masks, want) < 1e-4
    want.backward(dm.double().cpu())
    assert _nrel(f0r.grad, f64.grad.view(Z * 64, 256)) < 1e-4
    assert _nrel(hr.grad, h64.grad) < 1e-4
    for n, p in (("g", up[1].weight), ("b", up[1].bias), ("w3", up[3].weight), ("b3", up[3].bias)):
        assert _nrel(p.grad, p64[n].grad) < 1e-4, n


def test_head_backward_is_deterministic_and_honours_needs_input_grad():
    from psam_b200 import train

    md, aux, geo, f0, hyper, dm = _head_case(16, 8, 4096, 3, seed=9)
    up = md.output_upscaling
    args = (f0, hyper, up[1].weight.detach(), up[1].bias.detach(), up[3].weight.detach(), up[3].bias.detach(), geo, dm)
    a = train.head_backward(*args)
    b = train.head_backward(*args)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # partly frozen: only output_upscaling[3].weight and the hyper-network input train
    up.requires_grad_(False)
    up[3].weight.requires_grad_(True)
    hr = hyper.clone().requires_grad_(True)
    m = train.MaskHead.apply(f0, hr, up[1].weight, up[1].bias, up[3].weight, up[3].bias, geo)
    m.backward(dm)
    assert up[1].weight.grad is None and up[3].bias.grad is None
    assert torch.equal(up[3].weight.grad, a[4]) and torch.equal(hr.grad, a[1])


# ------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------
def _model(prompt_iters=5, seed=7, G=64, K=32):
    from pc_sam.model import build_point_sam

    oracle = torch_ref.build_model("eva02_test_tiny", G, K, prompt_iters=prompt_iters, seed=seed)
    m = build_point_sam("eva02_test_tiny", G, K, prompt_iters=prompt_iters)
    m.load_state_dict(oracle.state_dict())
    m = m.to(DEV)
    m.requires_grad_(False)
    m.mask_decoder.requires_grad_(True)
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


def test_training_forward_saves_nothing_per_point_and_feature():
    m = _model()
    xyz, rgb, gt = _batch(1, 2, 4096)
    Z, N, D = 2, 4096, 256
    sizes = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: sizes.append(t.numel()) or t, lambda t: t):
        outs = m(xyz, rgb, gt)
    assert sizes and max(sizes) < Z * N * D, max(sizes)
    assert all(o["masks"].grad_fn is not None and o["iou_preds"].grad_fn is not None for o in outs)


def test_whole_step_against_teacher_forced_fp64_oracle(monkeypatch):
    from pc_sam.model.loss import Criterion
    from psam_b200 import train

    m = _model(prompt_iters=5)
    xyz, rgb, gt = _batch(2, 4, 4096, seed=1)
    fed = []
    real = train.run_mask_decoder_train

    def record(md, pc_emb, pc_pe, sparse, dense, aux, multimask_output):
        fed.append((pc_emb, pc_pe, sparse.detach().clone(), dense.detach().clone(), aux))
        return real(md, pc_emb, pc_pe, sparse, dense, aux, multimask_output)

    monkeypatch.setattr(train, "run_mask_decoder_train", record)
    torch.manual_seed(123)
    outs = m(xyz, rgb, gt)
    loss, aux_out = Criterion()(outs, gt.flatten(0, 1))
    loss.backward()
    # the refinement schedule: the reference's torch.randint draw on the global CPU generator
    torch.manual_seed(123)
    want_refine = {4, torch.randint(1, 5, (1,)).item()}
    got_refine = {i for i in range(1, 5) if outs[i]["prompt_coords"].shape[1] == outs[i - 1]["prompt_coords"].shape[1]}
    assert got_refine == want_refine
    # oracle: the same decoder in fp64, teacher-forced with the CUDA path's encoder outputs, prompts and fed-back masks
    od = torch_ref.MaskDecoder(256, torch_ref.TwoWayTransformer(2, 256, 8, 2048))
    od.load_state_dict({k: v.detach().cpu() for k, v in m.mask_decoder.state_dict().items()})
    od = od.double()
    a = fed[0][4]
    oaux = torch_ref.AuxInputs(coords=None, features=None, centers=None, interp_index=a.interp_index.cpu(),
                               interp_weight=a.interp_weight.double().cpu())
    steps = [(s.double().cpu(), d.double().cpu()) for _, _, s, d, _ in fed]
    oouts = train_ref.decoder_loop(od, fed[0][0].double().cpu(), fed[0][1].double().cpu(), steps, oaux)
    wl, _ = train_ref.criterion(oouts, gt.flatten(0, 1).cpu(), hard_iou=[x["iou"].double().cpu() for x in aux_out])
    wl.backward()
    assert abs(float(loss) - float(wl)) <= 1e-4 * abs(float(wl))
    total = float(torch.sqrt(sum(q.grad.double().square().sum() for q in od.parameters())))
    for (n, p), (_, q) in zip(m.mask_decoder.named_parameters(), od.named_parameters()):
        if n.endswith("k_proj.bias"):
            # a key bias shifts every score of a query by the same amount, which the softmax ignores: the gradient is zero in
            # exact arithmetic, so only round-off remains, measured against the whole gradient
            assert float(p.grad.double().norm()) < 1e-6 * total, n
        else:
            assert _nrel(p.grad, q.grad) < 1e-4, n


def test_eval_after_optimizer_step_uses_the_new_weights():
    from pc_sam.model.loss import Criterion

    m = _model(prompt_iters=3)
    xyz, rgb, gt = _batch(1, 2, 4096, seed=2)
    opt = torch.optim.AdamW(m.mask_decoder.parameters(), lr=1e-3, weight_decay=0.1)
    m.eval()
    with torch.no_grad():
        m.predict_masks(xyz, rgb, xyz[:, :2].reshape(2, 1, 3), torch.ones(2, 1, dtype=torch.bool, device=DEV))  # packs the weights
    m.train()
    loss, _ = Criterion()(m(xyz, rgb, gt), gt.flatten(0, 1))
    loss.backward()
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
    for a, b in zip(outs, ev):
        np.testing.assert_allclose(a["masks"].cpu().numpy(), b["masks"].cpu().numpy(), atol=1e-3, rtol=1e-2)
        np.testing.assert_allclose(a["iou_preds"].cpu().numpy(), b["iou_preds"].cpu().numpy(), atol=1e-3, rtol=1e-2)


def test_readme_loop_lowers_the_loss():
    from pc_sam.model.loss import Criterion

    torch.manual_seed(0)
    model = _model()
    xyz, rgb, gt = _batch(2, 4, 4096, seed=4)
    criterion = Criterion()
    opt = torch.optim.AdamW(model.mask_decoder.parameters(), lr=3e-4, weight_decay=0.1)
    hist = []
    for _ in range(50):
        outputs = model(xyz, rgb, gt)
        loss, aux = criterion(outputs, gt.flatten(0, 1))
        loss.backward()
        opt.step()
        opt.zero_grad()
        hist.append((float(loss), float(aux[-1]["iou"].nanmean())))
    print("[finetune] first", hist[0], "last", hist[-1])
    assert hist[-1][0] < hist[0][0]
    assert hist[-1][1] > hist[0][1]
