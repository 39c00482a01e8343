"""Every epilogue form of the split-bf16 GEMM under each tile policy (throughput policy, explicit BN 64 / 128 / 256),
against fp64: multi-wave launches, ragged M / N / K (K tails inside a 32-wide k-block), split-K, batched operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu

POLICIES = {"throughput": (0, 1), "bn64": (64, 0), "bn128": (128, 0), "bn256": (256, 0)}


def _dev():
    return torch.device("cuda:0")


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(_dev())


@pytest.fixture(params=sorted(POLICIES))
def ops(request, monkeypatch):
    from psam_b200 import ops as o

    bn, hint = POLICIES[request.param]
    monkeypatch.setattr(o, "GEMM_TILE_BN", bn)
    monkeypatch.setattr(o, "GEMM_TILE_HINT", hint)
    return o


def _close(got, want, rel):
    err = float((got.double() - want).abs().max())
    assert err < rel * max(1.0, float(want.abs().max())), err


def _operands(ops, M, N, K, seed):
    a, w, b = _rand(M, K, seed=seed), _rand(N, K, seed=seed + 1, scale=K ** -0.5), _rand(N, seed=seed + 2)
    return a, w, b, ops.pack_weight(a), ops.pack_weight(w)


def test_f32_bias_alpha_activation_and_single_pass(ops):
    M, N, K = 4100, 300, 201  # > 1 wave of tiles at every width, tails in M, N and K
    a, w, b, A, W = _operands(ops, M, N, K, 1)
    acc = a.double() @ w.double().t()
    for act, fn in ((ops.ACT_NONE, lambda x: x), (ops.ACT_GELU, torch.nn.functional.gelu), (ops.ACT_RELU, torch.relu)):
        out = torch.empty(M, N, device=_dev())
        ops.gemm(A, W, bias=b, out_f32=out, act=act, alpha=0.5)
        _close(out, fn(0.5 * acc + b.double()), 3e-5)
    out1 = torch.empty(M, N, device=_dev())
    ops.gemm(A, W, bias=b, out_f32=out1, passes=1)
    _close(out1, acc + b.double(), 3e-2)


def test_residual_split_and_row_stats(ops):
    M, N, K = 1000, 512, 330
    a, w, b, A, W = _operands(ops, M, N, K, 11)
    r = _rand(M, N, seed=14)
    want = a.double() @ w.double().t() + b.double() + r.double()
    x, xs, st = r.clone(), ops.Split(M, N, _dev()), torch.zeros(M, 2, device=_dev())
    ops.gemm(A, W, bias=b, out_f32=x, resid=x, out_split=xs, stats_out=st)  # residual in place, both outputs
    _close(x, want, 3e-5)
    _close(xs.float(), want, 3e-5)
    torch.testing.assert_close(st[:, 0].double(), want.sum(-1), atol=2e-3, rtol=1e-5)
    torch.testing.assert_close(st[:, 1].double(), (want * want).sum(-1), atol=2e-3, rtol=2e-5)
    ys = ops.Split(M, N, _dev())
    ops.gemm(A, W, bias=b, out_split=ys, act=ops.ACT_GELU)  # split output alone
    _close(ys.float(), torch.nn.functional.gelu(want - r.double()), 3e-5)


def test_split_k_accumulate(ops):
    M, N, K = 700, 384, 2730
    a, w, b, A, W = _operands(ops, M, N, K, 21)
    r = _rand(M, N, seed=24)
    for sk in (2, 5):
        x = r.clone()
        ops.gemm(A, W, bias=b, out_f32=x, accumulate=True, split_k=sk)
        _close(x, a.double() @ w.double().t() + b.double() + r.double(), 1e-4)


def test_swiglu_both_forms_and_folded_layernorm(ops):
    M, D, H = 900, 288, 320
    xin = _rand(M, D, seed=31) + 2.0  # a row mean that is large against the spread
    gamma, beta = 1.0 + 0.2 * _rand(D, seed=32), 0.1 * _rand(D, seed=33)
    w1, b1 = _rand(2 * H, D, seed=34, scale=D ** -0.5), _rand(2 * H, seed=35, scale=0.1)  # rows: (gate, value) pairs
    eps = 1e-6
    xd = xin.double()
    xn = torch.nn.functional.layer_norm(xd, (D,), gamma.double(), beta.double(), eps)
    z = xn @ w1.double().t() + b1.double()
    h = torch.nn.functional.silu(z[:, 0::2]) * z[:, 1::2]
    X = ops.pack_weight(xin)
    st = torch.stack([xd.sum(-1), (xd * xd).sum(-1)], 1).float().contiguous()
    wg = w1.double() * gamma.double()[None]
    Wf = ops.pack_weight(wg.float())
    c, d = wg.sum(1).float().contiguous(), (w1.double() @ beta.double() + b1.double()).float().contiguous()
    hs, hst = ops.Split(M, H, _dev()), torch.zeros(M, 2, device=_dev())
    ops.gemm(X, Wf, bias=d, out_split=hs, swiglu=True, stats_out=hst, ln_fold=(st, c, D, eps))
    _close(hs.float(), h, 2e-4)
    torch.testing.assert_close(hst[:, 0].double(), h.sum(-1), atol=5e-3, rtol=1e-4)
    # SwiGLU to fp32, no LayerNorm
    zp = xd @ w1.double().t() + b1.double()
    hf = torch.empty(M, H, device=_dev())
    ops.gemm(X, ops.pack_weight(w1), bias=b1, out_f32=hf, swiglu=True)
    _close(hf, torch.nn.functional.silu(zp[:, 0::2]) * zp[:, 1::2], 1e-4)
    # folded LayerNorm with an fp32 output and a residual
    r = _rand(M, 2 * H, seed=36)
    y = r.clone()
    ops.gemm(X, Wf, bias=d, out_f32=y, resid=y, ln_fold=(st, c, D, eps))
    _close(y, z + r.double(), 2e-4)


def test_group_max_and_row_dot(ops):
    G, Kg, N, K = 70, 64, 320, 96
    M = G * Kg
    a, w, b, A, W = _operands(ops, M, N, K, 41)
    full = a.double() @ w.double().t() + b.double()
    y, xs = torch.full((G, N), float("-inf"), device=_dev()), ops.Split(M, N, _dev())
    ops.gemm(A, W, bias=b, out_split=xs, gmax=y, group_rows=Kg)
    _close(y, full.view(G, Kg, N).max(dim=1).values, 1e-4)
    _close(xs.float(), full, 3e-5)
    Z, R, C = 3, 1088, 4
    a, w, b, A, W = _operands(ops, Z * R, 256, 160, 44)
    hyper = _rand(Z, C, 256, seed=47)
    u = torch.nn.functional.gelu(a.double() @ w.double().t() + b.double()).view(Z, R, 256)
    masks = torch.zeros(Z, C, R, device=_dev())
    ops.gemm(A, W, bias=b, act=ops.ACT_GELU, rowdot=(hyper, masks))
    _close(masks, hyper.double() @ u.transpose(1, 2), 2e-4)


def test_batched_operands(ops):
    from psam_b200 import native as nv

    B, H, L, dh = 2, 3, 333, 88
    D = H * dh
    qkv = _rand(B * L, 3 * D, seed=51)
    QKV = ops.Split(B * L, 3 * D, _dev())
    ops.split_f32(qkv, QKV)
    s = torch.empty(B * H * L, L, device=_dev())
    qa = QKV.operand(rows=L, k=dh, col=0, nb1=H, b1_stride=dh, nb2=B, b2_stride=L * QKV.pitch)
    ka = QKV.operand(rows=L, k=dh, col=D, nb1=H, b1_stride=dh, nb2=B, b2_stride=L * QKV.pitch)
    o = ops.GemmOut()
    o.out_f32, o.ldo, o.out_b1, o.out_b2, o.alpha = nv.ptr(s), L, L * L, H * L * L, 1.0
    ops.gemm_raw(qa, ka, o, 3, 1)
    q = qkv[:, :D].reshape(B, L, H, dh).permute(0, 2, 1, 3).double()
    k = qkv[:, D:2 * D].reshape(B, L, H, dh).permute(0, 2, 1, 3).double()
    _close(s, (q @ k.transpose(-1, -2)).reshape(B * H * L, L), 3e-5)
