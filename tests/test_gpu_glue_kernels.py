"""The fp32 glue kernels (csrc/elementwise.cu, plus the GEMM's fused group max) against plain fp64 restatements, through
the C ABI, on every launch path of their host functions.

Two kinds of check:
  * integer-valued inputs (|x|, |w| <= 8, sums below 2^24), where every partial sum is exact in fp32 whatever the order,
    so the kernel must equal the fp64 result bit for bit: a dropped K tail, a wrong stride or batch offset fails at once;
  * random inputs against an elementwise bound of the form c * sqrt(K) * 2^-24 * (|x| @ |w|^T) for a reduction of length
    K, tight enough that a single wrong term fails.  Each case prints its largest error and its error / bound ratio.
Every case names the template instantiation it reaches; test_routing_guard checks those names under torch.profiler, so
the coverage stays true if a dispatch threshold moves."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24       # fp32 unit roundoff
SPLIT = 2.0 ** -16   # split-bf16: |hi + lo - y| <= 2^-17 |y|, with a factor 2 of slack
GELU_ABS = 1e-6      # the kernels' GELU uses the A&S 7.1.26 erf (|error| <= 1.5e-7): absolute error about 5e-7
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2


def _ops():
    from psam_b200 import ops

    return ops


def _nv():
    from psam_b200 import native as nv

    return nv


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, lo, hi, seed):
    """Integer-valued fp32 on the device, uniform in [lo, hi]."""
    return torch.randint(lo, hi + 1, shape, generator=_gen(seed)).float().to(_dev())


def _randn(shape, seed, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=_gen(seed)) * scale + shift).to(_dev())


def _nan(shape):
    return torch.full(shape, float("nan"), device=_dev())


def _nan_split(rows, cols, pitch=None):
    s = _ops().Split(rows, cols, _dev(), pitch=pitch)
    s.t.fill_(float("nan"))
    return s


def _act64(y, act):
    if act == ACT_GELU:
        return torch.nn.functional.gelu(y)
    if act == ACT_RELU:
        return torch.relu(y)
    return y


def _check_bound(name, got, want, bound):
    """|got - want| <= bound elementwise (want and bound fp64); prints the largest error and error / bound."""
    err = (got.double() - want).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    print(f"[glue] {name}: max|err| {float(err.max()):.3e}, max err/bound {ratio:.3f}")
    assert ratio <= 1.0, f"{name}: error {ratio:.2f}x its bound"


def _split_of(y):
    """The split-bf16 planes the kernels write for fp32 y: hi = bf16_rn(y), lo = bf16_rn(y - hi)."""
    hi = y.to(torch.bfloat16)
    return hi, (y - hi.float()).to(torch.bfloat16)


def _assert_split_is(sp, y, name):
    hi, lo = _split_of(y)
    D = y.shape[-1]
    assert torch.equal(sp.t[0, :, :D], hi) and torch.equal(sp.t[1, :, :D], lo), f"{name}: split planes != split(y)"


def _assert_pad_zero(sp, D, name):
    assert bool((sp.t[:, :, D:] == 0).all()), f"{name}: columns {D}..{sp.pitch} of the split output are not zero-filled"


def _ln64(x, g, b, eps):
    """fp64 LayerNorm; returns (y, rstd)."""
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    return (x - mean) * rstd * g + b, rstd


def _ln_bound(inmag, g, b, y_pre, rstd, act, c=4.0):
    """Bound of a two-pass fp32 LayerNorm of D-wide rows whose inputs have magnitude inmag [.., D]: the mean and variance
    sums carry c sqrt(D) u of the largest input (that is what a mean >> spread costs after normalisation), the affine
    map a few roundings; GELU has slope <= 1.13 plus its own absolute error."""
    D = inmag.shape[-1]
    bound = c * U * math.sqrt(D) * g.abs() * rstd * inmag.amax(-1, keepdim=True) + c * U * (y_pre.abs() + b.abs())
    return 1.2 * bound + GELU_ABS if act == ACT_GELU else bound


# ------------------------------------------------------------------------------------------------
# dispatch of the host functions, restated (test_routing_guard checks these against the kernels that run)
# ------------------------------------------------------------------------------------------------
def _linear_kernel(M, K, vec):
    if M <= 8 and vec and K >= 512:
        return f"linear_gemv_ksplit_kernel<{1 if M <= 1 else 4 if M <= 4 else 8}>"
    if M <= 16:
        mr = 1 if M <= 1 else 4 if M <= 4 else 8 if M <= 8 else 16
        return f"linear_gemv_kernel<{mr}, {'true' if vec else 'false'}>"
    return "linear_f32_v4_kernel" if vec else "linear_f32_kernel"


def _attn_kernel(dh, items, Lk):
    return f"attention_small_kernel<{dh}, {4 if items <= 512 and Lk >= 128 else 1}>"


def _ln_kernel(D, rows, policy, vec):
    block = D > 1024 or (D >= 256 and rows <= 8192 and policy != 1)
    pick = lambda n, steps: next(s for s in steps if n <= s or s == steps[-1])
    if block and vec:
        return f"layernorm_block_v4_kernel<{pick(-(-D // 1024), (1, 2, 4))}>"
    if vec:
        return f"layernorm_warp_v4_kernel<{pick(-(-D // 128), (1, 2, 4, 8))}>"
    if block:
        return f"layernorm_block_kernel<{pick(-(-D // 256), (1, 2, 4, 8, 16))}>"
    return f"layernorm_warp_kernel<{pick(-(-D // 32), (4, 8, 16, 32))}>"


def _id(kernel, **kw):
    return kernel.replace(", ", ",") + "-" + "-".join(f"{k}{v}" for k, v in kw.items())


# ------------------------------------------------------------------------------------------------
# psam_linear_f32
# ------------------------------------------------------------------------------------------------
def _linear_ref(x, w, b, x2, r, act):
    xx = x.double() + (x2.double() if x2 is not None else 0.0)
    y = xx @ w.double().t()
    if b is not None:
        y = y + b.double()
    y = _act64(y, act)
    return y + r.double() if r is not None else y


_LIN_M = [1, 2, 4, 5, 8, 9, 16, 17, 384, 1152]
_LIN_K = [3, 4, 256, 510, 511, 512, 516, 2048]
_LIN_N = [1, 4, 7, 8, 9, 65, 130, 2048]
_LIN_GRID = [(i, j, M, K, _LIN_N[(i + j) % len(_LIN_N)]) for i, M in enumerate(_LIN_M) for j, K in enumerate(_LIN_K)]


@pytest.mark.parametrize("i,j,M,K,N", _LIN_GRID, ids=[_id(_linear_kernel(M, K, K % 4 == 0), M=M, K=K, N=N)
                                                       for (i, j, M, K, N) in _LIN_GRID])
def test_linear_exact(i, j, M, K, N):
    """Every (M, K) of the dispatch grid on integer inputs: bias always, x2 / residual / ReLU in turn; bit for bit."""
    ops = _ops()
    s = 100 * i + j
    x, w, b = _ints((M, K), -8, 8, s), _ints((N, K), -8, 8, s + 1), _ints((N,), -64, 64, s + 2)
    x2 = _ints((M, K), -8, 8, s + 3) if (i + j) % 2 else None
    r = _ints((M, N), -64, 64, s + 4) if (i + j) % 3 == 0 else None
    act = ACT_RELU if j % 2 else ACT_NONE
    y = ops.linear_f32(x, w, b, x2=x2, r=r, act=act)
    want = _linear_ref(x, w, b, x2, r, act).float()
    assert torch.equal(y, want), f"{int((y != want).sum())} of {y.numel()} outputs differ"


_LIN_RAND = [(1, 512, 130), (4, 2048, 65), (5, 2048, 2048), (8, 516, 9), (1, 256, 130), (1, 3, 1), (4, 510, 7), (8, 256, 65),
             (16, 2048, 130), (9, 511, 8), (17, 256, 65), (384, 2048, 130), (1152, 516, 65), (17, 511, 9), (384, 3, 2048)]


@pytest.mark.parametrize("act", [ACT_NONE, ACT_GELU])
@pytest.mark.parametrize("M,K,N", _LIN_RAND, ids=[_id(_linear_kernel(M, K, K % 4 == 0), M=M, K=K, N=N) for (M, K, N) in _LIN_RAND])
def test_linear_random(M, K, N, act):
    """Random inputs with x2, bias and residual: elementwise bound 4 sqrt(K) u (|x| + |x2|) @ |w|^T."""
    ops = _ops()
    x, x2, w = _randn((M, K), 1), _randn((M, K), 2), _randn((N, K), 3, K ** -0.5)
    b, r = _randn((N,), 4), _randn((M, N), 5)
    y = ops.linear_f32(x, w, b, x2=x2, r=r, act=act)
    want = _linear_ref(x, w, b, x2, r, act)
    scale = (x.double().abs() + x2.double().abs()) @ w.double().abs().t() + b.double().abs()
    bound = 4 * math.sqrt(K) * U * scale * (1.2 if act == ACT_GELU else 1.0) + 2 * U * (want.abs() + r.double().abs())
    if act == ACT_GELU:
        bound = bound + GELU_ABS
    _check_bound(f"linear {_linear_kernel(M, K, K % 4 == 0)} M={M} K={K} N={N} act={act}", y, want, bound)


_LIN_SCALAR = [("odd_ldx", 4), ("odd_ldx", 384), ("odd_x_off", 8), ("odd_x_off", 1152), ("x_z_not_mult_4", 4),
               ("x_z_not_mult_4", 384)]


@pytest.mark.parametrize("form,M", _LIN_SCALAR, ids=[_id(_linear_kernel(M, 512, False), form=f, M=M) for (f, M) in _LIN_SCALAR])
def test_linear_scalar_forms(form, M):
    """K = 512 would take a float4 path; an odd ldx, an odd x_off or a batch stride x_z % 4 != 0 must force the scalar
    one and still be exact."""
    ops = _ops()
    K, N = 512, 65
    w, b = _ints((2, N, K), -8, 8, 11), _ints((2, N), -64, 64, 12)
    if form == "odd_ldx":
        xb, x2b = _ints((M, K + 1), -8, 8, 13), _ints((M, K + 1), -8, 8, 14)
        y = ops.linear_f32(xb, w[0], b[0], x2=x2b, M=M, K=K, ldx=K + 1)
        want = _linear_ref(xb[:, :K], w[0], b[0], x2b[:, :K], None, ACT_NONE)
    elif form == "odd_x_off":
        xb = _ints((M * K + 1,), -8, 8, 15)
        y = ops.linear_f32(xb, w[0], b[0], M=M, K=K, ldx=K, x_off=1)
        want = _linear_ref(xb[1:].view(M, K), w[0], b[0], None, None, ACT_NONE)
    else:
        xz = M * K + 1
        xb = _ints((xz + M * K,), -8, 8, 16)
        y = torch.empty(2 * M, N, device=_dev())
        ops.linear_f32(xb, w, b, out=y, M=M, K=K, ldx=K, Z=2, x_z=xz, w_z=N * K, b_z=N, y_z=M * N)
        want = torch.cat([_linear_ref(xb[z * xz:z * xz + M * K].view(M, K), w[z], b[z], None, None, ACT_NONE) for z in range(2)])
    assert torch.equal(y, want.float())


_HYPER = [(1, 256, 6, 0, 256, False), (8, 256, 7, 1, 32, True), (64, 256, 6, 1, 256, False), (5, 512, 6, 1, 512, True),
          (1, 512, 7, 0, 64, False)]


@pytest.mark.parametrize("Zp,D,T,i0,Do,with_x2", _HYPER,
                         ids=[_id(_linear_kernel(Zp, D, True), Zp=Zp, D=D, T=T, i0=i0, Do=Do) for (Zp, D, T, i0, Do, _) in _HYPER])
def test_linear_hypernetwork_batched(Zp, D, T, i0, Do, with_x2):
    """The decoder's hyper-network form: Z = C = 3 mask tokens batched through x_z / w_z / b_z / y_z, the tokens read in
    place from the [Zp*T, D] token stream (ldx = T*D, x_off = (1 + i0)*D), the outputs interleaved (ldy = C*Do)."""
    ops = _ops()
    C = 3
    hs = _ints((Zp * T, D), -8, 8, 21)
    x2 = _ints((Zp * T, D), -8, 8, 22) if with_x2 else None
    w, b = _ints((4, Do, D), -8, 8, 23), _ints((4, Do), -64, 64, 24)
    y = _nan((Zp, C, Do))
    x2_in = x2.view(-1)[(1 + i0) * D:] if with_x2 else None  # x_off moves x only; x2 shares x's strides from its own start
    ops.linear_f32(hs, w[i0:i0 + C], b[i0:i0 + C], x2=x2_in, act=ACT_RELU, out=y, M=Zp, K=D, ldx=T * D, Z=C, x_z=D,
                   x2_z=D if with_x2 else 0, w_z=Do * D, b_z=Do, y_z=Do, ldy=C * Do, x_off=(1 + i0) * D)
    tok = lambda t: t.view(Zp, T, D)
    want = torch.stack([_linear_ref(tok(hs)[:, 1 + i0 + c], w[i0 + c], b[i0 + c], tok(x2)[:, 1 + i0 + c] if with_x2 else None,
                                    None, ACT_RELU) for c in range(C)], 1)
    assert torch.equal(y, want.float())


# ------------------------------------------------------------------------------------------------
# psam_attention_f32
# ------------------------------------------------------------------------------------------------
def _heads(t, L, Z, H, dh, off):
    return t[:, off:off + H * dh].double().reshape(Z, L, H, dh).transpose(1, 2)  # [Z, H, L, dh]


def _unheads(t, Z, L, H, dh):
    return t.transpose(1, 2).reshape(Z * L, H * dh)


def _attn_check(name, o, q, k, v, Z, Lq, Lk, H, dh, q_off=0, k_off=0, v_off=0):
    """fp64 attention and the bound: score errors (a dh-term dot product, then the scale) move the probabilities by twice
    the largest of them, __expf adds a few u relative to the exponent's size, the sums over keys sqrt(Lk) u; all relative
    to sum_j p_j |v_j|."""
    qq, kk, vv = _heads(q, Lq, Z, H, dh, q_off), _heads(k, Lk, Z, H, dh, k_off), _heads(v, Lk, Z, H, dh, v_off)
    s = qq @ kk.transpose(-1, -2) / math.sqrt(dh)
    p = torch.softmax(s, -1)
    want = _unheads(p @ vv, Z, Lq, H, dh)
    sabs = qq.abs() @ kk.abs().transpose(-1, -2) / math.sqrt(dh)
    ds = (4 * math.sqrt(dh) * U * sabs + U * s.abs()).amax(-1, keepdim=True)
    spread = s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True)
    rel = 2 * ds + 4 * U * (2 + spread) + 4 * math.sqrt(Lk) * U
    bound = _unheads((rel * (p @ vv.abs())).expand(-1, -1, -1, dh), Z, Lq, H, dh) + 1e-30
    _check_bound(name, o, want, bound)


def _one_hot_qk(Z, Lq, Lk, H, dh, seed):
    """q / k whose scores peak at one key t(z, i, h) per query, every other key at least 128 lower after the 1/sqrt(dh)
    scale (score = S (t j - j^2 / 2)), so __expf of every other key underflows to 0 and the output must be exactly
    v[z, t, h, :]."""
    g = _gen(seed)
    t = torch.randint(0, Lk, (Z, Lq, H), generator=g)
    S = 4096.0
    q = torch.zeros(Z, Lq, H, dh)
    q[..., 0], q[..., 1] = S * t.float(), S
    j = torch.arange(Lk, dtype=torch.float32)
    k = torch.randn(Z, Lk, H, dh, generator=g)
    k[..., 0], k[..., 1] = j[None, :, None], -(j * j / 2)[None, :, None]
    return q.reshape(Z * Lq, H * dh).to(_dev()), k.reshape(Z * Lk, H * dh).to(_dev()), t.to(_dev())


def _one_hot_want(v, t, Z, Lk, H, dh, v_off=0):
    vv = v[:, v_off:v_off + H * dh].reshape(Z, Lk, H, dh)
    Lq = t.shape[1]
    idx = t[..., None].expand(Z, Lq, H, dh)
    return torch.gather(vv, 1, idx).reshape(Z * Lq, H * dh)


def _attn_limit(dh):
    """The largest Lk the 200 KB shared-memory check of psam_attention_f32 admits: 4 warps x (Lk + dh) scores and queries
    plus 4 x (dh + 2) combine slots, in floats."""
    return (200 * 1024 // 4 - 4 * (dh + 2)) // 4 - dh


_ATT = []
for _dh in (8, 16, 32, 64):
    _ATT += [(_dh, 2, 4, 64, 128), (_dh, 3, 3, 57, 128), (_dh, 2, 4, 64, 127), (_dh, 3, 3, 57, 127)]  # items 512 / 513
for _Z in (1, 64, 192):
    for _T in (6, 7):
        _ATT += [(16, _Z, 8, _T, 512), (16, _Z, 8, 512, _T)]  # decoder: tokens -> 512 patches, patches -> tokens
_ATT += [(64, 1, 1, 4, _attn_limit(64)), (16, 1, 2, 300, _attn_limit(16))]


@pytest.mark.parametrize("dh,Z,H,Lq,Lk", _ATT, ids=[_id(_attn_kernel(dh, Z * H * Lq, Lk), Z=Z, H=H, Lq=Lq, Lk=Lk) for (dh, Z, H, Lq, Lk) in _ATT])
def test_attention(dh, Z, H, Lq, Lk):
    """Random q / k / v against fp64 with a stated bound, then one-hot scores (logit spreads >= 128) that must return the
    selected V rows exactly."""
    ops = _ops()
    q, k, v = _randn((Z * Lq, H * dh), 31), _randn((Z * Lk, H * dh), 32), _randn((Z * Lk, H * dh), 33)
    o = ops.attention_f32(q, k, v, Z, Lq, Lk, H, dh)
    _attn_check(f"attention {_attn_kernel(dh, Z * H * Lq, Lk)} Z={Z} H={H} Lq={Lq} Lk={Lk}", o, q, k, v, Z, Lq, Lk, H, dh)
    if Lk <= 1024:
        q1, k1, t = _one_hot_qk(Z, Lq, Lk, H, dh, 34)
        o1 = ops.attention_f32(q1, k1, v, Z, Lq, Lk, H, dh)
        assert torch.equal(o1, _one_hot_want(v, t, Z, Lk, H, dh))


def test_attention_fused_kq_windows():
    """The decoder's fused [k of tokens->patches | q of patches->tokens] buffer: k_off = 0 and q_off = nk on a row stride
    wider than H*dh, in both directions, random and one-hot."""
    ops = _ops()
    Z, G, T, H, dh = 4, 512, 7, 8, 16
    nk = H * dh
    kq = _randn((Z * G, 2 * nk + 8), 41)
    qt, vv = _randn((Z * T, nk), 42), _randn((Z * G, nk), 43)
    kt, vt = _randn((Z * T, nk), 44), _randn((Z * T, nk), 45)
    o = ops.attention_f32(qt, kq, vv, Z, T, G, H, dh)
    _attn_check("attention fused kq, tokens -> patches", o, qt, kq, vv, Z, T, G, H, dh)
    o2 = ops.attention_f32(kq, kt, vt, Z, G, T, H, dh, q_off=nk)
    _attn_check("attention fused kq, patches -> tokens", o2, kq, kt, vt, Z, G, T, H, dh, q_off=nk)
    q1, k1, t1 = _one_hot_qk(Z, T, G, H, dh, 46)   # tokens -> patches: keys in columns [0, nk)
    q2, k2, t2 = _one_hot_qk(Z, G, T, H, dh, 47)   # patches -> tokens: queries in columns [nk, 2 nk)
    kq1 = torch.cat([k1, q2, _randn((Z * G, 8), 48)], 1).contiguous()
    assert torch.equal(ops.attention_f32(q1, kq1, vv, Z, T, G, H, dh), _one_hot_want(vv, t1, Z, G, H, dh))
    assert torch.equal(ops.attention_f32(kq1, k2, vt, Z, G, T, H, dh, q_off=nk), _one_hot_want(vt, t2, Z, T, H, dh))


@pytest.mark.parametrize("dh,Lq", [(64, 4), (16, 300)])
def test_attention_shared_memory_limit_refused(dh, Lq):
    """One key beyond the largest admitted Lk (test_attention runs that one) is refused with PSAM_ERR_UNSUPPORTED."""
    ops = _ops()
    Lk = _attn_limit(dh) + 1
    q, k = _randn((Lq, dh), 51), _randn((Lk, dh), 52)
    with pytest.raises(RuntimeError, match="unsupported configuration"):
        ops.attention_f32(q, k, k, 1, Lq, Lk, 1, dh)


# ------------------------------------------------------------------------------------------------
# psam_layernorm_f32
# ------------------------------------------------------------------------------------------------
_LN = [(96, 8193, 0, ""), (97, 1, 0, ""), (128, 8192, 1, ""), (255, 8193, 0, ""), (256, 1, 0, ""), (256, 8192, 0, ""),
       (256, 8193, 0, ""), (256, 1, 1, ""), (384, 64, 1, ""), (511, 64, 0, ""), (511, 64, 1, ""), (256, 64, 0, "odd_ldx"),
       (1000, 1, 0, ""), (1000, 8193, 0, ""), (1023, 64, 1, ""), (1023, 64, 0, ""), (1024, 8192, 0, ""), (1024, 64, 1, ""),
       (1025, 1, 0, ""), (2048, 64, 0, ""), (2730, 64, 0, ""), (4096, 1, 0, ""), (4096, 8193, 1, ""), (128, 64, 0, "odd_ldx")]


def _ln_case_kernel(D, rows, policy, form):
    return _ln_kernel(D, rows, policy, D % 4 == 0 and form != "odd_ldx")


@pytest.mark.parametrize("i", range(len(_LN)), ids=[_id(_ln_case_kernel(*c), D=c[0], rows=c[1], policy=c[2]) + (f"-{c[3]}" if c[3] else "")
                                                    for c in _LN])
def test_layernorm(i, monkeypatch):
    """Every instantiation through D, rows and policy; residual, group bias, GELU and a mean >> spread (+300) in turn;
    fp32 output against fp64, the split output equal to split(fp32 output), pad columns zero up to the pitch."""
    ops = _ops()
    D, rows, policy, form = _LN[i]
    monkeypatch.setattr(ops, "GEMM_TILE_HINT", policy)
    ldx = D + 1 if form == "odd_ldx" else D
    shift = 300.0 if i % 5 == 2 else 0.0
    xb = _randn((rows, ldx), 61, shift=shift)
    x = xb[:, :D]
    r = _randn((rows, D), 62) if i % 2 == 0 else None
    group_rows = 7
    gb = _randn((-(-rows // group_rows), D), 63) if i % 3 == 0 else None
    act = ACT_GELU if i % 4 == 1 else ACT_NONE
    g, b = _randn((D,), 64, 0.5, 1.0), _randn((D,), 65, 0.2)
    eps = 1e-6
    y = _nan((rows, D))
    sp = _nan_split(rows, D, pitch=(D + 63) // 64 * 64 + (64 if i % 2 else 0))
    ops.layernorm(xb, g, b, eps, rows=rows, D=D, ldx=ldx, r=r, gbias=gb, group_rows=group_rows if gb is not None else 0,
                  act=act, out_f32=y, out_split=sp)
    inp = x.double()
    inmag = x.double().abs()
    if r is not None:
        inp, inmag = inp + r.double(), inmag + r.double().abs()
    if gb is not None:
        gbr = gb.double().repeat_interleave(group_rows, 0)[:rows]
        inp, inmag = inp + gbr, inmag + gbr.abs()
    y_pre, rstd = _ln64(inp, g.double(), b.double(), eps)
    want = _act64(y_pre, act)
    _check_bound(f"layernorm {_ln_case_kernel(D, rows, policy, form)} D={D} rows={rows} policy={policy} shift={shift}", y, want,
                 _ln_bound(inmag, g.double(), b.double(), y_pre, rstd, act))
    _assert_split_is(sp, y, "layernorm")
    _assert_pad_zero(sp, D, "layernorm")


def test_layernorm_padded_swiglu_mlp_form():
    """padded = 1 as the SwiGLU MLP uses it: D = 2730 on rows of pitch 2752 whose pad columns are zero, gamma / beta zero
    padded; the float4 path (layernorm_block_v4_kernel<4>) writes the outputs up to roundup4(D) and zeros the rest."""
    ops = _ops()
    rows, D, P = 64, 2730, 2752
    x = _randn((rows, P), 71)
    x[:, D:] = 0
    g, b = torch.zeros(P, device=_dev()), torch.zeros(P, device=_dev())
    g[:D], b[:D] = _randn((D,), 72, 0.5, 1.0), _randn((D,), 73, 0.2)
    y = _nan((rows, P))
    sp = _nan_split(rows, D, pitch=P)
    ops.layernorm(x, g, b, 1e-6, D=D, padded=True, out_f32=y, out_split=sp)
    y_pre, rstd = _ln64(x[:, :D].double(), g[:D].double(), b[:D].double(), 1e-6)
    _check_bound("layernorm padded D=2730 pitch=2752", y[:, :D], y_pre,
                 _ln_bound(x[:, :D].double().abs(), g[:D].double(), b[:D].double(), y_pre, rstd, ACT_NONE))
    assert bool((y[:, D:D + 2] == 0).all())
    _assert_split_is(sp, y[:, :D].contiguous(), "layernorm padded")
    _assert_pad_zero(sp, D, "layernorm padded")


_LN_POST = [(256, 0), (256, 1), (258, 0), (258, 1)]


@pytest.mark.parametrize("D,policy", _LN_POST, ids=[_id(_ln_kernel(D, 1536, p, D % 4 == 0), D=D, policy=p) for (D, p) in _LN_POST])
def test_layernorm_decoder_keys_post_add(D, policy, monkeypatch):
    """The decoder's keys update: y = LN(keys + upd) as fp32 and split-bf16, and a second split output split(y + pe)."""
    ops = _ops()
    monkeypatch.setattr(ops, "GEMM_TILE_HINT", policy)
    rows = 3 * 512
    keys, upd, pe = _randn((rows, D), 81), _randn((rows, D), 82), _randn((rows, D), 83)
    g, b = _randn((D,), 84, 0.5, 1.0), _randn((D,), 85, 0.2)
    y, s1, s2 = _nan((rows, D)), _nan_split(rows, D), _nan_split(rows, D)
    ops.layernorm(keys, g, b, 1e-5, r=upd, out_f32=y, out_split=s1, post_add=pe, out_split2=s2)
    inp = keys.double() + upd.double()
    y_pre, rstd = _ln64(inp, g.double(), b.double(), 1e-5)
    _check_bound(f"layernorm post_add D={D} policy={policy}", y, y_pre,
                 _ln_bound(keys.double().abs() + upd.double().abs(), g.double(), b.double(), y_pre, rstd, ACT_NONE))
    _assert_split_is(s1, y, "layernorm keys")
    _assert_split_is(s2, y + pe, "layernorm keys + pe")


def test_layernorm_refuses_wide_rows():
    ops = _ops()
    x = _randn((2, 4097), 91)
    g = torch.ones(4097, device=_dev())
    with pytest.raises(RuntimeError, match="unsupported configuration"):
        ops.layernorm(x, g, g, 1e-6, out_f32=torch.empty_like(x))


# ------------------------------------------------------------------------------------------------
# psam_swiglu_ln, psam_small_in_linear, psam_group_max, psam_softmax_split
# ------------------------------------------------------------------------------------------------
def _swiglu_vpt(H):
    v = -(-H // 256)
    return next(s for s in (2, 4, 8, 12, 16, 24, 32) if v <= s)


@pytest.mark.parametrize("H", [344, 683, 1500, 2730, 3000, 4000, 6000, 8192], ids=lambda H: f"swiglu_ln_kernel<{_swiglu_vpt(H)}>-H{H}")
def test_swiglu_ln(H):
    """LN(silu(g) * x) with g and x in one [rows, 2 Hp + 8] buffer (x at column Hp), split output padded to Hp + 64."""
    ops = _ops()
    rows = 48
    Hp = (H + 63) // 64 * 64
    gx = _randn((rows, 2 * Hp + 8), 101)
    g, b = _randn((H,), 102, 0.5, 1.0), _randn((H,), 103, 0.2)
    out = _nan_split(rows, H, pitch=Hp + 64)
    ops.swiglu_ln(gx, H, Hp, g, b, 1e-6, out)
    h = torch.nn.functional.silu(gx[:, :H].double()) * gx[:, Hp:Hp + H].double()
    y, rstd = _ln64(h, g.double(), b.double(), 1e-6)
    bound = _ln_bound(h.abs(), g.double(), b.double(), y, rstd, ACT_NONE, c=8.0) + SPLIT * y.abs()
    _check_bound(f"swiglu_ln H={H}", out.float(), y, bound)
    _assert_pad_zero(out, H, "swiglu_ln")


def test_swiglu_ln_refuses_wide_rows():
    ops = _ops()
    H = 8193
    with pytest.raises(RuntimeError, match="unsupported configuration"):
        ops.swiglu_ln(_randn((2, 2 * H), 104), H, H, torch.ones(H, device=_dev()), torch.zeros(H, device=_dev()), 1e-6,
                      ops.Split(2, H, _dev()))


@pytest.mark.parametrize("ln", [False, True], ids=["plain", "ln"])
@pytest.mark.parametrize("Cin", [1, 3, 6, 16])
@pytest.mark.parametrize("Cout", [32, 64, 128, 256, 512], ids=lambda c: f"small_in_linear_kernel<{c // 32}>-Cout{c}")
def test_small_in_linear(Cout, Cin, ln):
    """y = act(LN?(x W^T + b)): GELU after the LayerNorm, ReLU without it; 777 rows (a ragged last CTA)."""
    ops = _ops()
    rows = 777
    x, W, b = _randn((rows, Cin), 111), _randn((Cout, Cin), 112), _randn((Cout,), 113)
    g, be = _randn((Cout,), 114, 0.5, 1.0), _randn((Cout,), 115, 0.2)
    act = ACT_GELU if ln else ACT_RELU
    out = _nan_split(rows, Cout)
    ops.small_in_linear(x, W, b, g if ln else None, be if ln else None, 1e-5, ln, act, out)
    o = x.double() @ W.double().t() + b.double()
    mag = x.double().abs() @ W.double().abs().t() + b.double().abs()
    if ln:
        y_pre, rstd = _ln64(o, g.double(), be.double(), 1e-5)
        want = _act64(y_pre, act)
        bound = _ln_bound(mag, g.double(), be.double(), y_pre, rstd, act)
    else:
        want = _act64(o, act)
        bound = 4 * math.sqrt(Cin) * U * mag
    _check_bound(f"small_in_linear Cout={Cout} Cin={Cin} ln={ln}", out.float(), want, bound + SPLIT * want.abs())


def test_small_in_linear_refuses_cout_96():
    ops = _ops()
    with pytest.raises(RuntimeError, match="unsupported configuration"):
        ops.small_in_linear(_randn((8, 3), 116), _randn((96, 3), 117), None, None, None, 0.0, False, ACT_NONE,
                            ops.Split(8, 96, _dev()))


@pytest.mark.parametrize("groups,K,D", [(5, 1, 300), (30, 16, 200), (7, 33, 700), (1, 1000, 4), (64, 32, 257)])
def test_group_max(groups, K, D):
    """Max over K rows per group, exact, to fp32 and to the split output (equal to split(max)); K = 1 and D > 256."""
    ops = _ops()
    x = _randn((groups * K, D), 121)
    want = x.view(groups, K, D).amax(1)
    y, sp = _nan((groups, D)), _nan_split(groups, D)
    ops.group_max(x, groups, K, out_f32=y, out_split=sp)
    assert torch.equal(y, want)
    _assert_split_is(sp, want, "group_max")
    sp2 = _nan_split(groups, D)
    ops.group_max(x, groups, K, out_split=sp2)
    _assert_split_is(sp2, want, "group_max (split only)")


@pytest.mark.parametrize("L,lds,scale", [(1, 32, 1.0), (33, 40, 0.125), (200, 256, 0.125), (1000, 1000, 1.0), (200, 256, 64.0),
                                         (77, 96, 1000.0)])
def test_softmax_split(L, lds, scale):
    """Row softmax of the first L of lds columns: L not a multiple of 32, scales that underflow most of a row."""
    ops = _ops()
    rows = 300
    s = _randn((rows, lds), 131)
    p = _nan_split(rows, L, pitch=(L + 63) // 64 * 64)
    ops.softmax_split(s, L, scale, p)
    t = s[:, :L].double() * scale
    want = torch.softmax(t, -1)
    m = t.amax(-1, keepdim=True)
    rel = 4 * U * (2 + t.abs() + m.abs() + (t - m).abs())
    rel = rel + (want * rel).sum(-1, keepdim=True) + 2 * math.sqrt(L) * U
    _check_bound(f"softmax_split L={L} scale={scale}", p.float(), want, want * (rel + SPLIT) + 2.0 ** -125)


# ------------------------------------------------------------------------------------------------
# psam_decoder_prepare, psam_mask_dot, psam_interp_ln_gelu, psam_add_bcast_f32, psam_split_f32 / psam_split_add_f32
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [0, 1, 5])
@pytest.mark.parametrize("rep", [1, 3])
@pytest.mark.parametrize("form", ["no_mask", "per_z", "batch1"])
def test_decoder_prepare(form, rep, P):
    """tokens = cat(iou_token, mask_tokens, sparse[z]) and src = repeat_interleave(pc_emb, rep) + dense in the three dense
    forms the engine passes; exact."""
    nv = _nv()
    B, nmt, G, D = 2, 4, 48, 256
    Z, T = B * rep, 1 + nmt + P
    iou, mt = _ints((D,), -99, 99, 141), _ints((nmt, D), -99, 99, 142)
    sparse = _ints((Z, P, D), -99, 99, 143) if P else None
    pc = _ints((B, G, D), -99, 99, 144)
    if form == "no_mask":
        dense, dz, dg = _ints((D,), -99, 99, 145), 0, 0
        dense_full = dense.expand(Z, G, D)
    elif form == "per_z":
        dense, dz, dg = _ints((Z, G, D), -99, 99, 146), G * D, D
        dense_full = dense
    else:
        dense, dz, dg = _ints((1, G, D), -99, 99, 147), 0, D
        dense_full = dense.expand(Z, G, D)
    tokens, src = _nan((Z * T, D)), _nan((Z * G, D))
    rc = nv.lib().psam_decoder_prepare(nv.ptr(iou), nv.ptr(mt), nmt, nv.ptr(sparse), P, nv.ptr(pc), nv.ptr(dense), dz, dg, Z, rep,
                                       G, D, nv.ptr(tokens), nv.ptr(src), nv.stream())
    assert rc == 0
    parts = [iou.expand(Z, 1, D), mt.expand(Z, nmt, D)] + ([sparse] if P else [])
    assert torch.equal(tokens, torch.cat(parts, 1).reshape(Z * T, D))
    want_src = (pc.double().repeat_interleave(rep, 0) + dense_full.double()).float()
    assert torch.equal(src, want_src.reshape(Z * G, D))


_MD = [(C, [33, 2047, 3000, 10000][C % 4], [128, 256][C % 2]) for C in range(1, 9)]


@pytest.mark.parametrize("C,N,D", _MD)
def test_mask_dot(C, N, D):
    """masks[z, c, n] = hyper[z, c] . u[z*N + n, :D] with Z = 3 and a row stride ldu = D + 3 whose extra columns hold NaN:
    exact on integers, then bounded on random inputs."""
    nv = _nv()
    Z, ldu = 3, D + 3

    def run(u, hyper):
        masks = _nan((Z, C, N))
        assert nv.lib().psam_mask_dot(nv.ptr(u), ldu, nv.ptr(hyper), Z, C, N, D, nv.ptr(masks), nv.stream()) == 0
        return masks

    u = _ints((Z * N, ldu), -8, 8, 151)
    u[:, D:] = float("nan")
    hyper = _ints((Z, C, D), -8, 8, 152)
    uz = u[:, :D].double().view(Z, N, D)
    assert torch.equal(run(u, hyper), (hyper.double() @ uz.transpose(1, 2)).float())
    u = _randn((Z * N, ldu), 153)
    u[:, D:] = float("nan")
    hyper = _randn((Z, C, D), 154)
    uz = u[:, :D].double().view(Z, N, D)
    bound = 4 * math.sqrt(D) * U * (hyper.double().abs() @ uz.abs().transpose(1, 2))
    _check_bound(f"mask_dot C={C} N={N} D={D}", run(u, hyper), hyper.double() @ uz.transpose(1, 2), bound)


def test_mask_dot_refuses_nine_masks():
    nv = _nv()
    u, h, m = _randn((64, 128), 155), _randn((9, 128), 156), _nan((9, 64))
    assert nv.lib().psam_mask_dot(nv.ptr(u), 128, nv.ptr(h), 1, 9, 64, 128, nv.ptr(m), nv.stream()) == -1


def _interp_call(f, Z, rep, G, D, idx, w, N, g, b, eps, out):
    nv = _nv()
    return nv.lib().psam_interp_ln_gelu(nv.ptr(f), Z, rep, G, D, nv.ptr(idx), nv.ptr(w), N, nv.ptr(g), nv.ptr(b), eps,
                                        out.ptr() if out is not None else None, out.plane if out is not None else 0,
                                        out.pitch if out is not None else 0, nv.stream())


@pytest.mark.parametrize("shift", [0.0, 100.0], ids=["centred", "mean_gg_spread"])
@pytest.mark.parametrize("D", [128, 256, 512, 1024], ids=lambda D: f"interp_ln_gelu_kernel<{D // 128},false>-D{D}")
def test_interp_ln_gelu(D, shift):
    """GELU(LN(sum_k w_k f[z, idx_k])) for Z = 4 prompts of B = 2 clouds (rep = 2), N = 1001 points (a ragged last CTA),
    repeated indices among a point's three."""
    B, rep, G, N = 2, 2, 64, 1001
    Z = B * rep
    f = _randn((Z, G, D), 161, shift=shift)
    idx = torch.randint(0, G, (B, N, 3), generator=_gen(162))
    idx[:, ::5, 1] = idx[:, ::5, 0]
    idx[:, ::7, 2] = idx[:, ::7, 0]
    idx = idx.to(_dev())
    w = torch.rand(B, N, 3, generator=_gen(163)) + 0.05
    w = (w / w.sum(-1, keepdim=True)).to(_dev())
    g, b = _randn((D,), 164, 0.5, 1.0), _randn((D,), 165, 0.2)
    out = _nan_split(Z * N, D)
    assert _interp_call(f, Z, rep, G, D, idx, w, N, g, b, 1e-5, out) == 0
    zb = torch.arange(Z, device=_dev()) // rep
    fz = f.double()[torch.arange(Z, device=_dev())[:, None, None], idx[zb]]    # [Z, N, 3, D]
    wz = w.double()[zb][..., None]                                              # [Z, N, 3, 1]
    v = (fz * wz).sum(2).reshape(Z * N, D)
    inmag = 2 * (fz.abs() * wz).sum(2).reshape(Z * N, D)
    y_pre, rstd = _ln64(v, g.double(), b.double(), 1e-5)
    want = _act64(y_pre, ACT_GELU)
    bound = _ln_bound(inmag, g.double(), b.double(), y_pre, rstd, ACT_GELU) + SPLIT * want.abs()
    _check_bound(f"interp_ln_gelu D={D} shift={shift}", out.float(), want, bound)


def test_interp_ln_gelu_refuses_d_192():
    B, G, D, N = 1, 8, 192, 16
    f = _randn((1, G, D), 166)
    idx = torch.zeros(B, N, 3, dtype=torch.int64, device=_dev())
    w = torch.full((B, N, 3), 1 / 3, device=_dev())
    g = torch.ones(D, device=_dev())
    assert _interp_call(f, 1, 1, G, D, idx, w, N, g, g, 1e-5, _ops().Split(N, D, _dev())) == -2


@pytest.mark.parametrize("chunk,rep", [(48, 2), (48, 1), (7, 3)])
def test_add_bcast(chunk, rep):
    """out[i] = a[i] + b[(((i / chunk) / rep) * chunk + i % chunk) % b_period], exact on integers."""
    ops = _ops()
    nb = 2
    a, b = _ints((nb * rep * chunk * 3,), -99, 99, 171), _ints((nb * chunk,), -99, 99, 172)
    got = ops.add_bcast(a, b, chunk=chunk, rep=rep)
    i = torch.arange(a.numel(), device=_dev())
    want = a + b[(((i // chunk) // rep) * chunk + i % chunk) % b.numel()]
    assert torch.equal(got, want)


@pytest.mark.parametrize("rows,D,pitch", [(300, 200, 256), (7, 64, 64), (1000, 2730, 2752)])
def test_split_and_split_add(rows, D, pitch):
    """split_f32 / split_add_f32: the planes equal split(x) / split(x + add) exactly, pad columns zero; on 16-bit integers
    times a power of two (which hi + lo represents exactly) hi + lo equals the input, and the sum with `add`."""
    ops = _ops()
    x, add = _randn((rows, D), 181), _randn((rows, D), 182)
    xi, addi = (_ints((rows, D), -2 ** 14, 2 ** 14, s) * 2.0 ** -7 for s in (183, 184))
    for (u, a) in ((x, None), (x, add), (xi, None), (xi, addi)):
        sp = _nan_split(rows, D, pitch=pitch)
        ops.split_f32(u, sp, add=a)
        want = u if a is None else u + a
        _assert_split_is(sp, want, "split_f32")
        _assert_pad_zero(sp, D, "split_f32")
        if u is xi:
            assert torch.equal(sp.t[0, :, :D].double() + sp.t[1, :, :D].double(), want.double())


# ------------------------------------------------------------------------------------------------
# psam_knn3_interp_f32
# ------------------------------------------------------------------------------------------------
def test_knn3_interp_order_and_weights():
    """Indices equal the C oracle's 3 nearest (distance, then lower index) exactly; weights = normalised
    1 / clamp(d^2, 1e-8) against fp64 at rel 1e-6, with queries that coincide with a centre and two duplicated centres
    (the hierarchical decoder's distance-0 case)."""
    from oracle import tokenizer_ref

    ops = _ops()
    B, N, G = 2, 5000, 64
    xyz = torch.rand(B, N, 3, generator=_gen(191)) * 2 - 1
    perm = torch.randperm(N, generator=_gen(192))[:G]
    centers = xyz[:, perm].clone()
    centers[:, 17] = centers[:, 5]  # duplicated centre: a point on it has two neighbours at distance 0
    xyz[:, 3] = centers[:, 5]
    idx, w = ops.knn3_interp(xyz.to(_dev()), centers.to(_dev()))
    widx, wd2 = tokenizer_ref.knn(xyz.numpy(), centers.numpy(), 3)
    assert np.array_equal(idx.cpu().numpy(), widx)
    assert (widx[:, 3, :2] == [5, 17]).all() and (wd2[:, 3, :2] == 0).all()
    assert (wd2[:, perm[:G].numpy(), 0] == 0).sum() >= B * (G - 2)
    inv = 1.0 / np.maximum(wd2.astype(np.float64), 1e-8)
    want = inv / inv.sum(-1, keepdims=True)
    got = w.cpu().numpy().astype(np.float64)
    ratio = float((np.abs(got - want) / (1e-6 * want)).max())
    print(f"[glue] knn3_interp weights: max rel err {ratio * 1e-6:.3e} (bound 1e-6)")
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------
# max-pools with atomics: psam_scatter_amax_f32 and the GEMM's group-max epilogue (-0.0 included)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,G,D", [(2, 3000, 64, 8), (1, 100000, 8, 16), (3, 517, 200, 4)],
                         ids=["cells64", "contention_1e5_points_8_cells", "sparse_cells"])
def test_scatter_amax(B, N, G, D):
    """Bit for bit equal to zeros.scatter_reduce_(1, idx, x, "amax", include_self=False): cells c = 1 (mod 4) hold only
    negative values, cells c = 2 (mod 4) negative values and -0.0 (the maximum is -0.0), the top eighth of the cells
    (when G >= 16) no point at all (0)."""
    ops = _ops()
    g = _gen(201)
    x = torch.randint(1, 9, (B, N, D), generator=g).float() * (torch.randint(0, 2, (B, N, D), generator=g) * 2 - 1)
    used = G - G // 8 if G >= 16 else G
    idx = torch.randint(0, used, (B, N), generator=g)
    neg = (idx % 4 == 1) | (idx % 4 == 2)
    x[neg] = -x[neg].abs()
    zero_cells = []
    for b in range(B):
        for c in range(2, used, 4):
            pts = (idx[b] == c).nonzero()
            if len(pts):
                x[b, pts[len(pts) // 2, 0]] = -0.0
                zero_cells.append((b, c))
    want = torch.zeros(B, G, D).scatter_reduce_(1, idx[..., None].expand(B, N, D), x, "amax", include_self=False)
    zc = torch.stack([want[b, c] for (b, c) in zero_cells])
    assert bool(((zc == 0) & zc.signbit()).all()), "fixture: the -0.0 cells must have maximum -0.0"
    got = ops.scatter_amax(x.to(_dev()), idx.to(_dev()), G).cpu()
    bad = got.view(torch.int32) != want.view(torch.int32)
    assert not bool(bad.any()), f"{int(bad.sum())} cells differ, first {bad.nonzero()[:3].tolist()}: got " \
                                f"{got[bad][:3].tolist()} want {want[bad][:3].tolist()}"


@pytest.mark.parametrize("N", [128, 100], ids=["vector_epilogue", "ragged_columns"])
def test_gemm_group_max_negative_zero(N):
    """GEMM with gmax, alpha = -1 and bias = -0.0: A and W hold positive integers (exact in bf16), so every product is
    exact and a zero row of A gives the accumulator +0 and the value fmaf(+0, -1, -0.0) = -0.0, the maximum of its
    32-row group.  The result is that -0.0, not the caller's -inf fill."""
    ops = _ops()
    M, K, gr = 128, 64, 32
    a, w = _ints((M, K), 1, 8, 211), _ints((N, K), 1, 4, 212)
    a[37] = 0.0
    bias = torch.full((N,), -0.0, device=_dev())
    y = torch.full((M // gr, N), float("-inf"), device=_dev())
    ops.gemm(ops.pack_weight(a), ops.pack_weight(w), bias=bias, alpha=-1.0, gmax=y, group_rows=gr)
    want = (-(a.double() @ w.double().t())).view(M // gr, gr, N).amax(1).float()
    assert not bool(torch.isinf(y).any()), f"{int(torch.isinf(y).sum())} group maxima left at -inf"
    assert torch.equal(y, want)
    assert bool(((y[1] == 0) & y[1].signbit()).all())


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def _kernels_launched(fn):
    """Names of the CUDA kernels fn launches, in launch order (torch.profiler, CUDA activity)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA and "_kernel" in e.name]
    ev.sort(key=lambda e: e.time_range.start)
    return [e.name for e in ev]


def _guard(calls):
    """calls: (expected instantiation, thunk) pairs, one launch each."""
    names = _kernels_launched(lambda: [fn() for _, fn in calls])
    assert len(names) == len(calls), f"{len(calls)} calls launched {len(names)} kernels: {names}"
    for (want, _), got in zip(calls, names):
        assert want + ("(" if "<" not in want else "") in got, f"expected {want}, ran {got}"


@pytest.mark.parametrize("family", ["linear", "attention", "layernorm"])
def test_routing_guard(family, monkeypatch):
    """One representative per dispatch branch runs under the profiler; the instantiation that ran must be the one the case
    ids above name."""
    ops = _ops()
    calls = []
    if family == "linear":
        N = 65
        for (M, K) in [(1, 512), (4, 512), (8, 2048), (1, 256), (4, 256), (8, 256), (16, 2048), (1, 255), (4, 255), (8, 255),
                       (16, 255), (17, 256), (17, 255)]:
            x, w = _randn((M, K), 1), _randn((N, K), 2)
            calls.append((_linear_kernel(M, K, K % 4 == 0), lambda x=x, w=w: ops.linear_f32(x, w)))
    elif family == "attention":
        for dh in (8, 16, 32, 64):
            for (Z, H, Lq, Lk) in [(2, 4, 64, 128), (3, 3, 57, 128)]:
                q, k = _randn((Z * Lq, H * dh), 3), _randn((Z * Lk, H * dh), 4)
                calls.append((_attn_kernel(dh, Z * H * Lq, Lk),
                              lambda q=q, k=k, a=(Z, Lq, Lk, H, dh): ops.attention_f32(q, k, k, *a)))
    else:
        for c in [(128, 64, 1, ""), (256, 64, 1, ""), (384, 64, 1, ""), (1024, 64, 1, ""), (256, 64, 0, ""), (2048, 64, 0, ""),
                  (4096, 64, 0, ""), (97, 64, 0, ""), (255, 64, 0, ""), (511, 64, 1, ""), (1023, 64, 1, ""), (256, 64, 0, "odd_ldx"),
                  (511, 64, 0, ""), (1023, 64, 0, ""), (1025, 64, 0, ""), (2730, 64, 0, "")]:
            D, rows, policy, form = c
            ldx = D + 1 if form else D
            x, g = _randn((rows, ldx), 5), torch.ones(D, device=_dev())
            y = torch.empty(rows, D, device=_dev())

            def run(x=x, g=g, y=y, D=D, rows=rows, ldx=ldx, policy=policy):
                monkeypatch.setattr(ops, "GEMM_TILE_HINT", policy)
                ops.layernorm(x, g, g, 1e-6, rows=rows, D=D, ldx=ldx, out_f32=y)

            calls.append((_ln_case_kernel(*c), run))
    _guard(calls)
