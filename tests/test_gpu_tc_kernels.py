"""The tensor-core kernels (csrc/gemm_tc.cu: psam_gemm_bf16x3, psam_gemm_rowln_bf16x3; csrc/attention_tc.cu:
psam_attention_bf16x3 and its two-pass form) against plain fp64 restatements, through the C ABI, on every launch path.

Two kinds of check:
  * integer-valued inputs (|a| <= 8, |w| <= 4), exact in bf16 (the lo planes are zero) with every partial sum below 2^23
    and power-of-two alphas, where passes = 1 and passes = 3 must both equal the fp64 result bit for bit: a wrong row,
    column, batch offset, k-block or K tail fails at once.  The attention's one-hot cases (every other key >= 128 below
    the peak after scaling) must return the selected V row exactly;
  * random inputs against an elementwise bound.  With P = |A| @ |W|^T the GEMM bound is
        passes = 3:  (C1 2^-16 + C2 sqrt(K) 2^-24) P     (two operand splits of <= 2^-18 each, the dropped lo*lo term,
        passes = 1:  (C1 2^-8  + C2 sqrt(K) 2^-24) P      fp32 accumulation; one bf16 rounding per operand at passes = 1)
    and each epilogue adds its own roundings.  Each case prints its largest error / bound, and test_bounds_have_teeth
    checks that every family's bound rejects a result with the lo passes of one k-block dropped, the last K column
    dropped, or one output row shifted.
Every operand sits in a NaN-filled buffer with more rows than `rows` and pad columns past `k` (the TMA reads must stop at
the logical extents), and every output buffer is NaN outside the window the call may write.  Case ids name the kernel
instantiation they reach; test_routing_guard checks those names under torch.profiler."""
import math
from ctypes import byref

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24       # fp32 unit roundoff
SPLIT = 2.0 ** -16   # split-bf16 output: |hi + lo - y| <= 2^-18 |y|, with slack
GELU_ABS = 1e-6      # the kernels' GELU uses the A&S 7.1.26 erf (|error| <= 1.5e-7)
EX2 = 2.0 ** -21     # relative error of ex2.approx.ftz.f32 (2 ulp), with slack
C1, C2 = 4.0, 4.0    # constants of the GEMM bound
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
ERR_ARG = -1
GV_SCALAR_EPI = 0x4


@pytest.fixture(autouse=True)
def _pinned_policy(monkeypatch):
    """The results must not depend on the experiment switches ops seeds from the environment."""
    ops = _ops()
    monkeypatch.setattr(ops, "GEMM_VARIANT", 0)
    monkeypatch.setattr(ops, "GEMM_TILE_BN", 0)
    monkeypatch.setattr(ops, "GEMM_TILE_HINT", 0)


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
    return torch.randint(lo, hi + 1, shape, generator=_gen(seed)).float().to(_dev())


def _randn(shape, seed, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=_gen(seed)) * scale + shift).to(_dev())


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=_dev())


def _act64(y, act):
    if act == ACT_GELU:
        return torch.nn.functional.gelu(y)
    if act == ACT_RELU:
        return torch.relu(y)
    return y


def _ratio(got, want, bound):
    return float(((got.double() - want).abs() / bound.clamp_min(1e-300)).max())


def _check_bound(name, got, want, bound):
    """|got - want| <= bound elementwise (want and bound fp64); prints the largest error and error / bound."""
    err = (got.double() - want).abs()
    ratio = _ratio(got, want, bound)
    print(f"[tc] {name}: max|err| {float(err.max()):.3e}, max err/bound {ratio:.3f}")
    assert ratio <= 1.0, f"{name}: error {ratio:.2f}x its bound"


def _rejects(name, wrong, want, bound):
    ratio = _ratio(wrong, want, bound)
    print(f"[tc] teeth {name}: wrong result at {ratio:.1f}x the bound")
    assert ratio > 1.0, f"{name}: the bound accepts a wrong result"


def _split_of(y):
    """The split-bf16 planes the kernels write for fp32 y: hi = bf16_rn(y), lo = bf16_rn(y - hi)."""
    hi = y.to(torch.bfloat16)
    return hi, (y - hi.float()).to(torch.bfloat16)


def _assert_split_is(hi, lo, y, name):
    h, l = _split_of(y)
    assert torch.equal(hi, h) and torch.equal(lo, l), f"{name}: split planes != split(fp32 output)"


def _exact(got, want, name):
    want = want.float()
    bad = got != want
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} of {got.numel()} differ, first {bad.nonzero()[:3].tolist()}"


def _only_window(buf, written, name):
    """Every element of buf outside the boolean mask `written` is still the NaN it was filled with."""
    outside = buf[~written]
    assert bool(torch.isnan(outside.float()).all()), f"{name}: {int((~torch.isnan(outside.float())).sum())} writes outside the window"


def _no_nan(t, name):
    assert not bool(torch.isnan(t.float()).any()), f"{name}: NaN in the output (operand padding was read)"


# ------------------------------------------------------------------------------------------------
# operands: split-bf16 planes in NaN-filled buffers
# ------------------------------------------------------------------------------------------------
class Planes:
    """x [R, K] fp32 as split-bf16 planes in a [2, R + extra, pitch] buffer whose extra rows and pad columns are NaN."""

    def __init__(self, x, extra_rows=5, pitch=None):
        R, K = x.shape
        self.R, self.K = R, K
        self.pitch = pitch or (K + 8 + 63) // 64 * 64
        self.t = _nan((2, R + extra_rows, self.pitch), torch.bfloat16)
        hi, lo = _split_of(x)
        self.t[0, :R, :K], self.t[1, :R, :K] = hi, lo
        self.x = x

    def seen(self, passes):
        """The operand the kernel multiplies, fp64: hi (+ lo)."""
        v = self.t[0, :self.R, :self.K].double()
        return v + self.t[1, :self.R, :self.K].double() if passes == 3 else v

    def operand(self, nb1=0, nb2=0, b1=0, b2=0, rows=None):
        nv = _nv()
        return nv.Operand(self.t.data_ptr(), self.t.shape[1] * self.pitch, rows or self.R, self.K, self.pitch, nb1, nb2, b1, b2)


def _gemm_err(A, W, K, passes):
    """The GEMM bound on inputs A [.., M, K], W [.., N, K] (fp64)."""
    P = A.abs() @ W.abs().transpose(-1, -2)
    return ((C1 * (2.0 ** -16 if passes == 3 else 2.0 ** -8)) + C2 * math.sqrt(K) * U) * P


def _call_gemm(ao, wo, o, passes, split_k):
    nv = _nv()
    return nv.lib().psam_gemm_bf16x3(byref(ao), byref(wo), byref(o), passes, split_k, nv.stream())


def _gemm_out(**fields):
    o = _nv().GemmOut()
    o.alpha = 1.0
    for k, v in fields.items():
        setattr(o, k, v)
    return o


# ------------------------------------------------------------------------------------------------
# dispatch of psam_gemm_bf16x3, restated (test_routing_guard checks these against the kernels that run)
# ------------------------------------------------------------------------------------------------
def _bn(M, N, K, batches, split_k, throughput):
    """choose_bn: the tile width minimising waves (latency) or SM-time (throughput) x per-CTA cost."""
    mt = -(-M // 128)
    kb = -(-(-(-K // 64)) // split_k)
    best, best_cost = 128, 1e30
    for bn in (64, 128, 256):
        if bn > 64 and bn // 2 >= N:
            break
        tiles = -(-N // bn) * mt * batches * split_k
        waves = (tiles + 131) // 132
        per = 6.0 * 256 + kb * (128 + bn) + 0.35 * bn * 4
        cost = tiles * per if throughput else waves * per
        if cost < best_cost - 1e-9:
            best_cost, best = cost, bn
    return best


def _tile(hint, M, N, K, batches=1, split_k=1):
    if 32 <= hint <= 256 and hint % 32 == 0:
        return 64 if hint <= 64 else 128 if hint <= 128 else 256
    return _bn(M, N, K, batches, split_k, hint == 1)


def _gk(bn):
    return f"gemm_wgmma_kernel<{bn}>"


def _id(kernel, **kw):
    return kernel.replace(", ", ",") + "-" + "-".join(f"{k}{v}" for k, v in kw.items())


# ------------------------------------------------------------------------------------------------
# psam_gemm_bf16x3: shapes, tile widths, K tails, exact
# ------------------------------------------------------------------------------------------------
_M = [1, 127, 128, 129, 300, 32768 + 5]
_N = [1, 31, 32, 33, 96, 200, 344, 1024]
_K = [1, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, 200, 2730]
_HINTS = [0, 1, 64, 128, 256]
_GRID = [(i, j, M, K, _N[(i + j) % len(_N)], _HINTS[(i + 2 * j) % len(_HINTS)], (1, 3)[j % 2])
         for i, M in enumerate(_M) for j, K in enumerate(_K)]


@pytest.mark.parametrize("i,j,M,K,N,hint,passes", _GRID,
                         ids=[_id(_gk(_tile(h, M, N, K)), M=M, K=K, N=N, hint=h, passes=p) for (i, j, M, K, N, h, p) in _GRID])
def test_gemm_shapes_exact(i, j, M, K, N, hint, passes):
    """Every M, N and K tail under every tile width (forced, and choose_bn's latency and throughput picks), fp32 output
    with bias, alpha in {1, 1/8, -1}, ReLU and a residual in turn; bit for bit, nothing written outside [M, N], no NaN
    from the operand padding."""
    s = 1000 + 100 * i + j
    A, W = Planes(_ints((M, K), -8, 8, s)), Planes(_ints((N, K), -4, 4, s + 1), extra_rows=3)
    b = _ints((N,), -64, 64, s + 2)
    alpha = (1.0, 0.125, -1.0)[(i + 2 * j) % 3]
    act = (ACT_NONE, ACT_RELU)[i % 2]
    ldo = (N + 3) // 4 * 4 + 4
    out = _nan((M + 2, ldo))
    r, rbuf = None, None
    if (i + j) % 3 == 0:   # the residual has out_f32's geometry, NaN in its pad columns
        r = _ints((M, N), -64, 64, s + 3)
        rbuf = _nan((M, ldo))
        rbuf[:, :N] = r
    o = _gemm_out(out_f32=out.data_ptr(), ldo=ldo, bias=b.data_ptr(), resid=rbuf.data_ptr() if r is not None else None,
                  alpha=alpha, act=act, tile_hint=hint)
    assert _call_gemm(A.operand(), W.operand(), o, passes, 1) == 0
    acc = A.x.double() @ W.x.double().t()
    want = _act64(alpha * acc + b.double() + (r.double() if r is not None else 0.0), act)
    _exact(out[:M, :N], want, f"M={M} N={N} K={K}")
    mask = torch.zeros_like(out, dtype=torch.bool)
    mask[:M, :N] = True
    _only_window(out, mask, "gemm")


_RAND = [(300, 200, 2730, 0), (129, 344, 65, 64), (1, 1024, 200, 128), (32768 + 5, 96, 33, 256), (127, 33, 17, 1), (300, 1024, 2730, 256)]


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("M,N,K,hint", _RAND, ids=[_id(_gk(_tile(h, M, N, K)), M=M, N=N, K=K, hint=h) for (M, N, K, h) in _RAND])
def test_gemm_random(M, N, K, hint, passes):
    """Random inputs with bias and GELU against fp64: the GEMM bound, GELU's slope and absolute error; no NaN from the
    operand padding."""
    a, w, b = _randn((M, K), 1), _randn((N, K), 2, K ** -0.5), _randn((N,), 3)
    A, W = Planes(a), Planes(w, extra_rows=3)
    out = _nan((M, N + 4))
    o = _gemm_out(out_f32=out.data_ptr(), ldo=N + 4, bias=b.data_ptr(), act=ACT_GELU, tile_hint=hint)
    assert _call_gemm(A.operand(), W.operand(), o, passes, 1) == 0
    a64, w64 = a.double(), w.double()
    pre = a64 @ w64.t() + b.double()
    want = _act64(pre, ACT_GELU)
    bound = 1.2 * (_gemm_err(a64, w64, K, passes) + 2 * U * pre.abs()) + GELU_ABS * (1 + pre.abs())
    _check_bound(f"gemm {_gk(_tile(hint, M, N, K))} passes={passes} M={M} N={N} K={K}", out[:, :N], want, bound)
    assert bool(torch.isnan(out[:, N:]).all())


# ------------------------------------------------------------------------------------------------
# psam_gemm_bf16x3: every output form under both epilogues
# ------------------------------------------------------------------------------------------------
_FORMS = {  # form: (epilogues, activations)
    "f32": (("vec", "scalar", "ldo"), (ACT_NONE, ACT_GELU, ACT_RELU)),
    "split": (("vec", "scalar", "ldo", "odd_col"), (ACT_NONE, ACT_GELU, ACT_RELU)),
    "split_f32": (("vec", "scalar", "ldo"), (ACT_NONE, ACT_GELU, ACT_RELU)),
    "acc": (("vec", "scalar", "ldo"), (ACT_NONE,)),
    "swiglu": (("vec", "scalar", "ldo"), (ACT_NONE,)),
    "swiglu_split": (("vec",), (ACT_NONE,)),
    "gmax": (("vec", "scalar"), (ACT_NONE,)),
    "gmax_outputs": (("vec", "scalar"), (ACT_NONE,)),
    "rowdot": (("scalar",), (ACT_NONE, ACT_GELU, ACT_RELU)),
}
_EPI = [(f, e, a) for f, (es, acts) in _FORMS.items() for e in es for a in acts]
_ACTN = {ACT_NONE: "none", ACT_GELU: "gelu", ACT_RELU: "relu"}


def _epi_shape(form):
    if form == "rowdot":
        return 3 * 96, 200, 200   # rd_rows = 96: M % 128 != 0, the last warps of the last m-tile lie past M
    if form == "swiglu_split":
        return 300, 256, 200
    return 300, 200, 200


def _run_form(form, epi, act, idx, ints, passes=3):
    """One call of the output form; returns a list of (name, got, want, bound or None for exact) checks."""
    M, N, K = _epi_shape(form)
    s = 5000 + 37 * idx + (0 if ints else 7)
    if ints:
        a, w, b = _ints((M, K), -8, 8, s), _ints((N, K), -4, 4, s + 1), _ints((N,), -64, 64, s + 2)
    else:
        a, w, b = _randn((M, K), s), _randn((N, K), s + 1, K ** -0.5), _randn((N,), s + 2)
    A, W = Planes(a), Planes(w, extra_rows=3)
    alpha = (1.0, 0.125, -1.0)[idx % 3]
    if form in ("gmax", "gmax_outputs", "swiglu", "swiglu_split", "rowdot"):
        alpha = (1.0, 0.125)[idx % 2]
    rkind = None
    if form in ("f32", "split_f32"):
        rkind = (None, "sep", "alias")[idx % 3]
    elif form == "split":
        rkind = (None, "sep")[idx % 2]
    elif form == "acc":
        rkind = (None, "alias")[idx % 2]   # out_f32 is its own residual; no other one is accepted
    a64, w64 = A.seen(passes), W.seen(passes)
    acc = a64 @ w64.t()
    E = None if ints else _gemm_err(a.double(), w.double(), K, passes)
    variant = GV_SCALAR_EPI if epi == "scalar" else 0
    has_f32 = form in ("f32", "split_f32", "acc", "swiglu", "gmax_outputs")
    has_split = form in ("split", "split_f32", "swiglu_split", "gmax_outputs")
    ncol = N // 2 if form.startswith("swiglu") else N
    # fp32 output buffer [M + 2, ldo]: ldo % 4 != 0 for "ldo"
    if epi == "ldo" and has_f32:
        ldo = ncol + (1 if (ncol + 1) % 4 else 2)
    else:
        ldo = (ncol + 3) // 4 * 4 + 4
    if epi == "ldo" and rkind == "sep" and not has_f32:
        ldo = ncol + 1   # the residual's row stride alone must keep the float4 loads out
    out = _nan((M + 2, ldo)) if has_f32 else None
    r = (_ints((M, ncol), -64, 64, s + 3) if ints else _randn((M, ncol), s + 3)) if rkind else None
    init = None
    if form == "acc":
        init = r if rkind == "alias" else (_ints((M, ncol), -64, 64, s + 4) if ints else _randn((M, ncol), s + 4))
        r = None
        out[:M, :ncol] = init
    elif rkind == "alias":
        out[:M, :ncol] = r
    rbuf = None
    if rkind == "sep":
        rbuf = _nan((M + 2, ldo))
        rbuf[:M, :ncol] = r
    # split output [2 planes of (M + 2) * ldo_s + 8]: ldo_s % 4 != 0 for "ldo", odd first column for "odd_col"
    ldo_s = ncol + 2 if epi in ("ldo", "odd_col") else (ncol + 3) // 4 * 4 + 8
    col0 = 1 if epi == "odd_col" else 0
    plane = (M + 2) * ldo_s + 8
    sp = _nan((2 * plane,), torch.bfloat16) if has_split else None
    stats = torch.zeros(M, 2, device=_dev()) if form == "swiglu_split" else None
    fields = dict(bias=b.data_ptr(), alpha=alpha, act=act, variant=variant, tile_hint=(0, 64, 128, 256)[idx % 4])
    if out is not None:
        fields.update(out_f32=out.data_ptr(), ldo=ldo)
    if sp is not None:
        fields.update(out_hi=sp.data_ptr() + 2 * col0, out_plane=plane, ldo_s=ldo_s)
    if rkind == "sep":
        fields.update(resid=rbuf.data_ptr(), ldo=ldo)
    if rkind == "alias":
        fields.update(resid=out.data_ptr())
    if form == "acc":
        fields.update(accumulate=1)
    if form.startswith("swiglu"):
        fields.update(swiglu=1)
    if stats is not None:
        fields.update(stats_out=stats.data_ptr())
    gr = 32 if idx % 2 else 64
    gmax = None
    if form.startswith("gmax"):
        gmax = torch.full((-(-M // gr) + 1, N + 4), float("-inf"), device=_dev())
        fields.update(gmax=gmax.data_ptr(), ld_gmax=N + 4, group_rows=gr)
    rd_c, rd_rows = 3, 96
    if form == "rowdot":
        rd_w = _ints((M // rd_rows, rd_c, N), -4, 4, s + 5) if ints else _randn((M // rd_rows, rd_c, N), s + 5)
        rd_out = torch.zeros(M // rd_rows, rd_c, rd_rows, device=_dev())
        fields.update(rd_w=rd_w.data_ptr(), rd_out=rd_out.data_ptr(), rd_rows=rd_rows, rd_c=rd_c)
    assert _call_gemm(A.operand(), W.operand(), _gemm_out(**fields), passes, 1) == 0
    torch.cuda.synchronize()

    # ---- fp64 restatement ----
    pre = alpha * acc + b.double()
    Epre = None if ints else abs(alpha) * E + 2 * U * (alpha * acc).abs() + 2 * U * b.double().abs()
    if r is not None:
        pre = pre + r.double()
        Epre = None if ints else Epre + 2 * U * (pre.abs() + r.double().abs())
    y = _act64(pre, act)
    Ey = None
    if not ints:
        Ey = 1.2 * Epre + 4 * U * y.abs() + GELU_ABS * (1 + pre.abs()) if act == ACT_GELU else Epre
    if form.startswith("swiglu"):
        g, v = pre[:, 0::2], pre[:, 1::2]
        sg = torch.nn.functional.silu(g)
        y = sg * v
        if not ints:
            Eg, Ev = Epre[:, 0::2], Epre[:, 1::2]
            Ey = 1.1 * Eg * v.abs() + sg.abs() * Ev + Eg * Ev + 8 * U * (2 + g.abs()) * y.abs()
    if form == "acc":
        y = y + init.double()
        Ey = None if ints else Ey + 2 * U * (y.abs() + init.double().abs())
    checks = []
    name = f"{form} {epi} act={_ACTN[act]} alpha={alpha} resid={rkind}"
    if out is not None:
        checks.append((name + " fp32", out[:M, :ncol], y, Ey))
        mask = torch.zeros_like(out, dtype=torch.bool)
        mask[:M, :ncol] = True
        _only_window(out, mask, name + " fp32")
    if sp is not None:
        pl = sp.view(2, plane)
        win = lambda p: pl[p, :M * ldo_s].view(M, ldo_s)[:, col0:col0 + ncol]
        hi, lo = win(0), win(1)
        if out is not None:
            _assert_split_is(hi, lo, out[:M, :ncol], name)
        else:
            checks.append((name + " split", hi.float() + lo.float(), y, None if ints else Ey + SPLIT * y.abs()))
        mask = torch.zeros(2, plane, dtype=torch.bool, device=_dev())
        mask.view(2, plane)[:, :M * ldo_s].view(2, M, ldo_s)[:, :, col0:col0 + ncol] = True
        _only_window(sp.view(2, plane), mask, name + " split planes")
    if stats is not None:
        yk = out[:M, :ncol].double() if out is not None else win(0).double() + win(1).double()
        depth = 6 + ncol // 32
        s1b = depth * U * yk.abs().sum(1) + (0 if out is not None else 2.0 ** -17 * yk.abs().sum(1))
        s2b = (depth + 1) * U * (yk * yk).sum(1) + (0 if out is not None else 2.0 ** -16 * (yk * yk).sum(1))
        _check_bound(name + " stats sum", stats[:, 0], yk.sum(1), s1b + 1e-30)
        _check_bound(name + " stats sum sq", stats[:, 1], (yk * yk).sum(1), s2b + 1e-30)
    if gmax is not None:
        G = -(-M // gr)
        pad = torch.full((G * gr - M, N), float("-inf"), dtype=torch.float64, device=_dev())
        gwant = torch.cat([pre, pad]).view(G, gr, N).amax(1)
        gb = None if ints else torch.cat([Epre, torch.zeros_like(pad)]).view(G, gr, N).amax(1)
        checks.append((name + " gmax", gmax[:G, :N], gwant, gb))
        assert bool(torch.isinf(gmax[G:]).all()) and bool(torch.isinf(gmax[:, N:]).all()), name + ": gmax written outside [G, N]"
    if form == "rowdot":
        Z = M // rd_rows
        yz = y.view(Z, rd_rows, N)
        want_rd = rd_w.double() @ yz.transpose(1, 2)
        rb = None
        if not ints:
            rb = rd_w.double().abs() @ Ey.view(Z, rd_rows, N).transpose(1, 2) \
                + (34 + N // 32) * U * (rd_w.double().abs() @ yz.abs().transpose(1, 2))
        checks.append((name + " rowdot", rd_out, want_rd, rb))
    return checks


@pytest.mark.parametrize("form,epi,act", _EPI, ids=[f"{_gk(_tile((0, 64, 128, 256)[i % 4], *_epi_shape(f)))}-{f}-{e}-{_ACTN[a]}"
                                                    for i, (f, e, a) in enumerate(_EPI)])
def test_gemm_epilogue_forms(form, epi, act):
    """Each output form under the vectorised epilogue, the scalar one forced by GV_SCALAR_EPI, and the scalar one reached
    by an fp32 row stride (or split row stride) % 4 != 0 or an odd first column of the split output; residual none /
    separate / aliasing out_f32 and alpha in {1, 1/8, -1} in turn.  Integer inputs bit for bit where the form is exact
    (no GELU, no SwiGLU), random inputs against the bound always; where fp32 and split outputs are both written the planes
    equal split(fp32) bit for bit."""
    idx = _EPI.index((form, epi, act))
    if act != ACT_GELU and not form.startswith("swiglu"):
        for name, got, want, _ in _run_form(form, epi, act, idx, ints=True):
            _exact(got, want, name)
    for name, got, want, bound in _run_form(form, epi, act, idx, ints=False):
        _check_bound(name, got, want, bound)


@pytest.mark.parametrize("epi", ["vec", "scalar"])
def test_gemm_accumulate_with_split_output_refused(epi):
    """accumulate + a split output: the vectorised epilogue added and dropped the planes, the scalar one stored and wrote
    them.  Both are refused now, and the output is left untouched."""
    M, N, K = 128, 128, 64
    A, W = Planes(_ints((M, K), -8, 8, 1)), Planes(_ints((N, K), -4, 4, 2))
    out, sp = torch.zeros(M, N, device=_dev()), _nan((2, M, N), torch.bfloat16)
    o = _gemm_out(out_f32=out.data_ptr(), ldo=N, out_hi=sp.data_ptr(), out_plane=M * N, ldo_s=N, accumulate=1,
                  variant=GV_SCALAR_EPI if epi == "scalar" else 0)
    assert _call_gemm(A.operand(), W.operand(), o, 3, 1) == ERR_ARG
    torch.cuda.synchronize()
    assert bool((out == 0).all()) and bool(torch.isnan(sp.float()).all())


# ------------------------------------------------------------------------------------------------
# split-K (empty splits included) and batched operands
# ------------------------------------------------------------------------------------------------
_SK = [(300, 200, 64, 256, 3), (300, 200, 64, 256, 7), (129, 96, 200, 64, 3), (300, 344, 2730, 128, 2), (300, 344, 2730, 0, 7),
       (1, 1024, 65, 256, 7), (127, 33, 17, 64, 2), (32768 + 5, 96, 200, 0, 3)]


def _kb_split(K, bn, sk):
    bk = 32 if bn == 256 else 64
    kb = -(-K // bk)
    per = -(-kb // sk)
    return sum(1 for z in range(sk) if z * per >= kb)


@pytest.mark.parametrize("M,N,K,hint,sk", _SK, ids=[_id(_gk(_tile(h, M, N, K, 1, sk)), M=M, N=N, K=K, split_k=sk,
                                                         empty_splits=_kb_split(K, _tile(h, M, N, K, 1, sk), sk))
                                                     for (M, N, K, h, sk) in _SK])
def test_gemm_split_k(M, N, K, hint, sk):
    """Split-K accumulation into out_f32 (out_f32 is its own residual, resid may alias it): integers bit for bit at
    passes 1 and 3 with alpha in {1, -1}, the bias added exactly once, also when some splits get no k-block; random
    inputs against the bound."""
    for passes, alpha in ((3, 1.0), (1, -1.0)):
        A, W = Planes(_ints((M, K), -8, 8, 7)), Planes(_ints((N, K), -4, 4, 8), extra_rows=3)
        b, init = _ints((N,), -64, 64, 9), _ints((M, N), -64, 64, 10)
        out = _nan((M + 1, N + 4))
        out[:M, :N] = init
        o = _gemm_out(out_f32=out.data_ptr(), ldo=N + 4, bias=b.data_ptr(), alpha=alpha, accumulate=1, tile_hint=hint,
                      resid=out.data_ptr() if passes == 1 else None)
        assert _call_gemm(A.operand(), W.operand(), o, passes, sk) == 0
        _exact(out[:M, :N], init.double() + alpha * (A.x.double() @ W.x.double().t()) + b.double(), f"split_k={sk} passes={passes}")
        mask = torch.zeros_like(out, dtype=torch.bool)
        mask[:M, :N] = True
        _only_window(out, mask, "split_k")
    a, w, b, init = _randn((M, K), 11), _randn((N, K), 12, K ** -0.5), _randn((N,), 13), _randn((M, N), 14)
    A, W = Planes(a), Planes(w, extra_rows=3)
    out = init.clone()
    assert _call_gemm(A.operand(), W.operand(), _gemm_out(out_f32=out.data_ptr(), ldo=N, bias=b.data_ptr(), accumulate=1,
                                                          tile_hint=hint), 3, sk) == 0
    want = init.double() + a.double() @ w.double().t() + b.double()
    bound = _gemm_err(a.double(), w.double(), K, 3) + (sk + 2) * U * (want.abs() + init.double().abs() + b.double().abs()
                                                                       + (a.double().abs() @ w.double().abs().t()))
    _check_bound(f"split_k={sk} M={M} N={N} K={K}", out, want, bound)


_BATCH = [(3, 2, 200, 96, 65, 0, 1, "f32_split"), (2, 3, 129, 200, 33, 64, 1, "split"), (4, 1, 64, 64, 200, 256, 3, "acc"),
          (1, 3, 300, 344, 17, 128, 2, "acc"), (2, 2, 1, 33, 2730, 0, 1, "f32"), (2, 2, 127, 256, 64, 256, 7, "acc")]


@pytest.mark.parametrize("nb1,nb2,M,N,K,hint,sk,form", _BATCH,
                         ids=[_id(_gk(_tile(h, M, N, K, b1 * b2, sk)), nb1=b1, nb2=b2, M=M, N=N, K=K, split_k=sk, form=f)
                              for (b1, b2, M, N, K, h, sk, f) in _BATCH])
def test_gemm_batched(nb1, nb2, M, N, K, hint, sk, form):
    """Batched operands (nb1, nb2) with outputs in a layout unlike the inputs': A is [b2][b1][M + 3][pitch], W is
    [b1][b2][N + 2][pitch], the fp32 output [b2][b1][M + 3][ldo] with 8 floats between clouds, the split output
    [b1][b2][M + 1][ldo_s]; integers bit for bit, NaN everywhere else."""
    Mp, Np = M + 3, N + 2
    a = _ints((nb2, nb1, M, K), -8, 8, 21)
    w = _ints((nb1, nb2, N, K), -4, 4, 22)
    b = _ints((N,), -64, 64, 23)
    pitch = (K + 8 + 63) // 64 * 64
    At = _nan((2, nb2, nb1, Mp, pitch), torch.bfloat16)
    Wt = _nan((2, nb1, nb2, Np, pitch), torch.bfloat16)
    At[0, :, :, :M, :K], At[1, :, :, :M, :K] = _split_of(a)
    Wt[0, :, :, :N, :K], Wt[1, :, :, :N, :K] = _split_of(w)
    nv = _nv()
    ao = nv.Operand(At.data_ptr(), At[0].numel(), M, K, pitch, nb1, nb2, Mp * pitch, nb1 * Mp * pitch)
    wo = nv.Operand(Wt.data_ptr(), Wt[0].numel(), N, K, pitch, nb1, nb2, nb2 * Np * pitch, Np * pitch)
    want = torch.einsum("zymk,yznk->zymn", a.double(), w.double()) + b.double()   # [b2][b1][M][N]
    fields = dict(bias=b.data_ptr(), tile_hint=hint)
    ldo = (N + 3) // 4 * 4 + 4
    cloud = nb1 * Mp * ldo + 8
    out = None
    if form in ("f32", "f32_split", "acc"):
        out = _nan((nb2 * cloud,))
        fields.update(out_f32=out.data_ptr(), ldo=ldo, out_b1=Mp * ldo, out_b2=cloud)
    owin = lambda t: t.view(-1)[:nb2 * cloud].view(nb2, cloud)[:, :nb1 * Mp * ldo].view(nb2, nb1, Mp, ldo)[:, :, :M, :N]
    init = None
    if form == "acc":
        init = _ints((nb2, nb1, M, N), -64, 64, 24)
        owin(out).copy_(init)
        want = want + init.double()
        fields.update(accumulate=1)
    ldo_s = (N + 3) // 4 * 4 + 8
    plane = nb1 * nb2 * (M + 1) * ldo_s
    sp = None
    if form in ("split", "f32_split"):
        sp = _nan((2, nb1, nb2, M + 1, ldo_s), torch.bfloat16)
        fields.update(out_hi=sp.data_ptr(), out_plane=plane, ldo_s=ldo_s, outs_b1=nb2 * (M + 1) * ldo_s, outs_b2=(M + 1) * ldo_s)
    assert _call_gemm(ao, wo, _gemm_out(**fields), 3, sk) == 0
    torch.cuda.synchronize()
    if out is not None:
        _exact(owin(out), want, "batched fp32")
        mask = torch.zeros_like(out, dtype=torch.bool)
        owin(mask).fill_(True)
        _only_window(out, mask, "batched fp32")
    if sp is not None:
        hi, lo = (sp[p, :, :, :M, :N].transpose(0, 1) for p in (0, 1))   # -> [b2][b1][M][N]
        if out is not None:
            _assert_split_is(hi, lo, owin(out), "batched")
        else:
            _exact(hi.float() + lo.float(), want, "batched split")
        mask = torch.zeros_like(sp, dtype=torch.bool)
        mask[:, :, :, :M, :N] = True
        _only_window(sp, mask, "batched split planes")


# ------------------------------------------------------------------------------------------------
# stats_out and the folded LayerNorm (ln_stats / ln_c)
# ------------------------------------------------------------------------------------------------
def _fold_ref(acc, st, c, H, eps, alpha, bias):
    """alpha rstd (acc - mean c) + bias, mean / rstd from the fp32 (sum, sum sq) of each row; returns (pre, rstd, mean)."""
    mean = st[:, 0:1].double() / H
    var = (st[:, 1:2].double() / H - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + eps)
    pre = alpha * rstd * (acc - mean * c.double()) + (bias.double() if bias is not None else 0.0)
    return pre, rstd, mean


def _fold_bound(E, acc, st, c, H, eps, alpha, bias, pre, rstd, mean, sk):
    """The GEMM error scaled by alpha rstd, the roundings of acc rstd alpha and mean rstd c (large when mean >> spread), the
    rstd error from the fp32 variance E[x^2] - mean^2 and rsqrtf, and the bias; split-K adds one rounding per split."""
    ex2 = st[:, 1:2].double() / H
    var = (ex2 - mean * mean).clamp_min(0)
    drstd = 4 * U * ex2 / (var + eps) + 8 * U
    core = rstd * (acc - mean * c.double())
    bound = abs(alpha) * rstd * (E + 6 * U * (acc.abs() + (mean * c.double()).abs())) + drstd * abs(alpha) * core.abs()
    return bound + (2 + sk) * U * (pre.abs() + (bias.double().abs() if bias is not None else 0.0))


_FOLD = [("f32", 1.0, True, 1, ACT_NONE, 0.0), ("split", 1.0, True, 1, ACT_GELU, 30.0), ("split_f32_resid_stats", 1.0, True, 1, ACT_NONE, 3.0),
         ("swiglu_split_stats", 1.0, True, 1, ACT_NONE, 0.0), ("acc", 1.0, True, 3, ACT_NONE, 3.0), ("f32", 1.0, False, 1, ACT_NONE, 3.0),
         ("split", 0.5, True, 1, ACT_RELU, 3.0), ("acc", -1.0, False, 2, ACT_NONE, 3.0), ("f32", 0.125, False, 1, ACT_NONE, 30.0)]


@pytest.mark.parametrize("form,alpha,with_bias,sk,act,shift", _FOLD,
                         ids=[_id(_gk(_tile(0, 300, 256, 384, 1, k)), form=f, alpha=a, bias=int(wb), split_k=k, act=_ACTN[ac], shift=sh)
                              for (f, a, wb, k, ac, sh) in _FOLD])
def test_gemm_ln_fold(form, alpha, with_bias, sk, act, shift):
    """LayerNorm folded into the GEMM: out = act(alpha rstd (acc - mean c) + bias (+ resid)) on every output form the
    header allows (fp32, split, split + fp32 with a residual and output statistics, SwiGLU pairs with statistics,
    accumulate with split-K), with bias = NULL and alpha != 1, and a mean up to 30x the spread."""
    M, N, H = 300, 256, 384
    x = _randn((M, H), 31, shift=shift)
    wg, bias = _randn((N, H), 32, H ** -0.5), (_randn((N,), 33) if with_bias else None)
    X, Wg = Planes(x), Planes(wg)
    x64 = X.seen(3)
    st = torch.stack([x64.sum(1), (x64 * x64).sum(1)], 1).float()
    c = wg.double().sum(1).float()
    eps = 1e-6
    fields = dict(ln_stats=st.data_ptr(), ln_c=c.data_ptr(), ln_h=H, ln_eps=eps, alpha=alpha, act=act,
                  bias=bias.data_ptr() if bias is not None else None)
    acc = x64 @ Wg.seen(3).t()
    pre, rstd, mean = _fold_ref(acc, st, c, H, eps, alpha, bias)
    Epre = _fold_bound(_gemm_err(x.double(), wg.double(), H, 3), acc, st, c, H, eps, alpha, bias, pre, rstd, mean, sk)
    out, sp, stats, r, init = None, None, None, None, None
    if form in ("f32", "split_f32_resid_stats", "acc"):
        out = _nan((M, N))
        fields.update(out_f32=out.data_ptr(), ldo=N)
    if form in ("split", "split_f32_resid_stats", "swiglu_split_stats"):
        ncol = N // 2 if form.startswith("swiglu") else N
        sp = _nan((2, M, ncol), torch.bfloat16)
        fields.update(out_hi=sp.data_ptr(), out_plane=M * ncol, ldo_s=ncol)
    if form.endswith("stats"):
        stats = torch.zeros(M, 2, device=_dev())
        fields.update(stats_out=stats.data_ptr())
    if form == "split_f32_resid_stats":
        r = _randn((M, N), 34)
        out.copy_(r)
        fields.update(resid=out.data_ptr())
        pre, Epre = pre + r.double(), Epre + 2 * U * (pre.abs() + r.double().abs())
    if form == "acc":
        init = _randn((M, N), 35)
        out.copy_(init)
        fields.update(accumulate=1)
    if form.startswith("swiglu"):
        fields.update(swiglu=1)
    assert _call_gemm(X.operand(), Wg.operand(), _gemm_out(**fields), 3, sk) == 0
    torch.cuda.synchronize()
    y = _act64(pre, act)
    Ey = 1.2 * Epre + 4 * U * y.abs() + GELU_ABS * (1 + pre.abs()) if act == ACT_GELU else Epre
    if form.startswith("swiglu"):
        g, v = pre[:, 0::2], pre[:, 1::2]
        sg = torch.nn.functional.silu(g)
        y = sg * v
        Ey = 1.1 * Epre[:, 0::2] * v.abs() + sg.abs() * Epre[:, 1::2] + Epre[:, 0::2] * Epre[:, 1::2] + 8 * U * (2 + g.abs()) * y.abs()
    if init is not None:
        y, Ey = y + init.double(), Ey + 2 * U * (y.abs() + init.double().abs())
    name = f"ln_fold {form} alpha={alpha} bias={with_bias} split_k={sk} shift={shift}"
    if out is not None:
        _check_bound(name, out, y, Ey)
    if sp is not None:
        if out is not None:
            _assert_split_is(sp[0], sp[1], out, name)
        else:
            _check_bound(name + " split", sp[0].float() + sp[1].float(), y, Ey + SPLIT * y.abs())
    if stats is not None:
        yk = out.double() if out is not None else sp[0].double() + sp[1].double()
        depth = 6 + yk.shape[1] // 32
        extra = 0.0 if out is not None else 1.0
        _check_bound(name + " stats sum", stats[:, 0], yk.sum(1), depth * U * yk.abs().sum(1) + extra * 2.0 ** -17 * yk.abs().sum(1) + 1e-30)
        _check_bound(name + " stats sum sq", stats[:, 1], (yk * yk).sum(1),
                     (depth + 1) * U * (yk * yk).sum(1) + extra * 2.0 ** -16 * (yk * yk).sum(1) + 1e-30)


# ------------------------------------------------------------------------------------------------
# psam_gemm_rowln_bf16x3
# ------------------------------------------------------------------------------------------------
_RL = [(N, K, [ACT_NONE, ACT_GELU, ACT_RELU][(i + j) % 3], (1, 3)[(i + j) % 2], [1, 7, 64][(i + 2 * j) % 3],
        [300, 128 * 132 * 2 + 5, 1000, 129][(i + j) % 4]) for i, N in enumerate((256, 512)) for j, K in enumerate((1, 17, 64, 65, 128))]


def _rowln_bound(x, E, g, b, y_pre, rstd, act):
    """Two-pass fp32 LayerNorm of N-wide rows x (the glue file's form), plus the GEMM error E of x passed through the
    normalisation: |g| rstd max_row(E) (2 + |x_hat|) for the shifted mean and the changed variance."""
    N = x.shape[-1]
    inmag = x.abs().amax(-1, keepdim=True)
    xh = (x - x.mean(-1, keepdim=True)) * rstd
    bound = 4 * U * math.sqrt(N) * g.abs() * rstd * inmag + 4 * U * (y_pre.abs() + b.abs())
    bound = bound + g.abs() * rstd * E.amax(-1, keepdim=True) * (2 + xh.abs())
    return 1.2 * bound + GELU_ABS * (1 + y_pre.abs()) if act == ACT_GELU else bound


@pytest.mark.parametrize("N,K,act,passes,group_rows,M", _RL,
                         ids=[_id("gemm_rowln_kernel", N=N, K=K, act=_ACTN[a], passes=p, group_rows=g, M=M) for (N, K, a, p, g, M) in _RL])
def test_gemm_rowln(N, K, act, passes, group_rows, M):
    """act(LayerNorm(A W^T + gbias[row / group_rows])) as split-bf16: W resident (N = 256) and the 0, 1, 0 halves (N = 512),
    K tails, ldo_s > N and ld_gbias > N, a group bias 30x the spread, and more m-tiles than SMs."""
    a, w = _randn((M, K), 41), _randn((N, K), 42, K ** -0.5)
    gamma, beta = _randn((N,), 43, 0.1, 1.0), _randn((N,), 44, 0.1)
    G = -(-M // group_rows)
    ldg = N + 12
    gb = _nan((G, ldg))
    gb[:, :N] = _randn((G, N), 45, shift=30.0)
    A, W = Planes(a), Planes(w, extra_rows=0)
    ldo_s = N + 64
    sp = _nan((2, M + 1, ldo_s), torch.bfloat16)
    nv = _nv()
    ao, wo = A.operand(), W.operand()
    rc = nv.lib().psam_gemm_rowln_bf16x3(byref(ao), byref(wo), gb.data_ptr(), ldg, group_rows, gamma.data_ptr(), beta.data_ptr(),
                                         1e-5, act, sp.data_ptr(), sp[0].numel(), ldo_s, passes, nv.stream())
    assert rc == 0
    torch.cuda.synchronize()
    a64, w64 = a.double(), w.double()
    gbr = gb[:, :N].double().repeat_interleave(group_rows, 0)[:M]
    x = a64 @ w64.t() + gbr
    E = _gemm_err(a64, w64, K, passes) + 2 * U * x.abs()
    y_pre = torch.nn.functional.layer_norm(x, (N,), gamma.double(), beta.double(), 1e-5)
    rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    want = _act64(y_pre, act)
    bound = _rowln_bound(x, E, gamma.double(), beta.double(), y_pre, rstd, act) + SPLIT * want.abs()
    _check_bound(f"rowln N={N} K={K} act={_ACTN[act]} passes={passes} M={M}", sp[0, :M, :N].float() + sp[1, :M, :N].float(), want, bound)
    mask = torch.zeros_like(sp, dtype=torch.bool)
    mask[:, :M, :N] = True
    _only_window(sp, mask, "rowln")


# ------------------------------------------------------------------------------------------------
# psam_attention_bf16x3 / _twopass
# ------------------------------------------------------------------------------------------------
_ATT_KERNELS = [(64, False), (88, False), (64, True)]
_L = [1, 63, 64, 65, 127, 128, 129, 200, 1100]
_ATT = [(dh, tp, L, (2, 1, 3)[(i + j) % 3], (3, 2, 1)[(i + 2 * j) % 3], ("inv_sqrt", 1.0, 0.01)[(i + j) % 3])
        for i, (dh, tp) in enumerate(_ATT_KERNELS) for j, L in enumerate(_L)]


def _ak(dh, tp):
    return f"attention_wgmma_kernel<{dh}, {'true' if tp else 'false'}>"


class _AttnIO:
    """Q in [B][L][H * dh + 8] (head h at column h dh), K in [B][H][L + 3][pitch_k], V in [H][B][L + 1][pitch_v], all split-bf16
    with NaN in every row and column the operand views do not cover; the output in [B][H][L + 2][ldo] (ldo = dh + 40) with
    64 elements between clouds, NaN outside the window."""

    def __init__(self, q, k, v, B, H, L, dh):
        self.B, self.H, self.L, self.dh = B, H, L, dh
        nv = _nv()
        pq, pk, pv = H * dh + 8, dh + 24, dh + 56
        self.Qt = _nan((2, B, L, pq), torch.bfloat16)
        self.Kt = _nan((2, B, H, L + 3, pk), torch.bfloat16)
        self.Vt = _nan((2, H, B, L + 1, pv), torch.bfloat16)
        for p, (qq, kk, vv) in enumerate(zip(_split_of(q), _split_of(k), _split_of(v))):   # q, k, v: [B, H, L, dh] fp32
            self.Qt[p, :, :, :H * dh] = qq.transpose(1, 2).reshape(B, L, H * dh)
            self.Kt[p, :, :, :L, :dh] = kk
            self.Vt[p, :, :, :L, :dh] = vv.transpose(0, 1)
        self.qo = nv.Operand(self.Qt.data_ptr(), self.Qt[0].numel(), L, dh, pq, H, B, dh, L * pq)
        self.ko = nv.Operand(self.Kt.data_ptr(), self.Kt[0].numel(), L, dh, pk, H, B, (L + 3) * pk, H * (L + 3) * pk)
        self.vo = nv.Operand(self.Vt.data_ptr(), self.Vt[0].numel(), L, dh, pv, H, B, B * (L + 1) * pv, (L + 1) * pv)
        self.ldo = dh + 40
        self.oh, self.ob = (L + 2) * self.ldo, H * (L + 2) * self.ldo + 64
        self.plane = B * self.ob
        self.out = _nan((2, self.plane), torch.bfloat16)

    def seen(self):
        """The operands the kernel multiplies (hi + lo), fp64 [B, H, L, dh]."""
        B, H, L, dh = self.B, self.H, self.L, self.dh
        q = self.Qt[:, :, :, :H * dh].double().sum(0).view(B, L, H, dh).transpose(1, 2)
        return q, self.Kt[:, :, :, :L, :dh].double().sum(0), self.Vt[:, :, :, :L, :dh].double().sum(0).transpose(0, 1)

    def run(self, entry, scale):
        nv = _nv()
        return getattr(nv.lib(), entry)(byref(self.qo), byref(self.ko), byref(self.vo), self.out.data_ptr(), self.plane, self.ldo,
                                        self.oh, self.ob, scale, nv.stream())

    def window(self, t):
        B, H, L, dh = self.B, self.H, self.L, self.dh
        return t.view(t.shape[0], B, self.ob)[:, :, :H * self.oh].view(t.shape[0], B, H, L + 2, self.ldo)[:, :, :, :L, :dh]

    def planes(self):
        torch.cuda.synchronize()
        mask = torch.zeros_like(self.out, dtype=torch.bool)
        self.window(mask).fill_(True)
        _only_window(self.out, mask, "attention output")
        w = self.window(self.out)
        return w[0], w[1]


def _att_ref(q, k, v, scale):
    s = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(s, -1)
    return p @ v, s, p


def _att_bound(q, k, v, scale, s, p, o):
    """Score errors (split-bf16 products and an fp32 dot product of dh terms, then the scale folded into exp2) move each
    probability by twice the largest of them; ex2.approx and the exponent's rounding add a relative error growing with
    the logit spread; P is split into bf16 hi + lo and multiplied by split V (the C1 2^-16 term), the sums over keys
    sqrt(L) u; all relative to sum_j p_j |v_j|.  Plus the split of the output."""
    dh, L = q.shape[-1], k.shape[-2]
    sabs = q.abs() @ k.abs().transpose(-1, -2) * scale
    ds = ((C1 * 2.0 ** -16 + C2 * math.sqrt(dh) * U) * sabs + 2 * U * s.abs()).amax(-1, keepdim=True)
    m = s.amax(-1, keepdim=True)
    spread = m - s.amin(-1, keepdim=True)
    rel = 2 * ds + 2 * EX2 + 8 * U * (2 + m.abs() + spread) + C1 * 2.0 ** -16 + C2 * math.sqrt(L) * U
    return rel * (p @ v.abs()) + SPLIT * o.abs() + 1e-30


def _scale(sc, dh):
    return dh ** -0.5 if sc == "inv_sqrt" else sc


@pytest.mark.parametrize("dh,twopass,L,B,H,sc", _ATT, ids=[_id(_ak(dh, tp), L=L, B=B, H=H, scale=sc) for (dh, tp, L, B, H, sc) in _ATT])
def test_attention(dh, twopass, L, B, H, sc):
    """Random Q, K, V in three buffers of different pitches and layouts, the output in a [B, H, L, dh] layout with padded
    strides, against fp64 with a stated bound; then one-hot scores that must return split(float(V)[peak]) bit for bit,
    with the peaks in the first key block, a middle block, the last block and at key L - 1."""
    entry = "psam_attention_bf16x3_twopass" if twopass else "psam_attention_bf16x3"
    scale = _scale(sc, dh)
    q, k, v = _randn((B, H, L, dh), 51), _randn((B, H, L, dh), 52), _randn((B, H, L, dh), 53)
    io = _AttnIO(q, k, v, B, H, L, dh)
    assert io.run(entry, scale) == 0
    hi, lo = io.planes()
    qs, ks, vs = io.seen()
    o, s, p = _att_ref(qs, ks, vs, scale)
    _check_bound(f"attention {_ak(dh, twopass)} L={L} B={B} H={H} scale={scale:.4g}", hi.float() + lo.float(), o,
                 _att_bound(qs, ks, vs, scale, s, p, o))
    # one-hot: query i peaks at key t[i % 4] through column i % 4 (q = 2^14 there, k = 1 at the peak key only); the peak
    # keys have no other non-zero column, so the peak score is exactly 2^14 and its exponent exactly 0; every other key
    # scores |r| <= 3.75 from columns 4.. (small dyadic values), >= 128 below the peak after any of the scales
    nkb = -(-L // 64)
    t = [min(5, L - 1), min((nkb // 2) * 64 + 3, L - 1), min((nkb - 1) * 64 + 1, L - 1), L - 1]
    g = _gen(54)
    qr = torch.randint(-2, 3, (B, H, L, dh), generator=g).float() / 8
    kr = torch.randint(-2, 3, (B, H, L, dh), generator=g).float() / 8
    qr[..., :4], kr[..., :4] = 0.0, 0.0
    for d in range(4):
        qr[:, :, d::4, d] = 2.0 ** 14
    kr[:, :, t] = 0.0
    for d in range(4):
        kr[:, :, t[d], d] = 1.0
    io1 = _AttnIO(qr.to(_dev()), kr.to(_dev()), v, B, H, L, dh)
    assert io1.run(entry, scale) == 0
    hi1, lo1 = io1.planes()
    vs1 = io1.seen()[2]
    peak = torch.tensor([t[i % 4] for i in range(L)], device=_dev())
    sel = vs1[:, :, peak].float()
    _assert_split_is(hi1, lo1, sel, f"one-hot {_ak(dh, twopass)} L={L}")


# ------------------------------------------------------------------------------------------------
# the bounds have teeth
# ------------------------------------------------------------------------------------------------
def _wrong_accs(a, w, K, bk=64):
    """fp64 a @ w^T (a, w exact fp32 values), and three wrong versions of it: the lo passes of the first k-block dropped,
    the last K column dropped, one output row shifted."""
    ah, wh = a.float().to(torch.bfloat16).double(), w.float().to(torch.bfloat16).double()
    acc = a @ w.t()
    kb = slice(0, min(bk, K))
    no_lo = acc - a[:, kb] @ w[:, kb].t() + ah[:, kb] @ wh[:, kb].t()
    no_last = acc - a[:, K - 1:] @ w[:, K - 1:].t()
    shifted = acc.clone()
    shifted[0] = acc[1]
    return acc, {"lo_passes_of_one_k_block_dropped": no_lo, "last_k_column_dropped": no_last, "one_row_shifted": shifted}


@pytest.mark.parametrize("family", ["gemm_passes3", "gemm_passes1", "split_k", "ln_fold", "rowln", "attention"])
def test_bounds_have_teeth(family):
    """Each family's bound, applied to a deliberately wrong fp64 result built on the host, must reject it (no kernel runs)."""
    M, N, K = 300, 200, 64
    a, w, b = _randn((M, K), 61).double(), _randn((N, K), 62, K ** -0.5).double(), _randn((N,), 63).double()
    acc, wrongs = _wrong_accs(a, w, K)
    if family == "gemm_passes1":
        wrongs.pop("lo_passes_of_one_k_block_dropped")   # that is what passes = 1 computes
    for name, bad in wrongs.items():
        if family.startswith("gemm"):
            passes = 3 if family == "gemm_passes3" else 1
            pre = acc + b
            bound = 1.2 * (_gemm_err(a, w, K, passes) + 2 * U * pre.abs()) + GELU_ABS * (1 + pre.abs())
            _rejects(f"{family} {name}", _act64(bad + b, ACT_GELU), _act64(pre, ACT_GELU), bound)
        elif family == "split_k":
            init = _randn((M, N), 64).double()
            want = init + acc + b
            sk = 7
            bound = _gemm_err(a, w, K, 3) + (sk + 2) * U * (want.abs() + init.abs() + b.abs() + a.abs() @ w.abs().t())
            _rejects(f"{family} {name}", init + bad + b, want, bound)
        elif family == "ln_fold":
            x = _randn((M, K), 65, shift=3.0).double()
            accx, wx = _wrong_accs(x, w, K)
            st = torch.stack([x.sum(1), (x * x).sum(1)], 1).float()
            c = w.sum(1).float()
            pre, rstd, mean = _fold_ref(accx, st, c, K, 1e-6, 0.5, b.float())
            bound = _fold_bound(_gemm_err(x, w, K, 3), accx, st, c, K, 1e-6, 0.5, b.float(), pre, rstd, mean, 1)
            badpre = _fold_ref(wx[name], st, c, K, 1e-6, 0.5, b.float())[0]
            _rejects(f"{family} {name}", badpre, pre, bound)
            if name != "one_row_shifted":
                continue
            # and the two forms the LayerNorm fold used to compute: the mean term dropped without a bias, unscaled by alpha
            nob = _fold_ref(accx, st, c, K, 1e-6, 0.5, None)[0]
            _rejects(f"{family} mean term dropped", nob + mean * rstd * 0.5 * c.double(), nob,
                     _fold_bound(_gemm_err(x, w, K, 3), accx, st, c, K, 1e-6, 0.5, None, nob, rstd, mean, 1))
            _rejects(f"{family} mean term not scaled by alpha", pre - 0.5 * mean * rstd * c.double(), pre, bound)
        elif family == "rowln":
            Nr = 256
            wr = _randn((Nr, K), 66, K ** -0.5).double()
            gamma, beta = _randn((Nr,), 67, 0.1, 1.0).double(), _randn((Nr,), 68, 0.1).double()
            accr, wrr = _wrong_accs(a, wr, K)
            x = accr + 30.0
            y = torch.nn.functional.layer_norm(x, (Nr,), gamma, beta, 1e-5)
            rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
            E = _gemm_err(a, wr, K, 3) + 2 * U * x.abs()
            bound = _rowln_bound(x, E, gamma, beta, y, rstd, ACT_NONE) + SPLIT * y.abs()
            _rejects(f"{family} {name}", torch.nn.functional.layer_norm(wrr[name] + 30.0, (Nr,), gamma, beta, 1e-5), y, bound)
        else:
            B, H, L, dh = 1, 2, 64, 64   # one key block; small scores, so the output's error is not dominated by theirs
            q, k, v = (_randn((B, H, L, dh), 69 + i, 0.1 if i < 2 else 1.0).double() for i in range(3))
            scale = dh ** -0.5
            o, s, p = _att_ref(q, k, v, scale)
            bound = _att_bound(q, k, v, scale, s, p, o)
            if name == "lo_passes_of_one_k_block_dropped":
                bad = p @ v.float().to(torch.bfloat16).double()       # P V with the lo plane of V dropped (all keys: one block)
            elif name == "last_k_column_dropped":
                bad = torch.softmax(s[..., :L - 1], -1) @ v[:, :, :L - 1]   # the last key dropped
            else:
                bad = o.clone()
                bad[:, :, 0] = o[:, :, 1]
            _rejects(f"{family} {name}", bad, o, bound)


# ------------------------------------------------------------------------------------------------
# refusals, with real device buffers
# ------------------------------------------------------------------------------------------------
def _refusal_gemm_case(case):
    M, N, K = 256, 128, 64
    A, W = Planes(_ints((M, K), -8, 8, 81)), Planes(_ints((N if case != "swiglu_odd_n" else 127, K), -4, 4, 82))
    out, out2 = torch.zeros(M, N, device=_dev()), torch.zeros(M, N, device=_dev())
    sp = torch.zeros(2, M, N, dtype=torch.bfloat16, device=_dev())
    gmax = torch.full((M // 32, N), float("-inf"), device=_dev())
    rd_w, rd_out = torch.zeros(3, 9, N, device=_dev()), torch.zeros(3, 9, M, device=_dev())
    stats = torch.zeros(M, 2, device=_dev())
    f32 = dict(out_f32=out.data_ptr(), ldo=N)
    spl = dict(out_hi=sp.data_ptr(), out_plane=M * N, ldo_s=N)
    sk = 1
    f = {"accumulate_with_split_output": dict(accumulate=1, **f32, **spl),
         "accumulate_with_gelu": dict(accumulate=1, act=ACT_GELU, **f32),
         "accumulate_with_relu": dict(accumulate=1, act=ACT_RELU, **f32),
         "accumulate_with_other_resid": dict(accumulate=1, resid=out2.data_ptr(), **f32),
         "rowdot_rows_not_multiple_of_32": dict(rd_w=rd_w.data_ptr(), rd_out=rd_out.data_ptr(), rd_rows=M // 2 + 16, rd_c=2),
         "rowdot_nine_vectors": dict(rd_w=rd_w.data_ptr(), rd_out=rd_out.data_ptr(), rd_rows=M, rd_c=9),
         "gmax_with_resid": dict(gmax=gmax.data_ptr(), ld_gmax=N, group_rows=32, resid=out2.data_ptr(), **f32),
         "gmax_with_act": dict(gmax=gmax.data_ptr(), ld_gmax=N, group_rows=32, act=ACT_RELU),
         "swiglu_odd_n": dict(swiglu=1, **f32),
         "stats_out_with_split_k": dict(stats_out=stats.data_ptr(), accumulate=1, **f32)}[case]
    if case == "stats_out_with_split_k":
        sk = 2
    return A, W, f, sk


_REFUSE_GEMM = ["accumulate_with_split_output", "accumulate_with_gelu", "accumulate_with_relu", "accumulate_with_other_resid",
                "rowdot_rows_not_multiple_of_32", "rowdot_nine_vectors", "gmax_with_resid", "gmax_with_act", "swiglu_odd_n",
                "stats_out_with_split_k"]


@pytest.mark.parametrize("case", _REFUSE_GEMM)
def test_gemm_refusals(case):
    """Combinations the epilogues would mis-compute are refused with PSAM_ERR_ARG (real, correctly sized buffers)."""
    A, W, f, sk = _refusal_gemm_case(case)
    assert _call_gemm(A.operand(), W.operand(), _gemm_out(**f), 3, sk) == ERR_ARG


_REFUSE_ATT = [("k_fewer_heads", 0.125), ("v_fewer_clouds", 0.125), ("scale_zero", 0.0), ("scale_negative", -0.125),
               ("scale_nan", float("nan")), ("scale_inf", float("inf"))]


@pytest.mark.parametrize("entry", ["psam_attention_bf16x3", "psam_attention_bf16x3_twopass"])
@pytest.mark.parametrize("case,scale", _REFUSE_ATT, ids=[c for c, _ in _REFUSE_ATT])
def test_attention_refusals(case, scale, entry):
    """K or V covering fewer heads or clouds than Q (TMA would fill zeros for the rest), and a scale that is not finite
    and > 0 (the kernels subtract the maximum of the unscaled scores), are refused with PSAM_ERR_ARG."""
    B, H, L, dh = 2, 2, 128, 64
    io = _AttnIO(_randn((B, H, L, dh), 91), _randn((B, H, L, dh), 92), _randn((B, H, L, dh), 93), B, H, L, dh)
    if case == "k_fewer_heads":
        io.ko.nb1 = 1
    if case == "v_fewer_clouds":
        io.vo.nb2 = 1
    assert io.run(entry, scale) == ERR_ARG
    torch.cuda.synchronize()
    assert bool(torch.isnan(io.out.float()).all())


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


def test_routing_guard():
    """One call per instantiation (the forced tile widths, choose_bn's picks under both policies, the row-LN GEMM, the three
    attention kernels) under the profiler; the kernel that ran must be the one the case ids above name.  It runs in a fresh
    interpreter: after the rest of the suite has run in this process, the profiler has been seen to record no CUDA activity
    at all, and what the guard sees must not depend on what ran before it."""
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_tc_kernels as t; t._routing_guard()" % (
        here, repo, os.path.join(repo, "point-sam_b200"))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def _routing_guard():
    nv = _nv()
    calls = []
    keep = []
    for (M, N, K, hint) in [(300, 200, 200, 64), (300, 200, 200, 128), (300, 200, 200, 256), (32768 + 5, 1024, 200, 0),
                            (32768 + 5, 1024, 200, 1), (300, 1024, 2730, 0), (128, 31, 64, 0), (1, 1024, 65, 1)]:
        A, W = Planes(_randn((M, K), 1)), Planes(_randn((N, K), 2))
        out = torch.empty(M, N, device=_dev())
        o = _gemm_out(out_f32=out.data_ptr(), ldo=N, tile_hint=hint)
        keep += [A, W, out]
        calls.append((_gk(_tile(hint, M, N, K)), lambda A=A, W=W, o=o: _call_gemm(A.operand(), W.operand(), o, 3, 1)))
    A, W = Planes(_randn((300, 64), 3)), Planes(_randn((256, 64), 4))
    gamma = torch.ones(256, device=_dev())
    sp = torch.empty(2, 300, 256, dtype=torch.bfloat16, device=_dev())
    keep += [A, W, gamma, sp]
    ao, wo = A.operand(), W.operand()
    calls.append(("gemm_rowln_kernel", lambda: nv.lib().psam_gemm_rowln_bf16x3(byref(ao), byref(wo), None, 0, 0, gamma.data_ptr(),
                                                                             gamma.data_ptr(), 1e-5, 0, sp.data_ptr(), sp[0].numel(),
                                                                             256, 3, nv.stream())))
    for dh, tp in _ATT_KERNELS:
        io = _AttnIO(_randn((1, 2, 200, dh), 5), _randn((1, 2, 200, dh), 6), _randn((1, 2, 200, dh), 7), 1, 2, 200, dh)
        keep.append(io)
        calls.append((_ak(dh, tp), lambda io=io, tp=tp: io.run("psam_attention_bf16x3_twopass" if tp else "psam_attention_bf16x3", 0.125)))
    rcs = []
    names = _kernels_launched(lambda: rcs.extend(fn() for _, fn in calls))
    assert rcs == [0] * len(calls), f"return codes {rcs}"
    assert len(names) == len(calls), f"{len(calls)} calls launched {len(names)} kernels: {names}"
    for (want, _), got in zip(calls, names):
        assert want + ("(" if "<" not in want else "") in got, f"expected {want}, ran {got}"
    print(f"[tc] routing guard: {len(calls)} calls, each ran the kernel its case id names")
