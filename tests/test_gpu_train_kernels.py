"""The fine-tuning kernels - the mask loss statistics and gradient, the inverse interpolation index, the head's elementwise
backward, the LayerNorm and interpolation backward, and the fixed-order partial sums (csrc/train.cu) - through the C ABI on
every launch path of their host functions, and the chunked head backward (psam_b200.train.head_backward) on every chunk
plan.

Each kernel is compared with a plain reference of the same operation: bit for bit where the header fixes the arithmetic
(counts, the inverse index as np.bincount + a stable argsort, the partial sums as a sequential fp64 loop over s), and
otherwise against fp64 within a bound derived next to each test from the fp32 operations the kernel performs.  Every
output sits inside a sentinel window (test_gpu_amg_kernels.Win) compared whole: dp's pitch padding and the gap between its
planes, offsets[B, G+1], the partial buffers.  Logits include +-0.0, subnormals, +-100 and +-1e4; LayerNorm rows include a
large common offset, near-constant rows and points whose three neighbours are one patch, with an eps of the order of the
rows' variance so that dropping or replacing it shows.

Every case id names the launch path it reaches, from the host dispatch restated below; test_routing_guard checks those
names, the fused or separate mask product of the forward, and the chunk plans of the head backward under torch.profiler."""
import itertools
import math
import os

import numpy as np
import pytest
import torch
from scipy.special import erf, expit

from test_gpu_amg_kernels import FSENT, GUARD, SENT, Win, _cmp, _id, _kernels_launched  # noqa: F401

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24            # fp32 unit roundoff
NAN, INF = float("nan"), float("inf")
BF_SENT = 0x7F7F          # sentinel of bf16 windows (a finite 3.4e38)


def _nv():
    from psam_b200 import native as nv

    return nv


def _dev():
    return torch.device("cuda:0")


def _cdiv(a, b):
    return -(-a // b)


def _np(t):
    return t.detach().cpu().numpy()


def _ok(err, bound, name):
    """err <= bound everywhere (both fp64 arrays); returns the worst err / bound."""
    bad = ~(err <= bound)
    if bad.any():
        at = np.argwhere(bad)[:4]
        raise AssertionError(f"{name}: {int(bad.sum())} of {err.size} entries past the bound, first at {at.tolist()}: "
                             f"err {[err[tuple(i)] for i in at]} bound {[bound[tuple(i)] for i in at]}")
    r = err / np.maximum(bound, 1e-300)
    return float(r.max()) if r.size else 0.0


def _report(name, ratio):
    print(f"[train kernels] {name}: worst err/bound {ratio:.3g}")


# ------------------------------------------------------------------------------------------------
# the host dispatch, restated (test_routing_guard checks it against the kernels that run)
# ------------------------------------------------------------------------------------------------
LOSS_GRID_CAP = 64        # blocks_for(N, 256, 64) of psam_mask_loss_grad
SUM_GRID_CAP = 132 * 32   # blocks_for(nb * n, 256) of psam_sum_partials
HEAD_RB = 128             # points per CTA of head_dp_kernel


def loss_grid(N):
    return min(max(_cdiv(N, 256), 1), LOSS_GRID_CAP)


def ln_kernel(D):
    return f"interp_ln_gelu_bwd_kernel<{D // 128}>"


def ib_kernel(D):
    return f"interp_bwd_kernel<{D // 128}>"


def sum_grid(nb, n):
    return min(max(_cdiv(nb * n, 256), 1), SUM_GRID_CAP)


def head_plan(Z, rep, N, backward_rows, dw_split_k):
    """head_backward's chunks (cloud, z0, z1) and, per chunk, _dw3_partials' (S, Kc, Kp)."""
    zc = max(1, min(rep, backward_rows // N))
    chunks = [(b, z0, min((b + 1) * rep, z0 + zc)) for b in range(Z // rep) for z0 in range(b * rep, (b + 1) * rep, zc)]
    splits = []
    for _, z0, z1 in chunks:
        R = (z1 - z0) * N
        S = max(1, _cdiv(R, dw_split_k))
        Kc = _cdiv(_cdiv(R, S), 64) * 64
        splits.append((S, Kc, S * Kc))
    return chunks, splits


# ------------------------------------------------------------------------------------------------
# 1. mask loss: psam_mask_loss_stats / psam_mask_loss_grad
# ------------------------------------------------------------------------------------------------
LOSS_SHAPES = [(1, 1, 7), (1, 3, 5), (21845, 3, 4)] + [(2, 3, N) for N in (1, 255, 256, 257, 16384, 16385, 100000)]
SPECIAL = np.array([0.0, -0.0, 1e-45, 1e-40, -1e-45, -1e-40, 100.0, -100.0, 1e4, -1e4], F32)


def _loss_inputs(Z, C, N, seed):
    """Logits with the special values, whole rows inside / outside against an empty and a full gt, and dloss with +0.0 /
    -0.0 rows that hold NaN and +-inf logits."""
    g = np.random.default_rng(seed)
    x = (g.standard_normal((Z, C, N)) * 4).astype(F32)
    at = g.random((Z, C, N)) < 0.3
    x[at] = SPECIAL[g.integers(0, len(SPECIAL), int(at.sum()))]
    gt = g.random((Z, N)) < 0.4
    gt[0] = False
    x[0, 0] = np.abs(x[0, 0]) + F32(0.5)                 # all inside, empty gt
    if C > 1:
        x[0, C - 1] = -np.abs(x[0, C - 1]) - F32(0.5)    # all outside, empty gt
    if Z > 1:
        gt[-1] = True
        x[-1, 0] = -np.abs(x[-1, 0]) - F32(0.5)          # all outside, full gt
        x[-1, C - 1] = np.abs(x[-1, C - 1]) + F32(0.5)   # all inside, full gt (C = 1: this one)
    up = g.standard_normal((Z, C)).astype(F32)
    flat, xf = up.reshape(-1), x.reshape(Z * C, N)
    zero = [i for i in range(1, Z * C, 7)][:4000] if Z * C > 1 else []
    for j, i in enumerate(zero):
        flat[i] = 0.0 if j % 2 == 0 else -0.0
        xf[i, g.integers(0, N, max(1, N // 5))] = np.array([NAN, INF, -INF], F32)[j % 3]
    return x, gt, up, zero


def _loss_ref(x, gt):
    """fp64 terms of every logit, in the stable forms (BCE = max(x, 0) - x t + log1p(exp(-|x|)), 1 - p_t = sigmoid(-+x))."""
    Z, C, N = x.shape
    xd = x.astype(np.float64)
    t = np.broadcast_to(gt[:, None, :], x.shape).astype(np.float64)
    with np.errstate(all="ignore"):
        p, pn = expit(xd), expit(-xd)
        q = np.where(t > 0, pn, p)
        ce = np.maximum(xd, 0.0) - xd * t + np.log1p(np.exp(-np.abs(xd)))
        stats = np.stack([(ce * q * q).sum(-1), (p * t).sum(-1), (p * p).sum(-1), t.sum(-1)], -1)
    pred = x > 0
    gb = np.broadcast_to(gt[:, None, :], x.shape)
    counts = np.stack([(pred & gb).sum(-1), (pred | gb).sum(-1)], -1).astype(np.int32)
    return dict(p=p, s=p * pn, q=q, ce=ce, t=t, stats=stats, counts=counts)


def _loss_id(Z, C, N):
    gx = loss_grid(N)
    return _id("mask_loss_grad_kernel", ZC=Z * C, N=N, grid=f"{gx}x{Z * C}", loop=int(gx * 256 < N))


@pytest.mark.parametrize("Z,C,N", LOSS_SHAPES, ids=[_loss_id(*s) for s in LOSS_SHAPES])
def test_mask_loss_stats_and_grad(Z, C, N):
    """counts bit-exact; each stat within 2 fp32 ulps of the fp64 sum (the kernel sums non-negative fp64 terms and rounds
    once); each dlogit within a per-element bound; rows with dloss = +-0.0 come back as +0.0 whatever their logits."""
    nv = _nv()
    L = nv.lib()
    x, gt, up, zero = _loss_inputs(Z, C, N, seed=Z * 7 + C * 131 + N)
    xw = Win(torch.from_numpy(x))
    gw = Win(torch.from_numpy(gt.astype(np.uint8)), fill=0x7F)
    uw = Win(torch.from_numpy(up))
    sw = Win(shape=(Z, C, 4), dtype=torch.float32)
    cw = Win(shape=(Z, C, 2), dtype=torch.int32)
    dw = Win(shape=(Z, C, N), dtype=torch.float32)
    assert L.psam_mask_loss_stats(xw.ptr, gw.ptr, Z, C, N, sw.ptr, cw.ptr, nv.stream()) == 0
    assert L.psam_mask_loss_grad(xw.ptr, gw.ptr, Z, C, N, sw.ptr, uw.ptr, dw.ptr, nv.stream()) == 0
    for w, n in ((sw, "stats"), (cw, "counts"), (dw, "dlogits"), (xw, "logits"), (uw, "dloss")):
        w.check(n)
    ref = _loss_ref(x, gt)
    _cmp(cw.cpu(), torch.from_numpy(ref["counts"]), "counts")
    st = _np(sw.t).astype(np.float64)
    want = ref["stats"]
    fin = np.isfinite(want)
    assert not np.isfinite(st[~fin]).any(), "stats: a row with non-finite logits gave a finite sum"
    ulp = np.spacing(np.abs(want[fin]).astype(F32)).astype(np.float64)
    r_st = _ok(np.abs(st[fin] - want[fin]), 2 * ulp, "stats")
    # dlogit = up (dfocal / N + ddice), ddice = 2 (t1 - t2) s with t1 = 2 A p / Bd^2, t2 = 2 t / Bd, A = 2 pt + 1e-3,
    # Bd = pp + ts + 1e-3.  The kernel evaluates it in fp64 from the fp32 stats: A and Bd carry the stats' rounding
    # (delta <= 2 ulp <= 4u, as asserted above; sums of non-negative terms), so t1 (A / Bd^2) is off by at most 3 delta = 12u
    # and t2 (1 / Bd) by 4u; the final store adds u/2 of the result.  dfocal is fp64 throughout.  Hence
    #   |err| <= 13 u |up| (|dfocal| / N + 2 s (|t1| + |t2|))   (12.5 rounded up),
    # plus half the fp32 subnormal spacing where the result is tiny.  t1 and t2 are kept apart: they cancel where p ~ t.
    with np.errstate(all="ignore"):
        p, s, q, ce, t = ref["p"], ref["s"], ref["q"], ref["ce"], ref["t"]
        dq = np.where(t > 0, -s, s)
        dfocal = (p - t) * q * q + 2 * ce * q * dq
        A = 2 * want[..., 1] + 1e-3
        Bd = want[..., 2] + want[..., 3] + 1e-3
        t1 = 2 * A[..., None] * p / (Bd[..., None] ** 2)
        t2 = 2 * t / Bd[..., None]
        upd = up.astype(np.float64)[..., None]
        dl = upd * (dfocal / N + 2 * (t1 - t2) * s)
        bound = 13 * U * np.abs(upd) * (np.abs(dfocal) / N + 2 * s * (np.abs(t1) + np.abs(t2))) + 2.0 ** -150
    got = _np(dw.t).astype(np.float64)
    live = np.ones((Z * C,), bool)
    live[zero] = False
    live = live.reshape(Z, C)
    r_dl = _ok(np.abs(got[live] - dl[live]), bound[live], "dlogits")
    if zero:  # dloss == +-0.0: exact +0.0, NaN and inf logits notwithstanding
        zz = np.array(zero)
        _cmp(dw.cpu().view(Z * C, N)[zz], torch.zeros(len(zz), N), "dlogits of dloss == 0 rows", raw=True)
    _report(f"mask_loss Z*C={Z * C} N={N}", max(r_st, r_dl))


def _crit_case(seed):
    g = np.random.default_rng(seed)
    Z, C, N = 6, 3, 3000
    x = (g.standard_normal((Z, C, N)) * 3).astype(F32)
    at = g.random((Z, C, N)) < 0.2
    x[at] = SPECIAL[g.integers(0, len(SPECIAL), int(at.sum()))]
    gt = g.random((Z, N)) < 0.4
    gt[0] = False
    gt[-1] = True
    return torch.from_numpy(x), torch.from_numpy(gt)


@pytest.mark.parametrize("soft", [False, True], ids=["hard_iou", "soft_iou"])
def test_criterion_with_signed_zero_and_subnormal_logits(soft):
    """Criterion (and Criterion(use_soft_iou=True)) over two iterations against oracle.train_ref.criterion in fp64, with
    logits of +-0.0 and +-subnormals, where the hard IoU's logit > 0 decides."""
    from oracle import train_ref
    from pc_sam.model.loss import Criterion

    dev = _dev()
    x, gt = _crit_case(11 + soft)
    Z, C, _ = x.shape
    ipd = torch.rand(Z, C, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    x1 = x[:, :1].clone()
    x1[:, :, ::3] = torch.tensor([0.0, -0.0, 1e-45])[torch.arange(x1[:, :, ::3].numel()) % 3].view(x1[:, :, ::3].shape)
    outs_d = [dict(masks=x.double().requires_grad_(True), iou_preds=ipd), dict(masks=x1.double().requires_grad_(True), iou_preds=ipd[:, :1])]
    wl, wa = train_ref.criterion(outs_d, gt, use_soft_iou=soft)
    wl.backward()
    xs = [x.to(dev).requires_grad_(True), x1.to(dev).requires_grad_(True)]
    outs_c = [dict(masks=xs[0], iou_preds=ipd.float().to(dev)), dict(masks=xs[1], iou_preds=ipd[:, :1].float().to(dev))]
    gl, ga = Criterion(use_soft_iou=soft)(outs_c, gt.to(dev))
    gl.backward()
    assert abs(float(gl) - float(wl)) <= 1e-5 * abs(float(wl)), (float(gl), float(wl))
    for a, b in zip(ga, wa):
        # the hard IoU: integer counts of logit > 0 (-0.0 and +0.0 outside, +1e-45 inside), one fp32 division
        _cmp(a["iou"].cpu(), b["iou"].float(), "iou")
        assert torch.equal(a["best_masks"].detach().cpu(), b["best_masks"].detach().float())
        assert abs(float(a["loss_iou"]) - float(b["loss_iou"])) <= 1e-5 * abs(float(b["loss_iou"])) + 1e-9
    for xc, o in zip(xs, outs_d):
        err = float((xc.grad.double().cpu() - o["masks"].grad).norm() / o["masks"].grad.norm())
        assert err < 1e-5, err


# ------------------------------------------------------------------------------------------------
# 2. psam_interp_inverse
# ------------------------------------------------------------------------------------------------
INV_G = [1, 3, 64, 1023, 1024, 1025, 4096, 8192]
INV_N = [1, 341, 342, 32768]
INV_DIST = ["uniform", "one_patch", "half_empty", "knn"]
INV_CASES = [(G, N, d, 3 if (G + N + i) % 2 else 1) for i, (G, N, d) in enumerate(itertools.product(INV_G, INV_N, INV_DIST))
             if not (d == "knn" and G < 3)]


def _inv_index(G, N, B, dist, seed):
    g = np.random.default_rng(seed)
    if dist == "uniform":
        return g.integers(0, G, (B, N, 3))
    if dist == "one_patch":  # every warp's 32 entries hit one patch: __match_any_sync with the full mask
        return np.full((B, N, 3), g.integers(0, G), np.int64)
    if dist == "half_empty":
        return 2 * g.integers(0, max(1, G // 2), (B, N, 3))  # odd patches (and the top one for odd G) stay empty
    from psam_b200 import ops

    xyz = torch.from_numpy(g.uniform(-1, 1, (B, N, 3)).astype(F32)).to(_dev())
    cen = torch.from_numpy(g.uniform(-1, 1, (B, G, 3)).astype(F32)).to(_dev())
    return _np(ops.knn3_interp(xyz, cen)[0])


def _inv_id(G, N, dist, B):
    per = _cdiv(G, 1024)
    return _id("interp_inverse_kernel", G=G, N=N, B=B, per=per, E=3 * N, tail=int((3 * N) % 1024 != 0), dist=dist)


@pytest.mark.parametrize("G,N,dist,B", INV_CASES, ids=[_inv_id(*c) for c in INV_CASES])
def test_interp_inverse_is_a_stable_counting_sort(G, N, dist, B):
    nv = _nv()
    idx = _inv_index(G, N, B, dist, seed=G * 31 + N + B)
    assert idx.min() >= 0 and idx.max() < G
    iw = Win(torch.from_numpy(np.ascontiguousarray(idx, np.int64)))
    ow = Win(shape=(B, G + 1), dtype=torch.int32)
    ew = Win(shape=(B, 3 * N), dtype=torch.int32)
    assert nv.lib().psam_interp_inverse(iw.ptr, B, N, G, ow.ptr, ew.ptr, nv.stream()) == 0
    ow.check("offsets")
    ew.check("entries")
    flat = idx.reshape(B, 3 * N)
    offs = np.stack([np.concatenate([[0], np.cumsum(np.bincount(flat[b], minlength=G))]) for b in range(B)]).astype(np.int32)
    ents = np.stack([np.argsort(flat[b], kind="stable") for b in range(B)]).astype(np.int32)
    _cmp(ow.cpu(), torch.from_numpy(offs), "offsets")
    _cmp(ew.cpu(), torch.from_numpy(ents), "entries")


OOR_CASES = [(64, 341, 2), (1025, 342, 1), (8192, 32768, 3)]


@pytest.mark.parametrize("G,N,B", OOR_CASES, ids=[_id("interp_inverse_kernel", G=G, N=N, B=B, per=_cdiv(G, 1024), oor=1)
                                                  for G, N, B in OOR_CASES])
def test_interp_inverse_skips_out_of_range_indices(G, N, B):
    """An index outside [0, G) (-1, G, a large int64) is neither counted nor placed (include/psam_b200.h): offsets and the
    first offsets[b, G] entries are the counting sort of the in-range entries, and the tail of entries keeps its sentinel."""
    nv = _nv()
    g = np.random.default_rng(G + N)
    idx = g.integers(0, G, (B, N, 3))
    bad = np.array([-1, G, 1 << 40, -(1 << 40)], np.int64)
    for b in range(B):
        at = g.choice(3 * N, min(3 * N, 5 + 7 * b), replace=False)
        idx[b].reshape(-1)[at] = bad[np.arange(len(at)) % len(bad)]
    iw = Win(torch.from_numpy(np.ascontiguousarray(idx, np.int64)))
    ow = Win(shape=(B, G + 1), dtype=torch.int32)
    ew = Win(shape=(B, 3 * N), dtype=torch.int32)
    assert nv.lib().psam_interp_inverse(iw.ptr, B, N, G, ow.ptr, ew.ptr, nv.stream()) == 0
    ow.check("offsets")
    ew.check("entries")
    flat = idx.reshape(B, 3 * N)
    offs = np.zeros((B, G + 1), np.int32)
    ents = np.full((B, 3 * N), SENT, np.int64).astype(np.uint32).view(np.int32)
    for b in range(B):
        ok = (flat[b] >= 0) & (flat[b] < G)
        offs[b, 1:] = np.cumsum(np.bincount(flat[b][ok], minlength=G))
        e = np.nonzero(ok)[0]
        ents[b, :len(e)] = e[np.argsort(flat[b][e], kind="stable")]
        assert offs[b, G] == len(e) < 3 * N
    _cmp(ow.cpu(), torch.from_numpy(offs), "offsets")
    _cmp(ew.cpu(), torch.from_numpy(ents), "entries")


# ------------------------------------------------------------------------------------------------
# 3. psam_head_dp
# ------------------------------------------------------------------------------------------------
HD_NS = [1, 127, 128, 129, 4097]
HD_CASES = [(C, D, HD_NS[i % 5], 32 * (i % 2)) for i, (C, D) in enumerate(itertools.product([1, 2, 3, 8], [32, 96, 128, 256, 512, 1024]))]
HD_CASES += [(8, 1024, 4097, 32), (3, 1024, 129, 0), (8, 32, 4097, 0)]


def _hd_id(C, D, N, pad):
    return _id("head_dp_kernel", C=C, D=D, N=N, chunks=_cdiv(N, HEAD_RB), last=N - (_cdiv(N, HEAD_RB) - 1) * HEAD_RB, ldp=D + pad)


def _gelu64(x):
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def _gelu_grad64(x):
    return 0.5 * (1.0 + erf(x / math.sqrt(2.0))) + x * np.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


@pytest.mark.parametrize("C,D,N,pad", HD_CASES, ids=[_hd_id(*c) for c in HD_CASES])
def test_head_dp_against_fp64(C, D, N, pad):
    """dp (hi + lo) against fp64 GELU'(p) sum_c dm h, and the per-chunk partials against fp64 sums; the pitch padding and
    the gap between the planes keep their sentinel."""
    nv = _nv()
    Z = 2
    R, ldp = Z * N, D + pad
    plane = R * ldp + 64  # a gap between the planes: the lo plane is found through dp_plane, not R * ldp
    g = np.random.default_rng(C * 1000 + D + N)
    p = (g.standard_normal((R, D)) * 1.5).astype(F32)
    dm = g.standard_normal((Z, C, N)).astype(F32)
    h = (g.standard_normal((Z, C, D)) / 4).astype(F32)
    K = nv.lib().psam_head_dp_chunks(N)
    pw, mw, hw = Win(torch.from_numpy(p)), Win(torch.from_numpy(dm)), Win(torch.from_numpy(h))
    dpw = Win(shape=(plane + R * ldp,), dtype=torch.int16, fill=BF_SENT)
    phw = Win(shape=(Z, K, C, D), dtype=torch.float32)
    pbw = Win(shape=(Z, K, D), dtype=torch.float32)
    assert nv.lib().psam_head_dp(pw.ptr, mw.ptr, hw.ptr, Z, C, N, D, dpw.ptr, plane, ldp, phw.ptr, pbw.ptr, nv.stream()) == 0
    for w, n in ((dpw, "dp"), (phw, "part_hyper"), (pbw, "part_b3")):
        w.check(n)
    raw = dpw.cpu()
    hi, lo = raw[:R * ldp].view(R, ldp), raw[plane:plane + R * ldp].view(R, ldp)
    keep = torch.full((R, ldp - D), BF_SENT, dtype=torch.int16)
    _cmp(hi[:, D:], keep, "dp hi pitch padding")
    _cmp(lo[:, D:], keep, "dp lo pitch padding")
    _cmp(raw[R * ldp:plane], torch.full((plane - R * ldp,), BF_SENT, dtype=torch.int16), "gap between the dp planes")
    dp = (hi[:, :D].view(torch.bfloat16).double() + lo[:, :D].view(torch.bfloat16).double()).numpy().reshape(Z, N, D)
    p64, dm64, h64 = p.astype(np.float64).reshape(Z, N, D), dm.astype(np.float64), h.astype(np.float64)
    S = np.einsum("zcn,zcd->znd", dm64, h64)
    Sa = np.einsum("zcn,zcd->znd", np.abs(dm64), np.abs(h64))
    want = _gelu_grad64(p64) * S
    # fp32 in the kernel: sum_c dm h by C fmas (<= C u Sa), GELU' with erff / expf (<= 16 u absolute; |GELU'| <= 1.13),
    # the product (u); E = (1.2 C + 18) u Sa covers the three.  hi = bf16(dp), lo = bf16(dp - hi), 8-bit significands:
    # |hi + lo - dp| <= 2^-16 |dp|.
    E = (1.2 * C + 18) * U * Sa
    r1 = _ok(np.abs(dp - want), 2.0 ** -16 * (np.abs(want) + E) + E, "dp")
    # partials over each chunk of 128 points, fp32 fma accumulators: GELU by the A&S erf (|erf err| <= 1.5e-7, evaluation
    # <= 10 u), so |GELU err| <= |x| (0.75e-7 + 5 u) + u |GELU|; an L-term sum adds (L + 1) u of its magnitude
    ge = np.abs(p64) * (0.75e-7 + 5 * U) + U * np.abs(_gelu64(p64))
    u2 = _gelu64(p64)
    Kp = K * HEAD_RB
    padN = lambda a: np.concatenate([a, np.zeros(a.shape[:-2] + (Kp - N, a.shape[-1]))], -2) if Kp > N else a
    padn = lambda a: np.concatenate([a, np.zeros(a.shape[:-1] + (Kp - N,))], -1) if Kp > N else a
    u2c, gec = padN(u2).reshape(Z, K, HEAD_RB, D), padN(ge).reshape(Z, K, HEAD_RB, D)
    dmc = padn(dm64).reshape(Z, C, K, HEAD_RB)
    L = min(N, HEAD_RB)
    wh = np.einsum("zckj,zkjd->zkcd", dmc, u2c)
    bh = np.einsum("zckj,zkjd->zkcd", np.abs(dmc), gec) + (L + 1) * U * np.einsum("zckj,zkjd->zkcd", np.abs(dmc), np.abs(u2c))
    r2 = _ok(np.abs(_np(phw.t).astype(np.float64) - wh), bh, "part_hyper")
    wb = padN(want).reshape(Z, K, HEAD_RB, D).sum(2)
    bb = padN(E).reshape(Z, K, HEAD_RB, D).sum(2) + (L + 1) * U * padN(np.abs(want)).reshape(Z, K, HEAD_RB, D).sum(2)
    r3 = _ok(np.abs(_np(pbw.t).astype(np.float64) - wb), bb, "part_b3")
    _report(f"head_dp C={C} D={D} N={N}", max(r1, r2, r3))


# ------------------------------------------------------------------------------------------------
# 4. psam_interp_ln_gelu_backward, 5. psam_interp_backward
# ------------------------------------------------------------------------------------------------
LN_EPS = 0.03  # about twice the variance of the ordinary rows (0.2^2 * sum w^2 ~ 0.016): the eps shows in rstd


def _ln_inputs(Z, rep, G, N, D, seed):
    """Patches of three kinds - ordinary (0.2 N(0,1)), offset (50 + 0.2 N(0,1): |mean| >> std) and near-constant (one value
    per patch + 2e-5 N(0,1): variance << eps) - and points of four: three distinct patches of one kind, or one patch three
    times.  Weights positive, summing to about 1 (fp32)."""
    g = np.random.default_rng(seed)
    B = Z // rep
    kind = np.arange(G) % 3
    base = g.standard_normal((Z, G, D)) * 0.2
    f = np.where(kind[None, :, None] == 1, 50.0 + base, base)
    f = np.where(kind[None, :, None] == 2, g.standard_normal((Z, G, 1)) + 1e-4 * base, f).astype(F32)
    idx = np.empty((B, N, 3), np.int64)
    for n in range(N):
        k = n % 4
        if k < 3:
            pool = np.nonzero(kind == k)[0]
            idx[:, n] = np.stack([g.choice(pool, 3, replace=False) for _ in range(B)])
        else:
            idx[:, n] = g.integers(0, G, (B, 1))
    w = g.random((B, N, 3)) + 0.05
    w = (w / w.sum(-1, keepdims=True)).astype(F32)
    gamma = (1.0 + 0.5 * g.standard_normal(D)).astype(F32)
    beta = (0.3 * g.standard_normal(D)).astype(F32)
    du = g.standard_normal((Z * N, D)).astype(F32)
    return f, idx, w, gamma, beta, du


def _interp64(f, idx, w, Z, rep, G, D):
    f64 = f.astype(np.float64).reshape(Z, G, D)
    zb = np.arange(Z) // rep
    ii, ww = idx[zb], w.astype(np.float64)[zb]  # [Z, N, 3]
    gathered = f64[np.arange(Z)[:, None, None], ii]  # [Z, N, 3, D]
    return (ww[..., None] * gathered).sum(2), (np.abs(ww[..., None]) * np.abs(gathered)).sum(2)


LN_CASES = [(D, rb) for D in (128, 256, 512) for rb in (1, 7, 256, 1000)]
LN_Z, LN_REP, LN_G, LN_N = 6, 2, 40, 300  # 1800 rows: a partial last block at every rows_per_block but 1


def _ln_id(D, rb):
    rows = LN_Z * LN_N
    return _id(ln_kernel(D), D=D, rb=rb, blocks=_cdiv(rows, rb), last=rows - (_cdiv(rows, rb) - 1) * rb)


@pytest.mark.parametrize("D,rb", LN_CASES, ids=[_ln_id(*c) for c in LN_CASES])
def test_interp_ln_gelu_backward_against_fp64_autograd(D, rb):
    nv = _nv()
    Z, rep, G, N = LN_Z, LN_REP, LN_G, LN_N
    f, idx, w, gamma, beta, du = _ln_inputs(Z, rep, G, N, D, seed=D + rb)
    eps = F32(LN_EPS)
    fw, iw, ww = Win(torch.from_numpy(f.reshape(Z * G, D))), Win(torch.from_numpy(idx)), Win(torch.from_numpy(w))
    gw, bw = Win(torch.from_numpy(gamma)), Win(torch.from_numpy(beta))
    dw = Win(torch.from_numpy(du))
    nblk = _cdiv(Z * N, rb)
    pw = Win(shape=(nblk, 2, D), dtype=torch.float32)
    assert nv.lib().psam_interp_ln_gelu_backward(fw.ptr, Z, rep, G, D, iw.ptr, ww.ptr, N, gw.ptr, bw.ptr, float(eps), dw.ptr,
                                                 pw.ptr, rb, nv.stream()) == 0
    dw.check("du")
    pw.check("part")
    # fp64 autograd of gelu(layer_norm(interp(f))) from the same fp32 inputs
    v, va = _interp64(f, idx, w, Z, rep, G, D)
    vt = torch.from_numpy(v.reshape(Z * N, D)).requires_grad_(True)
    g64, b64 = torch.from_numpy(gamma).double().requires_grad_(True), torch.from_numpy(beta).double().requires_grad_(True)
    y = torch.nn.functional.gelu(torch.nn.functional.layer_norm(vt, (D,), g64, b64, float(eps)))
    y.backward(torch.from_numpy(du).double())
    want = vt.grad.numpy()
    mean = v.reshape(Z * N, D).mean(-1, keepdims=True)
    var = ((v.reshape(Z * N, D) - mean) ** 2).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + float(eps))
    xh = (v.reshape(Z * N, D) - mean) * rstd
    dh = du.astype(np.float64) * _gelu_grad64(xh * gamma.astype(np.float64) + beta.astype(np.float64))
    # error model: the recompute rounds v (3 fp32 operations, <= 3u of sum |w f|) and the mean; both are amplified by
    # kappa = max|v| / sqrt(var + eps), the common offset over the row's spread, into x_hat and rstd; the D-long warp sums of
    # the mean, variance, m1 and m2 add (4 NV + 5) u each.  Every term of dv is at most rstd |du| |gamma| (1 + |x_hat|)
    # (GELU' <= 1.13, GELU'' <= 0.4 through gamma); 8 units of (kappa + 4 NV + 8) u of that scale bound the sum.
    NV = D // 128
    kappa = va.reshape(Z * N, D).max(-1, keepdims=True) * rstd
    gm = np.abs(gamma).max() + np.abs(beta).max() + 1.0
    X = np.abs(xh).max(-1, keepdims=True)
    scale = rstd * np.abs(du).max(-1, keepdims=True) * gm * gm * (1.0 + X)
    bound = 8 * U * (kappa + 4 * NV + 8) * scale
    r1 = _ok(np.abs(_np(dw.t).astype(np.float64) - want), np.broadcast_to(bound, want.shape), "du")
    # partials: per CTA of rb rows, 8 warps each summing its rows in order, then the warps in order
    rows = Z * N
    pad = nblk * rb - rows
    padr = lambda a: np.concatenate([a, np.zeros((pad,) + a.shape[1:])]) if pad else a
    term_g, term_b = dh * xh, dh
    tb = 8 * U * (kappa + 8) * np.abs(du) * gm * gm * (1.0 + np.abs(xh)) ** 2
    Lw = _cdiv(min(rb, rows), 8) + 8
    want_p = np.stack([padr(term_g).reshape(nblk, rb, D).sum(1), padr(term_b).reshape(nblk, rb, D).sum(1)], 1)
    bound_p = np.stack([padr(tb + Lw * U * np.abs(term_g)).reshape(nblk, rb, D).sum(1),
                        padr(tb + Lw * U * np.abs(term_b)).reshape(nblk, rb, D).sum(1)], 1)
    got_p = _np(pw.t).astype(np.float64)
    r2 = _ok(np.abs(got_p - want_p), bound_p, "dgamma/dbeta partials")
    # the partials summed: fp64 dgamma / dbeta
    r3 = _ok(np.abs(got_p[:, 0].sum(0) - g64.grad.numpy()), bound_p[:, 0].sum(0), "dgamma")
    r4 = _ok(np.abs(got_p[:, 1].sum(0) - b64.grad.numpy()), bound_p[:, 1].sum(0), "dbeta")
    _report(f"interp_ln_gelu_backward D={D} rb={rb}", max(r1, r2, r3, r4))


IB_CASES = [128, 256, 512, 1024]


@pytest.mark.parametrize("D", IB_CASES, ids=[_id(ib_kernel(D), D=D, Z=4, rep=2, G=50) for D in IB_CASES])
def test_interp_backward_against_fp64_scatter_add(D):
    """df against an fp64 scatter-add of w dv; odd patches have no entries and must be rows of +0.0."""
    nv = _nv()
    Z, rep, G, N = 4, 2, 50, 300
    B = Z // rep
    g = np.random.default_rng(D)
    idx = 2 * g.integers(0, G // 2, (B, N, 3))
    idx[:, : N // 3] = 8  # one crowded patch
    w = g.random((B, N, 3)).astype(F32)
    dv = g.standard_normal((Z * N, D)).astype(F32)
    flat = idx.reshape(B, 3 * N)
    offs = np.stack([np.concatenate([[0], np.cumsum(np.bincount(flat[b], minlength=G))]) for b in range(B)]).astype(np.int32)
    ents = np.stack([np.argsort(flat[b], kind="stable") for b in range(B)]).astype(np.int32)
    vw, ow, ew, ww = Win(torch.from_numpy(dv)), Win(torch.from_numpy(offs)), Win(torch.from_numpy(ents)), Win(torch.from_numpy(w))
    fw = Win(shape=(Z * G, D), dtype=torch.float32)
    assert nv.lib().psam_interp_backward(vw.ptr, Z, rep, G, D, ow.ptr, ew.ptr, ww.ptr, N, fw.ptr, nv.stream()) == 0
    fw.check("df")
    want, mag = np.zeros((Z, G, D)), np.zeros((Z, G, D))
    for z in range(Z):
        b = z // rep
        for k in range(3):
            c = w[b, :, k].astype(np.float64)[:, None] * dv[z * N:(z + 1) * N].astype(np.float64)
            np.add.at(want[z], idx[b, :, k], c)
            np.add.at(mag[z], idx[b, :, k], np.abs(c))
    cnt = np.bincount(flat.reshape(-1), minlength=G)  # an upper bound of each patch's entries in either cloud
    got = _np(fw.t).reshape(Z, G, D).astype(np.float64)
    r = _ok(np.abs(got - want), (cnt[None, :, None] + 1) * U * mag, "df")  # one fma per entry, in order
    empty = np.nonzero(cnt == 0)[0]
    assert len(empty) >= G // 2
    _cmp(fw.cpu().view(Z, G, D)[:, empty], torch.zeros(Z, len(empty), D), "df of empty patches", raw=True)
    _report(f"interp_backward D={D}", r)


# ------------------------------------------------------------------------------------------------
# 6. psam_sum_partials
# ------------------------------------------------------------------------------------------------
SP_CASES = [(2, 1, 600000), (3, 2, 400001), (2, 37, 20000), (4, 37, 300000), (5, 2, 7)]


@pytest.mark.parametrize("nb,S,n", SP_CASES, ids=[_id("sum_partials_kernel", nb=nb, S=S, n=n, grid=sum_grid(nb, n),
                                                      loop=int(sum_grid(nb, n) * 256 < nb * n)) for nb, S, n in SP_CASES])
def test_sum_partials_is_a_sequential_fp64_sum(nb, S, n):
    nv = _nv()
    g = np.random.default_rng(nb * 100 + S)
    part = (g.standard_normal((nb, S, n)) * 10.0 ** g.integers(-4, 5, (nb, S, n))).astype(F32)
    pw = Win(torch.from_numpy(part))
    ow = Win(shape=(nb, n), dtype=torch.float32)
    assert nv.lib().psam_sum_partials(pw.ptr, nb, S, n, ow.ptr, nv.stream()) == 0
    ow.check("out")
    acc = np.zeros((nb, n))
    for s in range(S):  # in order s = 0, 1, ..., one fp64 add each, then one cast
        acc += part[:, s].astype(np.float64)
    _cmp(ow.cpu(), torch.from_numpy(acc.astype(F32)), "sum_partials", raw=True)


# ------------------------------------------------------------------------------------------------
# the chunked head backward
# ------------------------------------------------------------------------------------------------
HEAD_EPS = 0.03
# name: (Z, rep, N, BACKWARD_ROWS, DW_SPLIT_K)
PLANS = {
    "one_chunk": (2, 2, 1000, 262144, 4096),       # one chunk per cloud, one dW3 batch with a zero-padded tail
    "uneven": (16, 8, 1000, 3000, 4096),           # zc = 3: chunks of 3, 3, 2 prompts per cloud
    "zc1": (4, 2, 5000, 4096, 4096),               # N > BACKWARD_ROWS: one prompt per chunk, two dW3 batches
    "pad_batches": (2, 2, 1000, 1000, 50),         # R = 1000: S = 20, Kc = 64, Kp = 1280: batches 16..19 are all padding
    "many_batches": (4, 4, 1000, 262144, 16),      # R = 4000: S = 250 batches of 64, 187 of them all padding
}
HEAD_CASES = [(p, 256) for p in PLANS] + [(p, D) for p in ("uneven", "zc1", "pad_batches") for D in (128, 512)]


def _plan_id(plan, D):
    Z, rep, N, br, dw = PLANS[plan]
    chunks, splits = head_plan(Z, rep, N, br, dw)
    return _id("head_backward", D=D, plan=plan, chunks=len(chunks), batches=sum(s for s, _, _ in splits),
               padded=int(any(kp != (z1 - z0) * N for (_, z0, z1), (_, _, kp) in zip(chunks, splits))))


def _dirty_allocator():
    """Release every cached block, then fill a large one with NaN and free it: it is the only memory the caching allocator
    holds, so later allocations come from it and a buffer that should have been zeroed shows."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    x = torch.full((256 << 20,), NAN, dtype=torch.float32, device=_dev())
    torch.cuda.synchronize()
    del x


def _head_inputs(D, Z, rep, N, G=64, seed=0):
    from oracle import train_ref
    from pc_sam.model.mask_decoder import AuxInputs, MaskDecoder
    from pc_sam.model.transformer import TwoWayTransformer
    from psam_b200 import train

    md = train_ref.fill_params(MaskDecoder(D, TwoWayTransformer(2, D, 8, 2048)), seed + 1).to(_dev())
    md.output_upscaling[1].eps = HEAD_EPS
    g = torch.Generator().manual_seed(seed)
    B = Z // rep
    coords = (torch.rand(B, N, 3, generator=g) * 2 - 1).to(_dev())
    centers = (torch.rand(B, G, 3, generator=g) * 2 - 1).to(_dev())
    aux = AuxInputs(coords=coords, features=None, centers=centers)
    geo = train.head_geometry(aux, G, rep, HEAD_EPS)
    f0 = (torch.randn(Z * G, D, generator=g) * 0.2).to(_dev())
    hyper = (torch.randn(Z, 3, D, generator=g) / 16).to(_dev())
    dm = torch.randn(Z, 3, N, generator=g).to(_dev())
    up = md.output_upscaling
    params = [t.detach().float().contiguous() for t in (up[1].weight, up[1].bias, up[3].weight, up[3].bias)]
    return f0, hyper, params, geo, dm


def _nrel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).norm() / want.norm().clamp_min(1e-30))


@pytest.mark.parametrize("plan,D", HEAD_CASES, ids=[_plan_id(*c) for c in HEAD_CASES])
def test_chunked_head_backward_against_fp64_autograd(plan, D, monkeypatch):
    """Every chunk plan against oracle.train_ref.mask_head in fp64 autograd, within the same normwise bound; two runs of one
    plan agree bit for bit."""
    from oracle import train_ref
    from psam_b200 import train

    Z, rep, N, br, dw = PLANS[plan]
    monkeypatch.setattr(train, "BACKWARD_ROWS", br)
    monkeypatch.setattr(train, "DW_SPLIT_K", dw)
    f0, hyper, (gm, bt, w3, b3), geo, dm = _head_inputs(D, Z, rep, N, seed=D + len(plan))
    runs = []
    for _ in range(2):
        _dirty_allocator()
        runs.append(train.head_backward(f0, hyper, gm, bt, w3, b3, geo, dm))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    G = geo.G
    p64 = [t.double().cpu().requires_grad_(True) for t in (gm, bt, w3, b3)]
    f64, h64 = f0.double().cpu().view(Z, G, D).requires_grad_(True), hyper.double().cpu().requires_grad_(True)
    want = train_ref.mask_head(f64, h64, p64[0], p64[1], HEAD_EPS, p64[2], p64[3], geo.idx.cpu(), geo.w.double().cpu(), rep)
    want.backward(dm.double().cpu())
    df0, dh, dg, db, dw3, db3 = runs[0]
    errs = dict(f0=_nrel(df0, f64.grad.view(Z * G, D)), hyper=_nrel(dh, h64.grad), gamma=_nrel(dg, p64[0].grad),
                beta=_nrel(db, p64[1].grad), w3=_nrel(dw3, p64[2].grad), b3=_nrel(db3, p64[3].grad))
    print(f"[train kernels] head_backward {plan} D={D}: " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 1e-4, (k, v)


def test_head_backward_needs_input_grad_combinations(monkeypatch):
    """Every (f0, gamma/beta, W3) combination on a plan of uneven chunks: what is asked for is bit for bit the full run's,
    the rest is None; dhyper and db3 always come."""
    from psam_b200 import train

    Z, rep, N, br, dw = PLANS["uneven"]
    monkeypatch.setattr(train, "BACKWARD_ROWS", br)
    f0, hyper, (gm, bt, w3, b3), geo, dm = _head_inputs(256, Z, rep, N, seed=5)
    _dirty_allocator()
    full = train.head_backward(f0, hyper, gm, bt, w3, b3, geo, dm)
    for nf, nl, nw in itertools.product([False, True], repeat=3):
        _dirty_allocator()
        got = train.head_backward(f0, hyper, gm, bt, w3, b3, geo, dm, need_f0=nf, need_ln=nl, need_w3=nw)
        need = (nf, True, nl, nl, nw, True)
        for i, (a, b, n) in enumerate(zip(got, full, need)):
            if n:
                assert a is not None and torch.equal(a, b), (nf, nl, nw, i)
            else:
                assert a is None, (nf, nl, nw, i)


def test_whole_step_with_several_chunks_per_cloud(monkeypatch):
    """The teacher-forced whole step (tests/test_gpu_finetune.py) with BACKWARD_ROWS = 3 N: four prompts per cloud run in
    chunks of 3 and 1 in every iteration's backward."""
    import test_gpu_finetune as tf
    from psam_b200 import engine, train

    monkeypatch.setattr(train, "BACKWARD_ROWS", 3 * 4096)
    calls = []
    real = engine.upscale_ln_gelu

    def record(f0, Z, rep, *a):
        calls.append((Z, rep))
        return real(f0, Z, rep, *a)

    monkeypatch.setattr(engine, "upscale_ln_gelu", record)
    tf.test_whole_step_against_teacher_forced_fp64_oracle(monkeypatch)
    fwd = [c for c in calls if c == (8, 4)]
    bwd = [z for z, r in calls if (z, r) != (8, 4)]
    assert len(fwd) == 5 and bwd == [3, 1, 3, 1] * 5, calls


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def test_routing_guard():
    """One call per kernel instance of csrc/train.cu, the forward's mask product with and without the fused row-dot, and
    every head chunk plan, under the profiler: the kernels that ran must be the restated ones.  It runs in a fresh
    interpreter, as the other routing guards do."""
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_train_kernels as t; t._routing_guard()" % (
        here, repo, os.path.join(repo, "point-sam_b200"))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def _names(got):
    return [n for n, _ in got]


def _expect(got, want, what):
    assert len(got) == len(want), f"{what}: {len(want)} kernels expected, {len(got)} launched: {_names(got)}"
    for w, (name, _) in zip(want, got):
        assert w in name and (w.endswith(">") or f"{w}<" not in name), f"{what}: expected {w}, ran {name}"


def _routing_guard():
    from psam_b200 import train

    nv = _nv()
    L, d, st = nv.lib(), _dev(), nv.stream()
    calls, keep = [], []

    def z(*shape, dtype=torch.float32):
        t = torch.zeros(shape, dtype=dtype, device=d)
        keep.append(t)
        return t

    Z, C, N, G = 2, 3, 300, 40
    x, gt, up = z(Z, C, N), z(Z, N, dtype=torch.uint8), torch.ones(Z, C, device=d)
    keep.append(up)
    stt, cnt, dl = z(Z, C, 4), z(Z, C, 2, dtype=torch.int32), z(Z, C, N)
    # (expected kernels, (kernel, restated grid x, grid y) or None, fn)
    calls.append((["mask_loss_stats_kernel"], None,
                  lambda: L.psam_mask_loss_stats(x.data_ptr(), gt.data_ptr(), Z, C, N, stt.data_ptr(), cnt.data_ptr(), st)))
    for Nl in (300, 100000):  # one block per 256 logits, and the 64-block cap that loops
        xl, gl, dll = z(Z, C, Nl), z(Z, Nl, dtype=torch.uint8), z(Z, C, Nl)
        calls.append((["mask_loss_grad_kernel"], ("mask_loss_grad_kernel", loss_grid(Nl), Z * C),
                      lambda xl=xl, gl=gl, dll=dll, Nl=Nl: L.psam_mask_loss_grad(xl.data_ptr(), gl.data_ptr(), Z, C, Nl, stt.data_ptr(),
                                                                                 up.data_ptr(), dll.data_ptr(), st)))
    idx = torch.from_numpy(np.random.default_rng(0).integers(0, G, (1, N, 3))).to(d)
    w = torch.full((1, N, 3), 1 / 3, device=d)
    keep += [idx, w]
    offs, ents = z(1, G + 1, dtype=torch.int32), z(1, 3 * N, dtype=torch.int32)
    calls.append((["interp_inverse_kernel"], None,
                  lambda: L.psam_interp_inverse(idx.data_ptr(), 1, N, G, offs.data_ptr(), ents.data_ptr(), st)))
    for D in (128, 256, 512):
        f, gam, bet, du, part = z(Z * G, D), z(D), z(D), z(Z * N, D), z(_cdiv(Z * N, 7), 2, D)
        calls.append(([ln_kernel(D)], None, lambda f=f, gam=gam, bet=bet, du=du, part=part, D=D: L.psam_interp_ln_gelu_backward(
            f.data_ptr(), Z, Z, G, D, idx.data_ptr(), w.data_ptr(), N, gam.data_ptr(), bet.data_ptr(), 0.03, du.data_ptr(), part.data_ptr(), 7, st)))
    for D in (128, 256, 512, 1024):
        dv, df = z(Z * N, D), z(Z * G, D)
        calls.append(([ib_kernel(D)], None, lambda dv=dv, df=df, D=D: L.psam_interp_backward(
            dv.data_ptr(), Z, Z, G, D, offs.data_ptr(), ents.data_ptr(), w.data_ptr(), N, df.data_ptr(), st)))
    p, dm, hy = z(Z * N, 1024), z(Z, 8, N), z(Z, 8, 1024)
    dp = z(2 * Z * N * 1024, dtype=torch.int16)
    K = L.psam_head_dp_chunks(N)
    ph, pb = z(Z, K, 8, 1024), z(Z, K, 1024)
    calls.append((["head_dp_kernel"], ("head_dp_kernel", K, Z), lambda: L.psam_head_dp(
        p.data_ptr(), dm.data_ptr(), hy.data_ptr(), Z, 8, N, 1024, dp.data_ptr(), Z * N * 1024, 1024, ph.data_ptr(), pb.data_ptr(), st)))
    for nb, S, n in ((2, 37, 1000), (2, 1, 600000)):  # below and past the grid-stride cap
        sp, so = z(nb, S, n), z(nb, n)
        calls.append((["sum_partials_kernel"], ("sum_partials_kernel", sum_grid(nb, n), 1),
                      lambda sp=sp, so=so, nb=nb, S=S, n=n: L.psam_sum_partials(sp.data_ptr(), nb, S, n, so.data_ptr(), st)))
    torch.cuda.synchronize()
    rcs = []
    got = _kernels_launched(lambda: rcs.extend(fn() for _, _, fn in calls))
    assert rcs == [0] * len(calls), f"return codes {rcs}"
    _expect(got, [n for names, _, _ in calls for n in names], "C ABI")
    pos, grids = 0, 0
    for names, g, _ in calls:
        if g is not None:
            grid = got[pos + names.index(g[0])][1]
            assert grid is not None, f"{g[0]}: the trace has no grid"
            assert (grid[0], grid[1]) == (g[1], g[2]), f"{g[0]}: grid {grid}, restated {g[1:]}"
            grids += 1
        pos += len(names)
    print(f"[train] routing guard: {len(calls)} calls, each the restated instance, {grids} grids as restated: "
          + ", ".join(sorted({n for names, _, _ in calls for n in names})))

    # the head: forward with the fused row-dot (N % 32 == 0) or psam_mask_dot (N % 32 != 0), and each chunk plan of the
    # backward: per chunk one head_dp, LayerNorm and interpolation backward, two transposes for dW3 and then its GEMM with one
    # batch per K split (grid z = S of the restated plan)
    fused = 0
    for plan, (Zp, rep, Np, br, dw) in PLANS.items():
        for Nf in ((Np, Np + 24) if plan == "one_chunk" else (Np,)):
            train.BACKWARD_ROWS, train.DW_SPLIT_K = br, dw
            f0, hyper, (gm, bt, w3, b3), geo, dmh = _head_inputs(256, Zp, rep, Nf)
            lv = [t.clone().requires_grad_(True) for t in (f0, hyper, gm, bt, w3, b3)]
            box = []
            fwd = _kernels_launched(lambda: box.append(train.MaskHead.apply(*lv, geo)))
            dots = sum("mask_dot_kernel" in n for n in _names(fwd))
            assert dots == (0 if Nf % 32 == 0 else 1), f"N = {Nf}: {dots} mask_dot_kernel launches, {_names(fwd)}"
            fused += dots == 0
            bwd = _kernels_launched(lambda: box[0].backward(dmh))
            chunks, splits = head_plan(Zp, rep, Nf, br, dw)
            names = _names(bwd)
            for k in ("head_dp_kernel", "interp_ln_gelu_bwd_kernel<2>", "interp_bwd_kernel<2>"):
                n = sum(k in s for s in names)
                assert n == len(chunks), f"{plan}: {n} {k} launches, restated {len(chunks)} chunks"
            assert sum("sum_partials_kernel" in s for s in names) == 4, names
            tr = [i for i, s in enumerate(names) if "transpose_split_kernel" in s]
            assert len(tr) == 2 * len(chunks), f"{plan}: {len(tr)} transposes, restated 2 per chunk ({len(chunks)} chunks)"
            batches = []
            for i in tr[1::2]:  # the dW3 GEMM follows the second transpose of its chunk
                assert "gemm_wgmma_kernel" in names[i + 1], f"{plan}: {names[i + 1]} after the dW3 transposes"
                grid = bwd[i + 1][1]
                assert grid is not None, f"{plan}: the trace has no grid for the dW3 GEMM"
                batches.append(grid[2])
            assert batches == [s for s, _, _ in splits], f"{plan}: dW3 GEMM batches {batches}, restated {[s for s, _, _ in splits]}"
            print(f"[train] {plan} N={Nf}: {len(chunks)} chunks and dW3 GEMM batches {batches} as restated, "
                  f"mask_dot {'no (fused row-dot)' if dots == 0 else 'yes'}")
    assert fused == 1, "the fused row-dot forward was not reached"
