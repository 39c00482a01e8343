"""The geometry kernels that feed every model - FPS, kNN, the group gather, the brute-force nearest search, the Voronoi
features and the border-prompt sampler - through the C ABI, on every launch path of their host functions.

Each kernel is compared with a plain reference of the same operation:
  * FPS and kNN bit for bit against the C oracle (oracle/tokenizer_ref.c: the reference's fmaf chain, -ffp-contract=off),
    and against an fp64 semantic check that shares no fp32 formula with either: every FPS pick is within (1 - 10u) of the
    farthest point, and every chosen kNN key within (1 + 10u) of the nearest key left out.  10u is the worst case of two
    distances computed as fmaf(dz,dz,fmaf(dy,dy,dx*dx)) from fp32 differences (5 roundings of at most u each);
  * the group gather and the Voronoi features exactly against the roundings the header states;
  * the border-prompt sampler bit for bit against oracle.torch_ref.sample_fixed_points, coordinates and labels.
Inputs sit inside NaN guards and outputs inside NaN (or sentinel) guards: nothing outside a window may be written, and
a padded cloud's padding is built to be chosen if a kernel read it.  Every case id names the instantiation it reaches,
from the host plans restated below; test_routing_guard checks those names under torch.profiler."""
import itertools
import json
import math
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24       # fp32 unit roundoff
DIST = 2.5 * U       # Voronoi dist: sqrtf of a product and two FMAs - 3u in the sum, halved, plus u in the sqrt
REL = 10 * U         # slack of the fp64 semantic checks (see the module docstring)
ERR_ARG, ERR_UNSUPPORTED = -1, -2
GUARD = 64           # guard elements on either side of every window (256 bytes of fp32: alignment is kept)


def _nv():
    from psam_b200 import native as nv

    return nv


def _dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------
# the host plans, restated (test_routing_guard checks them against the kernels that run)
# ------------------------------------------------------------------------------------------------
FPS_THREADS = 256


def fps_log2T(N):
    T = 1
    while T < N and T < 512:
        T *= 2
    return int(math.log2(T if T >= 64 else 32))


def fps_plan(N, max_cluster):
    c = max_cluster if max_cluster > 8 and N > 8 * FPS_THREADS * 32 else (8 if max_cluster > 8 else max_cluster)
    while c > 1 and (c // 2) * FPS_THREADS >= N:
        c //= 2
    per = -(-N // (c * FPS_THREADS))
    p = 1
    while p < per:
        p *= 2
    return c, (p if p <= 32 else 0)


def fps_route(N, max_cluster=16):
    """(cluster width, PPT) of fps_dispatch when the device co-schedules clusters of max_cluster CTAs (16 on H100; 8 when
    its probe declines).  PPT 0 is the streaming plan."""
    c, p = fps_plan(N, max_cluster if N > 8 * FPS_THREADS * 32 else 8)
    return (max_cluster if p == 0 else c), p


def _fps_kernel(N, varlen=False, max_cluster=16):
    return f"fps_cluster_kernel<{fps_route(N, max_cluster)[1]}, {'true' if varlen else 'false'}>"


def knn_sample_stride(N, K):
    s = 1
    while K * s * 2 <= 1024 and (N + 2 * s - 1) // (2 * s) >= 4 * K:
        s *= 2
    while (N + s - 1) // s > 16384:
        s *= 2
    return s


def knn_plan(B, Q, N, K):
    """(C, cap) of knn_dispatch: C query centres per CTA, cap candidates per centre."""
    stride = knn_sample_stride(N, K)
    sample_cap = (2 * K + 3) & ~3
    cap = min(max(2 * K * stride, 1024), 16384)
    if cap > N:
        cap = (N + 3) & ~3
    smem = lambda c: sample_cap * 4 + c * cap * 8 + (64 + c * 2048) * 4
    C = 4
    while C > 1 and (B * (-(-Q // C)) < 222 or smem(C) > 100 * 1024):
        C //= 2
    return C, cap


def _knn_kernel(B, Q, N, K, varlen=False):
    return f"knn_kernel<{knn_plan(B, Q, N, K)[0]}, {'true' if varlen else 'false'}>"


def _id(kernel, **kw):
    return kernel.replace(", ", ",") + "-" + "-".join(f"{k}{v}" for k, v in kw.items())


# ------------------------------------------------------------------------------------------------
# guarded device windows
# ------------------------------------------------------------------------------------------------
class Win:
    """A device tensor `t` inside a flat buffer with GUARD elements of `fill` on either side (`offset` more in front, to
    misalign it).  check() asserts that the guards are untouched, bit for bit."""

    def __init__(self, data=None, shape=None, dtype=torch.float32, fill=float("nan"), offset=0):
        if data is not None:
            data = torch.as_tensor(data)
            shape, dtype = tuple(data.shape), data.dtype
        n = int(np.prod(shape)) if len(shape) else 1
        self.flat = torch.full((GUARD + offset + n + GUARD,), fill, dtype=dtype)
        if data is not None:
            self.flat[GUARD + offset:GUARD + offset + n] = data.reshape(-1)
        self.before = self.flat[:GUARD + offset].clone()
        self.after = self.flat[GUARD + offset + n:].clone()
        self.flat = self.flat.to(_dev())
        self.lo, self.n = GUARD + offset, n
        self.t = self.flat[self.lo:self.lo + n].view(shape)

    @property
    def ptr(self):  # from the buffer: an empty window (C = 0 features) still has an address
        return self.flat.data_ptr() + self.lo * self.flat.element_size()

    def check(self, name):
        torch.cuda.synchronize()
        f = self.flat.cpu()
        same = lambda a, b: torch.equal(a.view(torch.uint8), b.view(torch.uint8))
        assert same(f[:self.lo], self.before) and same(f[self.lo + self.n:], self.after), f"{name}: wrote outside its window"

    def cpu(self):
        return self.t.cpu()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bits(got, want, name):
    bad = _bits(got) != _bits(want)
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} of {got.numel()} values differ, first at {bad.nonzero()[:3].tolist()}: "
                                 f"got {got[bad][:3].tolist()} want {want[bad][:3].tolist()}")


# ------------------------------------------------------------------------------------------------
# fp64 semantic checks (no fp32 formula shared with the kernels or the oracle)
# ------------------------------------------------------------------------------------------------
def fps_greedy_excess(xyz, idx):
    """Largest (M_i - d_i) / (REL * M_i) over the steps of one cloud: d_i is pick i's fp64 squared distance to the earlier
    picks, M_i the largest over all points.  A greedy FPS within rounding gives <= 1."""
    x = np.asarray(xyz, dtype=np.float64)
    md = np.full(len(x), np.inf)
    worst = 0.0
    for i in range(1, len(idx)):
        md = np.minimum(md, ((x - x[idx[i - 1]]) ** 2).sum(1))
        M = md.max()
        if M > 0:
            worst = max(worst, (M - md[idx[i]]) / (REL * M))
    return worst


def knn_set_excess(query, key, idx):
    """Largest (max chosen - min other) / (REL * min other) over the query rows of one cloud, fp64 squared distances.  The
    exact K nearest up to rounding give <= 1 (a zero `min other` allows only chosen distances of zero)."""
    q, k = np.asarray(query, dtype=np.float64), np.asarray(key, dtype=np.float64)
    d = ((q[:, None, :] - k[None, :, :]) ** 2).sum(-1)
    chosen = np.zeros(d.shape, dtype=bool)
    np.put_along_axis(chosen, np.asarray(idx), True, axis=1)
    if chosen.all():
        return 0.0
    hi = np.where(chosen, d, -np.inf).max(1)
    lo = np.where(chosen, np.inf, d).min(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(lo > 0, (hi - lo) / (REL * lo), np.where(hi > 0, np.inf, 0.0))
    return float(r.max())


def voronoi_dist_excess(xyz, centers, nn_idx, dist):
    """Largest |dist - |p - c|| / (DIST |p - c|) over the points of one cloud, fp64 norm of the fp32 differences.  The
    kernel's dist is the square root of one product and two FMAs, in whatever axis order the compiler picks: three
    roundings of at most u in a sum of non-negative terms (3u), halved by the square root, plus u for the correctly rounded
    square root - 2.5u.  2u is not enough: d = (1.0175835, -0.23071885, 0.0535804), with the x square taken first, rounds
    to 1.07 x 2u.  A zero norm requires dist == 0."""
    d = (torch.as_tensor(xyz) - torch.as_tensor(centers)[torch.as_tensor(nn_idx)]).double()
    n = d.norm(dim=-1)
    err = (torch.as_tensor(dist).double() - n).abs()
    r = torch.where(n > 0, err / (DIST * n), torch.where(err > 0, torch.inf, 0.0))
    return float(r.max())


# ------------------------------------------------------------------------------------------------
# clouds
# ------------------------------------------------------------------------------------------------
def _lattice(N, seed):
    """N distinct points of an integer lattice in random order: exact distances, many equal maxima and ties."""
    L = 1
    while L ** 3 < N:
        L += 1
    g = torch.stack(torch.meshgrid(*(torch.arange(L),) * 3, indexing="ij"), -1).reshape(-1, 3).float()
    return g[torch.randperm(len(g), generator=_gen(seed))[:N]].contiguous()


def _cloud(kind, N, seed, distinct=None):
    g = _gen(seed)
    if kind == "random":
        return torch.rand(N, 3, generator=g) * 2 - 1
    if kind == "lattice":
        return _lattice(N, seed)
    if kind == "duplicates":
        base = torch.rand(max(N // 4, 1), 3, generator=g) * 2 - 1
        return base[torch.randint(0, len(base), (N,), generator=g)]
    if kind == "few":
        base = torch.rand(distinct, 3, generator=g) * 2 - 1
        return base[torch.randint(0, distinct, (N,), generator=g)]
    if kind == "identical":
        return (torch.rand(1, 3, generator=g) * 2 - 1).expand(N, 3).contiguous()
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------
# FPS
# ------------------------------------------------------------------------------------------------
def _run_fps(xyz, G, lengths=None):
    """psam_fps_f32 (or the varlen form) on guarded windows; returns (idx, centres) on the host."""
    nv = _nv()
    B, N, _ = xyz.shape
    x, idx, cen = Win(xyz), Win(shape=(B, G), dtype=torch.int64, fill=-7), Win(shape=(B, G, 3))
    nb = nv.lib().psam_fps_workspace_bytes(B, N, G)
    ws = Win(shape=(nb // 4,), fill=-3.0) if nb else None
    if lengths is None:
        rc = nv.lib().psam_fps_f32(x.ptr, B, N, G, idx.ptr, cen.ptr, ws.ptr if ws else None, nv.stream())
    else:
        ln = torch.tensor(lengths, dtype=torch.int32, device=_dev())
        rc = nv.lib().psam_fps_varlen_f32(x.ptr, ln.data_ptr(), B, N, G, idx.ptr, cen.ptr, ws.ptr if ws else None, nv.stream())
    assert rc == 0
    for w, name in ((x, "xyz"), (idx, "idx"), (cen, "centers")) + (((ws, "workspace"),) if ws else ()):
        w.check(name)
    return idx.cpu(), cen.cpu()


def _check_fps(xyz, G, idx, cen, name):
    from oracle import tokenizer_ref

    want = tokenizer_ref.fps(xyz.numpy(), G)
    got = idx.numpy()
    assert np.array_equal(got, want), f"{name}: {int((got != want).sum())} picks differ, first at {np.argwhere(got != want)[:3].tolist()}"
    _assert_bits(cen, xyz[torch.arange(len(xyz))[:, None], idx], f"{name} centres")
    ex = max(fps_greedy_excess(xyz[b].numpy(), got[b]) for b in range(len(xyz)))
    print(f"[geom] fps {name}: greedy excess {ex:.3f} of its bound")
    assert ex <= 1.0
    return ex


_FPS_N = [32, 33, 63, 64, 65, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192, 8193, 16384, 16385, 32768,
          32769, 65536, 65537, 131072, 131073]
_FPS_CASES = [(N, min(N, 96) if N <= 16384 else 24, kind) for N in _FPS_N for kind in ("random", "lattice", "duplicates")]
_FPS_CASES += [(1000, 64, "few"), (40000, 40, "few"), (33, 5, "identical"), (70000, 8, "identical"), (513, 1, "random"),
               (513, 2, "random"), (513, 513, "random"), (2049, 2049, "lattice"), (131073, 2, "lattice"), (257, 257, "few")]


def _fps_case_id(N, G, kind):
    c, p = fps_route(N)
    return _id(_fps_kernel(N), c=c, T=2 ** fps_log2T(N), N=N, G=G, kind=kind)


@pytest.mark.parametrize("N,G,kind", _FPS_CASES, ids=[_fps_case_id(*c) for c in _FPS_CASES])
def test_fps(N, G, kind):
    """Every plan and tie-break boundary of N, on random clouds, lattices (equal maxima), duplicated points, clouds with
    fewer distinct points than G (the maximum reaches 0 and the previous index repeats) and identical points; B = 2 below
    16385 points."""
    B = 2 if N <= 16384 else 1
    xyz = torch.stack([_cloud(kind, N, 1000 * N + 7 * b + G, distinct=max(G // 3, 1) if kind == "few" else None) for b in range(B)])
    idx, cen = _run_fps(xyz, G)
    _check_fps(xyz, G, idx, cen, f"N={N} G={G} {kind}")
    if kind == "identical":
        assert bool((idx == 0).all())


_FPS_VARLEN = [(8193, [32, 33, 512, 513, 4097, 8193, 64, 65], 40), (65537, [63, 1025, 65537, 16385], 24),
               (300, [1, 2, 300, 257], 8), (131073, [131073, 8192, 33], 16)]


@pytest.mark.parametrize("Nmax,lengths,G", _FPS_VARLEN,
                         ids=[_id(_fps_kernel(n, True), c=fps_route(n)[0], Nmax=n, B=len(l), G=g) for (n, l, g) in _FPS_VARLEN])
def test_fps_varlen(Nmax, lengths, G):
    """Clouds whose lengths sit on plan and T boundaries, inside one padded batch whose N_max lies in another plan.  The
    padding rows are far points (a kernel that read them would pick them); slots past a cloud's length repeat sample 0."""
    B = len(lengths)
    xyz = torch.stack([_cloud("random" if b % 2 else "lattice", Nmax, 31 * b + Nmax) for b in range(B)])
    for b, L in enumerate(lengths):
        xyz[b, L:] = 1e3 + torch.rand(Nmax - L, 3, generator=_gen(b))
    idx, cen = _run_fps(xyz, G, lengths)
    for b, L in enumerate(lengths):
        g = min(G, L)
        _check_fps(xyz[b:b + 1, :L], g, idx[b:b + 1, :g], cen[b:b + 1, :g], f"varlen cloud {b} L={L}")
        assert bool((idx[b, g:] == 0).all())
        _assert_bits(cen[b, g:], xyz[b, 0].expand(G - g, 3), "varlen repeated slots")


# ------------------------------------------------------------------------------------------------
# kNN
# ------------------------------------------------------------------------------------------------
def _run_knn(query, key, K, lengths=None, key_offset=0, want_d2=True, same=False):
    nv = _nv()
    B, Q, _ = query.shape
    N = key.shape[1]
    k = Win(key, offset=key_offset)
    q = k if same else Win(query)
    idx, d2 = Win(shape=(B, Q, K), dtype=torch.int64, fill=-7), Win(shape=(B, Q, K)) if want_d2 else None
    if lengths is None:
        rc = nv.lib().psam_knn_f32(q.ptr, k.ptr, B, Q, N, K, idx.ptr, d2.ptr if d2 else None, nv.stream())
    else:
        ln = torch.tensor(lengths, dtype=torch.int32, device=_dev())
        rc = nv.lib().psam_knn_varlen_f32(q.ptr, k.ptr, ln.data_ptr(), B, Q, N, K, idx.ptr, d2.ptr if d2 else None, nv.stream())
    assert rc == 0
    for w, name in ((q, "query"), (k, "key"), (idx, "idx")) + (((d2, "d2"),) if d2 else ()):
        w.check(name)
    return idx.cpu(), (d2.cpu() if d2 else None)


def _check_knn(query, key, K, idx, d2, name, semantic=True):
    from oracle import tokenizer_ref

    widx, wd2 = tokenizer_ref.knn(query.numpy(), key.numpy(), K)
    got = idx.numpy()
    assert np.array_equal(got, widx), f"{name}: {int((got != widx).sum())} indices differ, first at {np.argwhere(got != widx)[:3].tolist()}"
    if d2 is not None:
        _assert_bits(d2, torch.from_numpy(wd2), f"{name} d2")
        dd, ii = d2.numpy(), got
        ok = (dd[..., 1:] > dd[..., :-1]) | ((dd[..., 1:] == dd[..., :-1]) & (ii[..., 1:] > ii[..., :-1]))
        assert ok.all(), f"{name}: a row is not sorted by (d2, index)"
    if semantic:
        ex = max(knn_set_excess(query[b].numpy(), key[b].numpy(), got[b]) for b in range(len(query)))
        print(f"[geom] knn {name}: set excess {ex:.3f} of its bound")
        assert ex <= 1.0


def _queries(key, Q, seed, jitter=0.05):
    g = _gen(seed)
    B, N, _ = key.shape
    pick = torch.randint(0, N, (B, Q), generator=g)
    return (key[torch.arange(B)[:, None], pick] + jitter * torch.randn(B, Q, 3, generator=g)).contiguous()


_SWEEPS = {"vec": (1004, 0), "pointwise_misaligned": (1004, 1), "pointwise_ragged": (1001, 0)}
_KNN_C = [(2, 445), (2, 223), (2, 101)]  # C = 4, 2, 1 at K = 9, each with Q % C != 0 where C > 1
_KNN_C_CASES = [(B, Q, sw) for (B, Q) in _KNN_C for sw in _SWEEPS]


@pytest.mark.parametrize("B,Q,sweep", _KNN_C_CASES,
                         ids=[_id(_knn_kernel(B, Q, _SWEEPS[sw][0], 9), sweep=sw, B=B, Q=Q) for (B, Q, sw) in _KNN_C_CASES])
def test_knn_c_and_sweep(B, Q, sweep):
    """Each centres-per-CTA instantiation with a ragged last group, under the vectorised sweep (N % 4 == 0, 16-byte aligned
    clouds) and the point-wise one (a cloud pointer misaligned by 4 bytes, or N % 4 != 0)."""
    N, off = _SWEEPS[sweep]
    key = torch.rand(B, N, 3, generator=_gen(Q)) * 2 - 1
    query = _queries(key, Q, Q + 1)
    idx, d2 = _run_knn(query, key, 9, key_offset=off)
    _check_knn(query, key, 9, idx, d2, f"C sweep {sweep} B={B} Q={Q}")


_KNN_K = [(1, 2, 300, 5000), (3, 1, 256, 5000), (9, 1, 256, 5000), (64, 2, 500, 5000), (256, 1, 300, 4096),
          (1023, 1, 37, 2000), (1024, 1, 889, 2000), (64, 1, 64, 64), (200, 2, 130, 200), (16, 2, 40, 16)]


@pytest.mark.parametrize("K,B,Q,N", _KNN_K, ids=[_id(_knn_kernel(B, Q, N, K), K=K, B=B, Q=Q, N=N) for (K, B, Q, N) in _KNN_K])
def test_knn_k(K, B, Q, N):
    """K from 1 to the 1024 limit (1024 takes the C the shared memory allows, not the occupancy rule), and K = N."""
    key = torch.rand(B, N, 3, generator=_gen(K)) * 2 - 1
    query = _queries(key, Q, K + 1)
    idx, d2 = _run_knn(query, key, K)
    _check_knn(query, key, K, idx, d2, f"K={K} B={B} Q={Q} N={N}")


def _knn_special(case):
    """(query, key, K, key_offset, semantic) of the constructed cases."""
    g = _gen(zlib.crc32(case.encode()))
    if case.startswith("coincident_beyond_cap"):
        N, K = 5000, 9
        key = torch.rand(1, N, 3, generator=g) * 2 - 1
        query = key[:, :64].clone()
        C, cap = knn_plan(1, 64, N, K)
        key[0, torch.randperm(N, generator=g)[:cap + 48]] = query[0, 5]  # more than cap keys at distance 0 from query 5
        return query, key, K, 1 if case.endswith("pointwise") else 0, True
    if case == "identical_cloud":
        key = torch.full((1, 5000, 3), 0.25)
        return key[:, :70].clone(), key, 9, 0, True
    if case == "offset_1e-3_spacing":
        key = (_lattice(4096, 5) * 1e-3 + torch.tensor([512.0, 300.0, 1000.0]))[None]
        return _queries(key, 80, 6, jitter=2e-3), key, 9, 0, True
    if case.startswith("lattice_ties"):
        key = _lattice(4096, 7)[None]
        K = 9 if "9" in case else 27
        q = key[:, :60].clone()
        q[:, 30:] += 0.5  # cell centres: 8 keys at 0.75, 24 at 2.75
        return q, key, K, 1 if case.endswith("pointwise") else 0, True
    if case.startswith("subnormal"):
        key = (torch.rand(1, 4096, 3, generator=g) * 2 - 1) * 2.0 ** -64
        return _queries(key, 100, 8, jitter=2.0 ** -70), key, 9, 1 if case.endswith("pointwise") else 0, False
    if case == "far_query":
        key = torch.rand(1, 3000, 3, generator=g) * 2 - 1
        q = _queries(key, 64, 9)
        q[0, 7] = torch.tensor([1e15, -1e15, 1e15])
        return q, key, 16, 0, True
    raise ValueError(case)


_KNN_SPECIAL = ["coincident_beyond_cap", "coincident_beyond_cap_pointwise", "identical_cloud", "offset_1e-3_spacing",
                "lattice_ties_9", "lattice_ties_27", "lattice_ties_9_pointwise", "subnormal", "subnormal_pointwise", "far_query"]


def _special_id(case):
    q, k, K, off, _ = _knn_special(case)
    return _id(_knn_kernel(1, q.shape[1], k.shape[1], K), case=case, K=K, cap=knn_plan(1, q.shape[1], k.shape[1], K)[1])


@pytest.mark.parametrize("case", _KNN_SPECIAL, ids=[_special_id(c) for c in _KNN_SPECIAL])
def test_knn_special(case):
    """The candidate-overflow fallback (more than cap keys at distance 0 from a query; an identical cloud), the
    over-accepting sweep filter (a cloud offset by 300-1000 with 1e-3 spacing: the bias of the 3-FMA filter,
    2e-6 (|p|^2 + |c|^2) ~ 3, admits every key, and the exact re-test against tau must drop all but the true candidates),
    ties at the K-th distance on a lattice (queries on lattice points and at cell centres), subnormal distances (denormals
    are kept) and a query far from every key.  The fp64 check is skipped for subnormal distances, where rounding is
    absolute."""
    query, key, K, off, semantic = _knn_special(case)
    idx, d2 = _run_knn(query, key, K, key_offset=off)
    _check_knn(query, key, K, idx, d2, case, semantic=semantic)
    if case == "subnormal":
        assert bool(((d2 > 0) & (d2 < 2.0 ** -126)).any()), "fixture: distances must be subnormal"


def test_knn_self():
    """Self-kNN (query = key, one buffer, Q = N) as small-region cleanup builds its graph, k = 9."""
    key = torch.rand(1, 3001, 3, generator=_gen(11)) * 2 - 1
    idx, d2 = _run_knn(key, key, 9, same=True)
    _check_knn(key, key, 9, idx, d2, "self")
    assert bool((idx[0, :, 0] == torch.arange(3001)).all()) and bool((d2[..., 0] == 0).all())


_KNN_VARLEN = [(1004, [5, 1004, 517, 800], 223), (1001, [1000, 1001, 8, 4], 111), (1004, [9, 1004, 1000, 12], 50)]


@pytest.mark.parametrize("Nmax,lengths,Q", _KNN_VARLEN,
                         ids=[_id(_knn_kernel(len(l), q, n, 9, True), Nmax=n, B=len(l), Q=q) for (n, l, q) in _KNN_VARLEN])
def test_knn_varlen(Nmax, lengths, Q):
    """Lengths below K (the cloud's first K rows are its keys), equal to N_max, and clouds whose pointers are not 16-byte
    aligned (N_max = 1001).  Padding rows coincide with the queries, so a kernel that read them would choose them."""
    B, K = len(lengths), 9
    key = torch.rand(B, Nmax, 3, generator=_gen(Nmax + Q)) * 2 - 1
    query = _queries(key, Q, Q)
    for b, L in enumerate(lengths):
        n = max(L, K)
        key[b, n:] = query[b, torch.arange(Nmax - n) % Q]
    idx, d2 = _run_knn(query, key, K, lengths=lengths)
    for b, L in enumerate(lengths):
        n = max(L, K)
        _check_knn(query[b:b + 1], key[b:b + 1, :n], K, idx[b:b + 1], d2[b:b + 1], f"varlen cloud {b} L={L}")


def test_knn_without_d2():
    key = torch.rand(2, 1004, 3, generator=_gen(12)) * 2 - 1
    query = _queries(key, 445, 13)
    idx, _ = _run_knn(query, key, 16, want_d2=False)
    _check_knn(query, key, 16, idx, None, "d2_out NULL")


# ------------------------------------------------------------------------------------------------
# psam_nn_distance_f32
# ------------------------------------------------------------------------------------------------
def _run_nn(q, k, want_idx=True):
    nv = _nv()
    qw, kw = Win(q), Win(k)
    dist, idx = Win(shape=(len(q),)), Win(shape=(len(q),), dtype=torch.int64, fill=-7) if want_idx else None
    assert nv.lib().psam_nn_distance_f32(qw.ptr, kw.ptr, len(q), len(k), dist.ptr, idx.ptr if idx else None, nv.stream()) == 0
    for w, name in ((qw, "query"), (kw, "key"), (dist, "dist")) + (((idx, "idx"),) if idx else ()):
        w.check(name)
    return dist.cpu(), (idx.cpu() if idx else None)


@pytest.mark.parametrize("n1,n2,want_idx", [(1000, 777, True), (300, 1, True), (257, 513, False), (4097, 2000, True)],
                         ids=["n1_1000-n2_777", "n2_1", "idx_null", "n1_4097-n2_2000"])
def test_nn_distance(n1, n2, want_idx):
    """Against the C oracle's kNN at K = 1 (distance and lower index on ties), with lattice keys so ties occur."""
    from oracle import tokenizer_ref

    k = _lattice(n2, n1) if n2 > 1 else torch.rand(1, 3, generator=_gen(1))
    q = (_lattice(n1, n2) + torch.randint(0, 2, (n1, 3), generator=_gen(n1)) * 0.5).contiguous()
    dist, idx = _run_nn(q, k, want_idx)
    widx, wd2 = tokenizer_ref.knn(q.numpy()[None], k.numpy()[None], 1)
    _assert_bits(dist, torch.from_numpy(wd2[0, :, 0]), "nn dist")
    if want_idx:
        assert np.array_equal(idx.numpy(), widx[0, :, 0])


def test_nn_distance_non_finite():
    """A NaN or inf key is never chosen; a NaN or inf query gets (3.4e38, -1), as the header states."""
    from oracle import tokenizer_ref

    k = torch.rand(600, 3, generator=_gen(21)) * 2 - 1
    bad = torch.tensor([3, 100, 255, 256, 599])
    q = torch.rand(300, 3, generator=_gen(22)) * 2 - 1
    q[:5] = k[bad] + 1e-3  # right next to where a key turns non-finite
    k[bad[:3], 1] = float("nan")
    k[bad[3:], 0] = float("inf")
    q[10, 2], q[11, 0] = float("nan"), float("-inf")
    dist, idx = _run_nn(q, k)
    good = torch.ones(600, dtype=torch.bool)
    good[bad] = False
    fin = torch.ones(300, dtype=torch.bool)
    fin[[10, 11]] = False
    widx, wd2 = tokenizer_ref.knn(q[fin].numpy()[None], k[good].numpy()[None], 1)
    assert np.array_equal(idx[fin].numpy(), torch.nonzero(good)[:, 0].numpy()[widx[0, :, 0]])
    _assert_bits(dist[fin], torch.from_numpy(wd2[0, :, 0]), "nn dist, finite queries")
    assert dist[10].item() == np.float32(3.4e38) and dist[11].item() == np.float32(3.4e38)
    assert idx[10].item() == -1 and idx[11].item() == -1


# ------------------------------------------------------------------------------------------------
# psam_group_gather_f32
# ------------------------------------------------------------------------------------------------
def _group_want(xyz, feats, centers, knn_idx, center_idx, rep, radius):
    """The header's roundings on the host: fp32(p - c) times fp32(1 / radius), copies, fp32(f - f_centre)."""
    B2 = feats.shape[0]
    bo = torch.arange(B2) // rep
    d = xyz[bo[:, None, None], knn_idx[bo]] - centers[bo][:, :, None, :]
    if radius:
        d = d * (torch.tensor(1.0) / torch.tensor(radius, dtype=torch.float32))
    f = feats[torch.arange(B2)[:, None, None], knn_idx[bo]]
    parts = [d, f]
    if center_idx is not None:
        parts.append(f - feats[torch.arange(B2)[:, None], center_idx[bo]][:, :, None, :])
    return torch.cat(parts, -1)


def _run_group(xyz, feats, centers, knn_idx, center_idx, rep, radius):
    nv = _nv()
    B, N, _ = xyz.shape
    B2, _, C = feats.shape
    _, G, K = knn_idx.shape
    w = [Win(xyz), Win(feats), Win(centers), Win(knn_idx, fill=-7), Win(center_idx, fill=-7) if center_idx is not None else None]
    out = Win(shape=(B2, G, K, 3 + C + (C if center_idx is not None else 0)))
    rc = nv.lib().psam_group_gather_f32(w[0].ptr, w[1].ptr, w[2].ptr, w[3].ptr, w[4].ptr if w[4] else None, B, rep, N, G, K, C,
                                        float(radius or 0.0), out.ptr, nv.stream())
    assert rc == 0
    for x in w + [out]:
        if x is not None:
            x.check("group gather")
    return out.cpu()


_GG = [(r, C, ci) for r in (None, 0.05, 0.1, 0.5) for C in (0, 1, 3, 128) for ci in (False, True)]


@pytest.mark.parametrize("radius,C,centre", _GG, ids=[f"group_gather_kernel-r{r}-C{C}-{'centred' if ci else 'plain'}-rep{(1, 2, 4)[i % 3]}"
                                                      for i, (r, C, ci) in enumerate(_GG)])
def test_group_gather(radius, C, centre):
    """Every value exact: coordinates fp32(p - c) times fp32(1 / radius) (radius None, 0.05, 0.1 and the power of two 0.5),
    feature copies, centralised features fp32(f - f_centre); rep = 1, 2, 4 prompt copies per cloud; the indices include
    the last point."""
    rep = (1, 2, 4)[_GG.index((radius, C, centre)) % 3]
    B, N, G, K = 2, 517, 33, 7
    g = _gen(int((radius or 0) * 100) + 10 * C + centre)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    feats = torch.randn(B * rep, N, C, generator=g)
    knn_idx = torch.randint(0, N, (B, G, K), generator=g)
    knn_idx[:, ::5, -1] = N - 1
    center_idx = torch.randint(0, N, (B, G), generator=g) if centre else None
    centers = xyz[torch.arange(B)[:, None], torch.randint(0, N, (B, G), generator=g)]
    got = _run_group(xyz, feats, centers, knn_idx, center_idx, rep, radius)
    _assert_bits(got, _group_want(xyz, feats, centers, knn_idx, center_idx, rep, radius), "group gather")


@pytest.mark.parametrize("shape", [(1, 2, 1024, 600, 1, 0.1), (2, 1, 40, 1, 128, 0.05)],
                         ids=["group_gather_kernel-grid_stride_1228800_rows-r0.1", "group_gather_kernel-K1-C128-last_point-r0.05"])
def test_group_gather_shapes(shape):
    """More rows than one grid-stride pass (132 * 16 * 256 = 540672), and K = 1 with every index at the last point."""
    B, rep, G, K, C, radius = shape
    N = 2000
    g = _gen(K)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    feats = torch.randn(B * rep, N, C, generator=g)
    knn_idx = torch.randint(0, N, (B, G, K), generator=g) if K > 1 else torch.full((B, G, K), N - 1)
    center_idx = torch.randint(0, N, (B, G), generator=g)
    centers = xyz[:, :G].clone()
    got = _run_group(xyz, feats, centers, knn_idx, center_idx, rep, radius)
    _assert_bits(got, _group_want(xyz, feats, centers, knn_idx, center_idx, rep, radius), "group gather")


def test_torch_cuda_divides_by_scalar_through_its_reciprocal():
    """The premise of the group gather's rounding: torch on CUDA computes `tensor / radius` for a Python-float radius as
    tensor * fp32(1 / fp32(radius)), which differs from an fp32 division (what torch does on the CPU) for some values."""
    x = (torch.rand(200000, generator=_gen(31)) * 2 - 1)
    for r in (0.05, 0.1):
        inv = (torch.tensor(1.0) / torch.tensor(r, dtype=torch.float32)).item()
        gpu = (x.to(_dev()) / r).cpu()
        _assert_bits(gpu, x * inv, f"CUDA x / {r}")
        frac = float((_bits(x / r) != _bits(x * inv)).double().mean())
        print(f"[geom] radius {r}: fp32 division and the reciprocal product differ in {100 * frac:.2f} % of 200000 values")
        assert frac > 0.005


# ------------------------------------------------------------------------------------------------
# psam_voronoi_features_f32
# ------------------------------------------------------------------------------------------------
def _voronoi_inputs(B, rep, N, G, C, seed):
    g = _gen(seed)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    sel = torch.randperm(N, generator=g)[:G]
    sel[0] = 1  # point 1 is a centre: distance 0
    centers = xyz[:, sel].clone()
    nn_idx = torch.cdist(xyz.double(), centers.double()).argmin(-1)
    feats = torch.randn(B * rep, N, C, generator=g)
    return xyz, centers, nn_idx, feats


def _run_voronoi(xyz, centers, nn_idx, feats, rep, form, pitch):
    nv = _nv()
    B, N, _ = xyz.shape
    G, C = centers.shape[1], feats.shape[2]
    rows = B * rep * N
    w = [Win(xyz), Win(centers), Win(nn_idx, fill=-7), Win(feats)]
    out = Win(shape=(B * rep, N, 4 + C)) if form in ("f32", "both") else None
    sp = Win(shape=(2, rows, pitch), dtype=torch.bfloat16) if form in ("split", "both") else None
    rc = nv.lib().psam_voronoi_features_f32(w[0].ptr, w[1].ptr, w[2].ptr, w[3].ptr, B, rep, N, G, C, out.ptr if out else None,
                                            sp.ptr if sp else None, rows * pitch if sp else 0, pitch if sp else 0, nv.stream())
    assert rc == 0
    for x in w + [out, sp]:
        if x is not None:
            x.check("voronoi")
    return (out.cpu() if out else None), (sp.cpu() if sp else None)


def _check_voronoi(xyz, centers, nn_idx, rep, out):
    """Direction == fp32(d / max(dist, 1e-8)) bit for bit given the kernel's own dist; dist within 2.5u of the fp64 norm."""
    B = xyz.shape[0]
    bo = torch.arange(B * rep) // rep
    d = xyz[bo] - centers[bo[:, None], nn_idx[bo]]
    dist = out[..., 3]
    _assert_bits(out[..., :3], d / torch.clamp(dist, min=1e-8)[..., None], "voronoi direction")
    ex = max(voronoi_dist_excess(xyz[b], centers[b], nn_idx[b], out[b * rep, :, 3]) for b in range(B))
    print(f"[geom] voronoi dist: excess {ex:.3f} of its 2.5u bound")
    assert ex <= 1.0


_VOR = [("f32", 1, 3, None), ("f32", 3, 0, None), ("split", 2, 3, 64), ("both", 3, 0, 4), ("both", 2, 5, 16), ("both", 1, 128, 136)]


@pytest.mark.parametrize("form,rep,C,pitch", _VOR, ids=[f"voronoi_features_kernel-{f}-rep{r}-C{c}-pitch{p}" for (f, r, c, p) in _VOR])
def test_voronoi(form, rep, C, pitch):
    """fp32 output only, split only and both; pitch above 4 + C (the pad columns must be zero); rep > 1; point 1 of every
    cloud sits on its centre (dist 0, then the 1e-8 clamp)."""
    B, N, G = 2, 3001, 64
    xyz, centers, nn_idx, feats = _voronoi_inputs(B, rep, N, G, C, 41 + C)
    out, sp = _run_voronoi(xyz, centers, nn_idx, feats, rep, form, pitch)
    if out is None:  # split only: the planes must be the split of what the fp32 output holds (a second call writes it)
        out, _ = _run_voronoi(xyz, centers, nn_idx, feats, rep, "f32", pitch)
    _check_voronoi(xyz, centers, nn_idx, rep, out)
    assert bool((out[:, 1, :4] == 0).all())
    _assert_bits(out[..., 4:], feats, "voronoi features")
    if sp is not None:
        v = out.reshape(-1, 4 + C)
        hi = v.to(torch.bfloat16)
        lo = (v - hi.float()).to(torch.bfloat16)
        assert torch.equal(sp[0, :, :4 + C].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(sp[1, :, :4 + C].view(torch.int16), lo.view(torch.int16))
        assert bool((sp[:, :, 4 + C:].float() == 0).all()), "pad columns not zero-filled"


def test_voronoi_worst_case_distance():
    """An offset whose dist rounds to 0.85 of the 2.5u bound (1.07 times 2u) when its first coordinate is squared first,
    from a centre at the origin, in all six axis orders (one of them meets the kernel's summation order): the bound the
    header states is needed, and the kernel stays inside it."""
    v = (1.0175834894180298, -0.23071885108947754, 0.053580403327941895)
    xyz = torch.tensor([[list(o) for o in itertools.permutations(v)] + [[0.0, 0.0, 0.0]]])
    centers = torch.zeros(1, 1, 3)
    nn_idx = torch.zeros(1, 7, dtype=torch.int64)
    out, _ = _run_voronoi(xyz, centers, nn_idx, torch.zeros(1, 7, 0), 1, "f32", None)
    _check_voronoi(xyz, centers, nn_idx, 1, out)
    assert voronoi_dist_excess(xyz[0], centers[0], nn_idx[0], out[0, :, 3]) > 0.8, "the kernel's dist must round as stated"


def test_voronoi_grid_stride():
    """More rows than one grid-stride pass: B * rep * N = 600000 > 132 * 16 * 256."""
    xyz, centers, nn_idx, feats = _voronoi_inputs(2, 2, 150000, 16, 1, 51)
    out, _ = _run_voronoi(xyz, centers, nn_idx, feats, 2, "f32", None)
    _check_voronoi(xyz, centers, nn_idx, 2, out)


# ------------------------------------------------------------------------------------------------
# psam_border_prompt_f32
# ------------------------------------------------------------------------------------------------
def _border_want(xyz, gt, logits, mode):
    """Per (cloud, mask): oracle.torch_ref.sample_fixed_points, or None where the reference fails (no candidate)."""
    from oracle import torch_ref

    B, M, N = gt.shape
    want = []
    for b in range(B):
        for m in range(M):
            lg = logits[b * M + m][None] if logits is not None else None
            try:
                c, l = torch_ref.sample_fixed_points(xyz[b:b + 1], gt[b:b + 1, m:m + 1], lg, None, mode == 0)
                want.append((c.reshape(3), bool(l.reshape(-1)[0])))
            except TypeError:  # torch.stack of None
                want.append(None)
    return want


def _run_border(xyz, gt, logits, masks, mode, status=None):
    nv = _nv()
    B, M, N = gt.shape
    c, g = Win(xyz), Win(gt.to(torch.uint8), fill=7)
    lg = Win(logits) if logits is not None else None
    pm = Win(masks.to(torch.uint8), fill=7) if masks is not None else None
    out, lab = Win(shape=(B * M, 3)), Win(shape=(B * M,), dtype=torch.uint8, fill=0xA5)
    st = Win(torch.tensor([status or 0], dtype=torch.int32), fill=-9)
    ws = Win(shape=(nv.lib().psam_border_prompt_workspace_bytes(B, M, N) // 4,), dtype=torch.int32, fill=-5)
    rc = nv.lib().psam_border_prompt_f32(c.ptr, g.ptr, lg.ptr if lg else None, pm.ptr if pm else None, B, M, N, int(mode == 0),
                                         out.ptr, lab.ptr, st.ptr, ws.ptr, nv.stream())
    assert rc == 0
    for x in (c, g, lg, pm, out, lab, st, ws):
        if x is not None:
            x.check("border prompt")
    return out.cpu(), lab.cpu(), int(st.cpu()[0])


def _check_border(xyz, gt, forms, mode, name, expect_status=None):
    """Kernel against the oracle; a pair the reference cannot sample must give zeros and status 1."""
    want = _border_want(xyz, gt, forms[0], mode)
    out, lab, st = _run_border(xyz, gt, forms[1], forms[2], mode)
    for i, w in enumerate(want):
        if w is None:
            assert bool((out[i] == 0).all()) and int(lab[i]) == 0, f"{name}: pair {i} without a candidate is not zero"
        else:
            _assert_bits(out[i], w[0], f"{name}: pair {i} coordinates")
            assert bool(lab[i]) == w[1], f"{name}: pair {i} label"
    assert st == (1 if any(w is None for w in want) else 0), f"{name}: status {st}"
    if expect_status is not None:
        assert st == expect_status, f"{name}: fixture should give status {expect_status}"
    return want


def _pred_forms(pred_bool, form, g):
    """(oracle logits, kernel logits, kernel byte masks) for one prediction.  Logits put 0.0 and -0.0 (not > 0) on a
    tenth of the negatives; the oracle reads byte masks in their logits form +-1."""
    if form == "none":
        return None, None, None
    if form == "bytes":
        return pred_bool.float() * 2 - 1, None, pred_bool
    lg = torch.where(pred_bool, torch.rand(pred_bool.shape, generator=g) + 0.01, -torch.rand(pred_bool.shape, generator=g))
    z = (~pred_bool) & (torch.rand(pred_bool.shape, generator=g) < 0.1)
    lg[z] = torch.where(torch.rand(pred_bool.shape, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))[z]
    return lg, lg, None


def _spheres(xyz, M, g, r=(0.3, 0.8)):
    B, N, _ = xyz.shape
    c = xyz[torch.arange(B)[:, None], torch.randint(0, N, (B, M), generator=g)]
    rad = r[0] + (r[1] - r[0]) * torch.rand(B, M, 1, generator=g)
    return (xyz[:, None] - c[:, :, None]).norm(dim=-1) < rad


@pytest.mark.parametrize("mode", [0, 1], ids=["error_region", "fn_fp_gt"])
@pytest.mark.parametrize("form", ["none", "logits", "bytes"])
@pytest.mark.parametrize("size", ["batch_4x64_N300", "blocks_N5000"])
def test_border_prompt(size, form, mode):
    """Both modes, each prediction form; a batch of 256 (cloud, mask) pairs, or one cloud of 5000 points (not a multiple of
    256) whose regions hold more than 512 foreground and 2048 background points, so several blocks meet in the atomicMin."""
    g = _gen(zlib.crc32(f"{size}{form}{mode}".encode()))
    B, M, N = (4, 64, 300) if size.startswith("batch") else (1, 3, 5000)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    gt = _spheres(xyz, M, g) if N < 1000 else xyz[:, None, :, 0] < torch.rand(B, M, 1, generator=g) * 0.2 - 0.1  # half-spaces
    flip = torch.rand(B, M, N, generator=g) < (0.3 if N > 1000 else 0.15)
    pred = (gt ^ flip).reshape(B * M, N)
    want = _check_border(xyz, gt, _pred_forms(pred, form, g), mode, f"{size} {form} mode{mode}")
    if N > 1000 and form != "none":
        fn = (gt.reshape(B * M, N) & ~pred).sum(-1)
        assert bool((fn > 512).all() and (N - fn > 2048).all()), "fixture: regions must span several blocks"
    assert sum(w is not None for w in want) > 0


def _line_lattice(seed):
    """Points (x, y, z), x in 0..24, y, z in {0, 1}, in random order: gt = x < 20, pred = 5 <= x < 25.  The fn region
    x < 5 and the fp region x >= 20 are both 5 columns deep: pd == nd == 25, with four tied points at each end."""
    p = torch.stack(torch.meshgrid(torch.arange(25), torch.arange(2), torch.arange(2), indexing="ij"), -1).reshape(-1, 3).float()
    p = p[torch.randperm(100, generator=_gen(seed))]
    return p, p[:, 0] < 20, (p[:, 0] >= 5)


_REGIONS = ["fn_empty", "fp_empty", "both_empty", "pd_equals_nd", "lattice_ties"]


@pytest.mark.parametrize("mode", [0, 1], ids=["error_region", "fn_fp_gt"])
@pytest.mark.parametrize("form", ["logits", "bytes"])
@pytest.mark.parametrize("region", _REGIONS)
def test_border_prompt_regions(region, form, mode):
    """The selection rules: fn empty, fp empty, both empty (mode 1 falls back to the ground truth; mode 0 has no
    candidate), pd == nd (the reference's `not pd > nd` takes fp), and lattice clouds where the lowest index wins ties."""
    g = _gen(_REGIONS.index(region) + 10 * mode)
    if region in ("pd_equals_nd",):
        pts = [_line_lattice(s) for s in (1, 2)]
        xyz = torch.stack([p[0] for p in pts])
        gt = torch.stack([p[1] for p in pts])[:, None]
        pred = torch.stack([p[2] for p in pts])
    else:
        B, M, N = 2, 6, 343
        xyz = torch.stack([_lattice(N, s) for s in (3, 4)])
        gt = _spheres(xyz, M, g, r=(2.0, 3.5))
        flip = torch.rand(B, M, N, generator=g) < 0.2
        if region == "fn_empty":
            pred = gt | flip
        elif region == "fp_empty":
            pred = gt & ~flip
        elif region == "both_empty":
            pred = gt.clone()
        else:
            pred = gt ^ flip
        pred = pred.reshape(B * M, N)
    want = _check_border(xyz, gt, _pred_forms(pred, form, g), mode, f"{region} {form} mode{mode}",
                         expect_status=1 if (region == "both_empty" and mode == 0) else 0)
    if region == "pd_equals_nd" and mode == 1:
        assert all(not w[1] for w in want), "pd == nd must sample the fp region (label 0)"


@pytest.mark.parametrize("mode", [0, 1], ids=["error_region", "fn_fp_gt"])
def test_border_prompt_status(mode):
    """An empty and a full ground truth have no candidate: their outputs are zero and status becomes 1.  Status is sticky:
    a second call on valid masks leaves it at 1 (the caller clears it)."""
    g = _gen(61 + mode)
    B, M, N = 2, 4, 700
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    gt = _spheres(xyz, M, g)
    gt[0, 1] = False
    gt[1, 2] = True
    _check_border(xyz, gt, (None, None, None), mode, f"status mode{mode}", expect_status=1)
    gt2 = _spheres(xyz, M, g)
    want = _border_want(xyz, gt2, None, mode)
    out, lab, st = _run_border(xyz, gt2, None, None, mode, status=1)
    assert st == 1
    for i, w in enumerate(want):
        _assert_bits(out[i], w[0], "after status")


# ------------------------------------------------------------------------------------------------
# the fp64 checks have teeth (host only: no kernel runs)
# ------------------------------------------------------------------------------------------------
def test_checks_have_teeth():
    """Each check rejects a wrong answer: the fp64 kNN check a neighbour swapped for the (K+1)-th, the fp64 FPS check one
    pick replaced by the runner-up, and the Voronoi check a direction built from the second-nearest centre (the direction
    is checked bit for bit given the kernel's dist) as well as a distance measured to it (the fp64 distance check)."""
    from oracle import tokenizer_ref

    g = _gen(71)
    key = torch.rand(1, 2000, 3, generator=g) * 2 - 1
    query = key[:, :50] + 0.01
    widx, _ = tokenizer_ref.knn(query.numpy(), key.numpy(), 17)
    right, wrong = widx[0, :, :16].copy(), widx[0, :, :16].copy()
    wrong[7, 15] = widx[0, 7, 16]
    assert knn_set_excess(query[0], key[0], right) <= 1.0 < knn_set_excess(query[0], key[0], wrong)

    xyz = torch.rand(3000, 3, generator=g) * 2 - 1
    idx = tokenizer_ref.fps(xyz.numpy()[None], 20)[0]
    x = xyz.double().numpy()
    md = np.full(3000, np.inf)
    for i in range(1, 12):
        md = np.minimum(md, ((x - x[idx[i - 1]]) ** 2).sum(1))
    bad = idx.copy()
    bad[11] = np.argsort(md)[-2]  # the runner-up of step 11
    assert fps_greedy_excess(xyz.numpy(), idx) <= 1.0 < fps_greedy_excess(xyz.numpy(), bad)

    centers = xyz[:64].clone()
    d = torch.cdist(xyz.double(), centers.double())
    nn_idx, second = d.argmin(-1), d.topk(2, largest=False).indices[:, 1]
    dist = lambda ci: (xyz - centers[ci]).norm(dim=-1)
    assert voronoi_dist_excess(xyz, centers, nn_idx, dist(nn_idx)) <= 1.0 < voronoi_dist_excess(xyz, centers, nn_idx, dist(second))

    def vor_out(ci):  # [direction, dist] as the kernel writes it, from centre ci (dist correctly rounded)
        dd = xyz - centers[ci]
        dn = dd.double().norm(dim=-1).float()
        return torch.cat([dd / torch.clamp(dn, min=1e-8)[:, None], dn[:, None]], -1)[None]

    _check_voronoi(xyz[None], centers[None], nn_idx[None], 1, vor_out(nn_idx))
    wrong = vor_out(nn_idx)
    wrong[0, :, :3] = vor_out(second)[0, :, :3]
    with pytest.raises(AssertionError, match="voronoi direction"):
        _check_voronoi(xyz[None], centers[None], nn_idx[None], 1, wrong)


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def test_routing_guard():
    """One call per instantiation - fps_cluster_kernel<PPT, VARLEN> for every PPT (0 is the streaming plan) and
    knn_kernel<C, VARLEN> for C = 1, 2, 4 and both VARLEN - under the profiler; the kernel that ran must be the one the case
    ids name, and (from the trace's grid) the FPS cluster width must be the planned one.  It runs in a fresh interpreter,
    as the other routing guards do: what the profiler records must not depend on what ran before it."""
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_geometry_kernels as t; t._routing_guard()" % (
        here, repo, os.path.join(repo, "point-sam_b200"))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def _kernels_launched(fn):
    """(name, grid) of every CUDA kernel fn launches, in launch order (torch.profiler; grid None if the trace lacks it)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel" and "_kernel" in e.get("name", "")), key=lambda e: e["ts"])
    if ks:
        return [(e["name"], (e.get("args") or {}).get("grid")) for e in ks]
    from torch.autograd import DeviceType  # a trace without kernel records: names from the event list, no grids

    es = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and "_kernel" in e.name), key=lambda e: e.time_range.start)
    return [(e.name, None) for e in es]


def _routing_guard():
    nv = _nv()
    calls, keep = [], []

    def fps_call(N, lengths=None):
        xyz = torch.rand(1, N, 3, device=_dev())
        idx, cen = torch.empty(1, 4, dtype=torch.int64, device=_dev()), torch.empty(1, 4, 3, device=_dev())
        nb = nv.lib().psam_fps_workspace_bytes(1, N, 4)
        ws = torch.empty(max(nb, 4), dtype=torch.uint8, device=_dev())
        ln = torch.tensor(lengths or [N], dtype=torch.int32, device=_dev())
        keep.extend([xyz, idx, cen, ws, ln])
        if lengths is None:
            return lambda: nv.lib().psam_fps_f32(xyz.data_ptr(), 1, N, 4, idx.data_ptr(), cen.data_ptr(), ws.data_ptr(), nv.stream())
        return lambda: nv.lib().psam_fps_varlen_f32(xyz.data_ptr(), ln.data_ptr(), 1, N, 4, idx.data_ptr(), cen.data_ptr(),
                                                    ws.data_ptr(), nv.stream())

    fps_ns = [200, 512, 2048, 4096, 8192, 16384, 32768, 65536, 65537, 131072, 131073]
    for N in fps_ns:
        calls.append((_fps_kernel(N), ("fps", N), fps_call(N)))
    for N in (513, 65537):
        calls.append((_fps_kernel(N, True), ("fps", N), fps_call(N, [N - 7])))

    def knn_call(B, Q, N, varlen):
        key = torch.rand(B, N, 3, device=_dev())
        q = key[:, :Q].contiguous()
        idx = torch.empty(B, Q, 9, dtype=torch.int64, device=_dev())
        ln = torch.full((B,), N, dtype=torch.int32, device=_dev())
        keep.extend([key, q, idx, ln])
        if varlen:
            return lambda: nv.lib().psam_knn_varlen_f32(q.data_ptr(), key.data_ptr(), ln.data_ptr(), B, Q, N, 9, idx.data_ptr(), None,
                                                        nv.stream())
        return lambda: nv.lib().psam_knn_f32(q.data_ptr(), key.data_ptr(), B, Q, N, 9, idx.data_ptr(), None, nv.stream())

    for varlen in (False, True):
        for (B, Q) in _KNN_C:
            calls.append((_knn_kernel(B, Q, 1004, 9, varlen), ("knn",), knn_call(B, Q, 1004, varlen)))
    rcs = []
    got = _kernels_launched(lambda: rcs.extend(fn() for _, _, fn in calls))
    assert rcs == [0] * len(calls), f"return codes {rcs}"
    assert len(got) == len(calls), f"{len(calls)} calls launched {len(got)} kernels: {[n for n, _ in got]}"
    # N in 65537..131072 takes the 16-CTA register-resident plan; if the device's probe declines 16-CTA clusters, it takes
    # the streaming plan over 8-CTA clusters instead (and so does every streaming cloud)
    declined = any(w[0] == "fps" and 65536 < w[1] <= 131072 and "fps_cluster_kernel<0," in n for (_, w, _), (n, _) in zip(calls, got))
    mc = 8 if declined else 16
    for (want, what, _), (name, grid) in zip(calls, got):
        if what[0] == "fps":
            want = want.replace("<32,", "<0,") if declined and 65536 < what[1] <= 131072 else want
            c = fps_route(what[1], mc)[0]
            if 65536 < what[1] <= 131072:
                print(f"[geom] FPS N={what[1]}: {name.split('(')[0]}, grid {grid}: "
                      + ("streaming plan, 16-CTA clusters declined" if declined else "register-resident plan on 16-CTA clusters"))
        assert want in name, f"expected {want}, ran {name}"
        if what[0] == "fps" and grid is not None:
            assert grid[0] == c, f"FPS N={what[1]}: grid {grid}, planned cluster width {c}"
    print(f"[geom] routing guard: {len(calls)} calls, each ran the kernel its case id names"
          f"{'' if got[0][1] is not None else ' (the trace has no grids)'}")
