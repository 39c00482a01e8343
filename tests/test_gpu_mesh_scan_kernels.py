"""The mesh, dense-scan and crop-extraction kernels - surface sampling, face centres, mask lifting and the label map
(csrc/mesh.cu), the grid nearest search and the voxel subsample (csrc/scan.cu), and the crop layout, count and gather of
csrc/crops.cu in both BATCH forms - through the C ABI, on every launch path of their host functions.

Each kernel is compared with a plain reference of the same operation: oracle.mesh_ref, oracle.scan_ref and
oracle.amg_crops_ref (numpy, one rounding per operation, in the header's order) bit for bit; the grid search bit for bit
against the brute-force psam_nn_distance_f32, against oracle.tokenizer_ref.knn(q, k, 1) on a subset of the queries, and
against an fp64 check that shares no fp32 formula with the kernel: the chosen key's fp64 squared distance is within
(1 + 10u) of the nearest key's (10u: two distances of five roundings of at most u each).

Every output sits inside a larger buffer prefilled with a sentinel (test_gpu_amg_kernels.Win), and every case compares
the whole buffer: lifted words past ceil(M/32) up to Wm, voxel indices past the kept count (-1) and nothing past S, edge
words up to ceil(n_out/32), batched gather rows past a pair's count.  Every workspace starts dirty (0xA5 bytes), and some
are reused from a larger call first.  Poison inputs are in range but wrong: bits past S in the source rows of a lift and
past N in the label rows, padding rows of batched clouds that would win the bounding box if read (and NaN rows), pairs
outside their ranges.

-0.0 orders below +0.0 in the mesh clamp and in the crop bounding box (include/psam_b200.h); the signed-zero cases pin
that.  Every case id names the launch path it reaches, from the host dispatch restated below; test_routing_guard checks
those names, the conditional launches and the crop count grid under torch.profiler."""
import math
import os

import numpy as np
import pytest
import torch

from test_gpu_amg_kernels import FSENT, GUARD, SENT, Win, _cmp, _id, _kernels_launched, _tf  # noqa: F401

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24
REL = 10 * U
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
DIRT = 0xA5                # every workspace byte before a call
OVR = 512 / 1500           # SAM's default crop overlap ratio


def _nv():
    from psam_b200 import native as nv

    return nv


def _dev():
    return torch.device("cuda:0")


def _dirty(nbytes):
    """A workspace full of leftover bytes (torch allocations are 512-byte aligned)."""
    return torch.full((max(int(nbytes), 16),), DIRT, dtype=torch.uint8, device=_dev())


def _cdiv(a, b):
    return -(-a // b)


def _pack(m, W):
    """bool [K, n] -> [K, W] int32 words (point i = bit i % 32 of word i // 32), zero past n."""
    K, n = m.shape
    pad = np.zeros((K, W * 32), bool)
    pad[:, :n] = m
    return torch.from_numpy(np.packbits(pad, axis=1, bitorder="little").view("<u4").reshape(K, W).view(np.int32).copy())


def _poison_tail(words, n):
    """Sets every bit at or past n of each row of words [K, W] (uint32 view of an int32 tensor)."""
    w = words.numpy().view(np.uint32)
    if n % 32:
        w[:, n // 32] |= np.uint32((0xFFFFFFFF << (n % 32)) & 0xFFFFFFFF)
    w[:, _cdiv(n, 32):] = 0xFFFFFFFF
    return words


# ------------------------------------------------------------------------------------------------
# the host dispatch, restated (test_routing_guard checks it against the kernels that run)
# ------------------------------------------------------------------------------------------------
SCAN = 1024                # elements per CTA of every block scan
MAX_CELLS = 1 << 22        # the grid search's cell cap
COUNT_THREADS, COUNT_MAX_BLOCKS, CHUNK = 256, 512, 1024


def mesh_kernels(F):
    """psam_mesh_sample_f32: the add pass only with more than one chunk of 1024 faces."""
    return (["mesh_area_kernel", "mesh_scan_block_kernel", "mesh_scan_sums_kernel"] + (["mesh_scan_add_kernel"] if F > SCAN else [])
            + ["mesh_sample_kernel"])


def mesh_id(F, colour):
    nb = _cdiv(F, SCAN)  # scan_block_sums loops when the chunk totals outnumber its 1024 threads
    return _id("mesh_sample_kernel", F=F, add=_tf(F > SCAN), sumsloop=_tf(nb > SCAN), colour=colour)


def grid_plan(n2):
    """(cap, nb): psam_nn_grid_f32's cell capacity min(n2, 2^22) and scan chunks ceil((cap + 1) / 1024)."""
    cap = min(max(n2, 1), MAX_CELLS)
    return cap, _cdiv(cap + 1, SCAN)


def grid_kernels(n2):
    _, nb = grid_plan(n2)
    return (["nn_box_kernel", "nn_boxhist_kernel", "nn_setup_kernel", "nn_hist_kernel", "nn_scan_block_kernel"]
            + (["nn_scan_sums_kernel", "nn_scan_add_kernel"] if nb > 1 else []) + ["nn_scatter_kernel", "nn_query_kernel"])


def grid_id(n2, n1, what):
    cap, nb = grid_plan(n2)
    return _id("nn_query_kernel", n2=n2, cap=cap, nb=nb, sums=_tf(nb > 1), sumsloop=_tf(nb > SCAN), n1=n1, keys=what)


VOX_KERNELS = (["vox_quant_kernel"] + ["vox_count_kernel", "vox_step_kernel"] * 5 + ["vox_insert_kernel", "vox_rep_kernel", "vox_list_kernel"]
               + ["vox_hist_kernel", "vox_pick_kernel"] * 8 + ["vox_mark_kernel", "vox_flag_scan_kernel", "nn_scan_sums_kernel",
                                                                 "vox_compact_kernel"])


def vox_id(P, what):
    return _id("vox_compact_kernel", P=P, chunks=_cdiv(P, SCAN), S=what)


def count_grid(N):
    """crop_count_kernel's grid on x: min(ceil(N / 256), 512) CTAs (times B for the batched layout)."""
    return min(_cdiv(N, COUNT_THREADS), COUNT_MAX_BLOCKS)


def layout_id(batch, N, layers):
    return _id(f"crop_count_kernel<{_tf(batch)}>", N=N, T=sum(8 ** i for i in range(layers + 1)), grid=count_grid(N))


def gather_id(batch, N):
    nchunks = _cdiv(N, CHUNK)  # the write kernel's offset loop takes a second pass past 1024 chunks
    return _id(f"crop_gather_write_kernel<{_tf(batch)}>", N=N, chunks=nchunks, offloop=_tf(nchunks > CHUNK))


# ------------------------------------------------------------------------------------------------
# mesh sampling
# ------------------------------------------------------------------------------------------------
def _mesh_run(v, faces, S, seed, vcol=None, uv=None, tex=None, ws=None):
    """psam_mesh_sample_f32 in guarded windows; returns (xyz, rgb, face, stats) windows after checking every guard."""
    nv = _nv()
    L = nv.lib()
    V, F = len(v), len(faces)
    ins = [Win(torch.from_numpy(np.ascontiguousarray(v, F32))), Win(torch.from_numpy(np.ascontiguousarray(faces, np.int32)), fill=0)]
    cw = Win(torch.from_numpy(np.ascontiguousarray(vcol, F32))) if vcol is not None else None
    uw = Win(torch.from_numpy(np.ascontiguousarray(uv, F32))) if uv is not None else None
    tw = Win(torch.from_numpy(np.ascontiguousarray(tex, np.uint8).reshape(-1)), fill=255) if tex is not None else None
    H, Wt, C = tex.shape if tex is not None else (0, 0, 0)
    outs = [Win(shape=(S, 3)), Win(shape=(S, 3)), Win(shape=(S,), dtype=torch.int32, fill=SENT), Win(shape=(3,), dtype=torch.int64, fill=SENT)]
    nb = L.psam_mesh_sample_workspace_bytes(F)
    if ws is None:
        ws = _dirty(nb)
    assert ws.numel() >= nb
    rc = L.psam_mesh_sample_f32(ins[0].ptr, V, ins[1].ptr, F, S, seed, cw.ptr if cw else None, uw.ptr if uw else None,
                                tw.ptr if tw else None, H, Wt, C, *[o.ptr for o in outs], ws.data_ptr(), nv.stream())
    assert rc == 0
    for w, name in zip(ins + [x for x in (cw, uw, tw) if x] + outs, ["v", "faces"] + [n for n, x in (("vcol", cw), ("uv", uw), ("tex", tw)) if x]
                       + ["xyz", "rgb", "face", "stats"]):
        w.check(name)
    return outs


def _mesh_check(v, faces, S, seed, vcol=None, uv=None, tex=None, ws=None, name=""):
    from oracle import mesh_ref

    xyz, rgb, face, stats = _mesh_run(v, faces, S, seed, vcol, uv, tex, ws)
    want = mesh_ref.sample(v, faces, S, seed, vertex_colors=vcol, uv=uv, texture=tex)
    _cmp(stats.cpu(), torch.from_numpy(want[3]), f"{name} stats")
    _cmp(face.cpu(), torch.from_numpy(want[2]), f"{name} face")
    _cmp(xyz.cpu(), torch.from_numpy(want[0]), f"{name} xyz")
    _cmp(rgb.cpu(), torch.from_numpy(want[1]), f"{name} rgb")
    return want


def _mesh(kind, rng):
    """(vertices, faces, vertex colours, uv, texture) of one mesh kind."""
    if kind == "random":  # 3000 faces of mixed sizes, a few bad ones
        V, F = 2000, 3000
        v = (rng.uniform(-1, 1, (V, 3)) * rng.choice([1.0, 1e-3, 0.3], (V, 1))).astype(F32)
        f = rng.integers(0, V, (F, 3)).astype(np.int32)
        f[::97, 1] = V + 3
        f[5::101] = f[5::101, :1]  # zero area
        return v, f, rng.uniform(0, 1, (V, 3)).astype(F32), None, None
    if kind == "flat":  # every face in z = 0.3 or x = -0.7: the barycentric sum misses the plane, the clamp restores it
        V, F = 1500, 500
        v = rng.uniform(-1, 1, (V, 3)).astype(F32)
        v[:V // 2, 2] = F32(0.3)
        v[V // 2:, 0] = F32(-0.7)
        f = np.concatenate([rng.integers(0, V // 2, (F // 2, 3)), rng.integers(V // 2, V, (F // 2, 3))]).astype(np.int32)
        c = np.full((V, 3), F32(0.1))
        return v, f, c, None, None
    if kind == "signed_zero":  # each face flat on one axis at +0.0 / -0.0, colour channels +-0.0 per vertex
        F = 600
        v = rng.uniform(-1, 1, (F * 3, 3)).astype(F32)
        axis = np.repeat(rng.integers(0, 3, F), 3)
        v[np.arange(3 * F), axis] = np.where(rng.random(3 * F) < 0.5, F32(-0.0), F32(0.0))
        v[:3] = [[0.5, 0.25, 0.0], [-0.5, 0.75, 0.0], [0.25, -0.5, -0.0]]  # z = (+0, +0, -0): the bary sum is +0.0
        c = np.where(rng.random((3 * F, 3)) < 0.5, F32(-0.0), F32(0.0)).astype(F32)
        c[:3] = [[0.0, -0.0, 0.0], [0.0, -0.0, -0.0], [-0.0, -0.0, 0.0]]
        return v, np.arange(3 * F, dtype=np.int32).reshape(F, 3), c, None, None
    if kind in ("tiny", "huge"):
        # Right triangles of legs X: A2 = sqrt(nz * nz) with nz = X * X.  tiny: nz * nz is subnormal (down to 1.6e-45), so
        # the twice-areas are the smallest there are, about 1e-21 (A2 is a square root of at least 2^-149, so it is never
        # subnormal itself).  huge: the largest finite A2, 1.8e19 (nz * nz just below FLT_MAX), a face whose nz * nz
        # overflows (bad), and faces below 2^-32 of the largest (weight 0).
        s = math.sqrt(1e-21) if kind == "tiny" else math.sqrt(1.8e19)
        base = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F32)
        scales = rng.uniform(0.2, 1.0, 64).astype(F32) * F32(s)
        if kind == "huge":
            scales[:4] = [F32(s), F32(math.sqrt(1.95e19)), F32(1e3), F32(1.0)]
        v = (base[None] * scales[:, None, None]).reshape(-1, 3).astype(F32)
        return v, np.arange(64 * 3, dtype=np.int32).reshape(64, 3), None, None, None
    if kind == "texture":  # uv on the texel half-points (k + 0.5) / 8, the same at the three vertices of a face, and 0 / 1
        F = 400
        v = rng.uniform(-1, 1, (F * 3, 3)).astype(F32)
        k = rng.integers(-1, 9, (F, 2)).astype(F32)
        uv = np.repeat(np.clip((k + F32(0.5)) / F32(8), F32(0), F32(1)), 3, 0).astype(F32)
        tex = rng.integers(0, 256, (8, 8, 4), dtype=np.uint8)
        tex[..., 3] = rng.integers(1, 256, (8, 8))  # a nonzero alpha, never read
        return v, np.arange(3 * F, dtype=np.int32).reshape(F, 3), None, uv, tex
    raise ValueError(kind)


_MESH = [("random", 3000, "vcol", 0), ("random", 3000, "none", 2 ** 64 - 1), ("flat", 500, "vcol", 7), ("signed_zero", 600, "vcol", 3),
         ("tiny", 64, "none", 1), ("huge", 64, "none", 2), ("texture", 400, "tex3", 5), ("texture", 400, "tex4", 6)]


@pytest.mark.parametrize("kind,F,colour,seed", _MESH, ids=[mesh_id(F, c) + f"-{k}-seed{s}" for k, F, c, s in _MESH])
def test_mesh_sample(kind, F, colour, seed):
    """Every sample, colour, face index and the stats bit for bit against oracle.mesh_ref, the whole window each.  The
    signed-zero mesh holds the clamp's -0.0 / +0.0 rule; the flat mesh makes the clamp bind; tiny and huge reach both ends
    of the weight's exponent; the texture cases land uv on texel half-points, in RGB and in RGBA."""
    rng = np.random.default_rng(F + seed % 1000)
    v, f, c, uv, tex = _mesh(kind, rng)
    assert len(f) == F
    if colour == "none":
        c = None
    if colour == "tex3":
        tex = tex[..., :3].copy()
    want = _mesh_check(v, f, 20000, seed, vcol=c, uv=uv, tex=tex, name=kind)
    if kind == "signed_zero":  # the clamp keeps a point that lies inside its face's box: the sign of the bary sum survives
        assert np.signbit(want[0][:, :]).any() and (want[0] == 0).sum() > 1000
    print(f"[mesh] {kind}: total weight {want[3][0]}, bad faces {want[3][1]}")


_ENDS = [("first", 2048), ("last", 2048), ("one_good", 3001), ("single", 1)]


@pytest.mark.parametrize("which,F", _ENDS, ids=[mesh_id(F, "none") + f"-{w}" for w, F in _ENDS])
def test_mesh_sample_ends(which, F):
    """Weight on one face only: the first (binary search's low end), the last (its high end), one good face among bad ones
    (indices out of range, a NaN vertex, zero area, an infinite area), a single face.  Every sample lies on it."""
    rng = np.random.default_rng(F)
    V = 64
    v = rng.uniform(-1, 1, (V, 3)).astype(F32)
    v[60] = [np.nan, 0, 0]
    v[61] = [3e38, 0, 0]
    v[62] = [0, 3e38, 0]
    f = np.zeros((F, 3), np.int32)  # zero area
    if which == "one_good":
        f[0::4] = [0, V, 1]
        f[1::4] = [60, 1, 2]
        f[2::4] = [0, 61, 62]
    good = {"first": 0, "last": F - 1, "one_good": F // 2 + 1, "single": 0}[which]
    f[good] = [3, 4, 5]
    want = _mesh_check(v, f, 4099, 11, vcol=rng.uniform(0, 1, (V, 3)).astype(F32), name=which)
    assert (want[2] == good).all()


def test_mesh_sample_boundaries():
    """F = 2^20 + 1000 faces (1025 chunks: the chunk-total scan loops): one face of twice-area 1.5 and the rest 2^-31, so
    their weights are exactly 1 and u lands on a cdf boundary for about one sample in 2000 - where the strict cdf[f] > u of
    the binary search decides.  The workspace is reused from this call by a smaller mesh."""
    F = (1 << 20) + 1000
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1.5, 0], [2.0 ** -16, 0, 0], [0, 2.0 ** -15, 0]], F32)
    f = np.tile(np.array([[0, 3, 4]], np.int32), (F, 1))
    f[F // 3] = [0, 1, 2]
    L = _nv().lib()
    ws = _dirty(L.psam_mesh_sample_workspace_bytes(F))
    want = _mesh_check(v, f, 1 << 18, 5, ws=ws, name="boundaries")
    assert want[3][0] == F - 1 + 3 * 2 ** 30
    rng = np.random.default_rng(1)
    v2, f2, c2, _, _ = _mesh("random", rng)
    _mesh_check(v2, f2, 5000, 9, vcol=c2, ws=ws, name="reused workspace")


def test_mesh_face_centers():
    """((a + b) + c) / 3 per axis, NaN for a face with an index outside [0, V); nothing outside the window."""
    from oracle import mesh_ref

    nv = _nv()
    rng = np.random.default_rng(3)
    V, F = 500, 1027
    v = rng.uniform(-1, 1, (V, 3)).astype(F32)
    v[:7] = -0.0
    f = rng.integers(0, V, (F, 3)).astype(np.int32)
    f[::13, 2] = V
    f[1::17, 0] = -1
    vw, fw, cw = Win(torch.from_numpy(v)), Win(torch.from_numpy(f), fill=0), Win(shape=(F, 3))
    assert nv.lib().psam_mesh_face_centers_f32(vw.ptr, V, fw.ptr, F, cw.ptr, nv.stream()) == 0
    for w, n in ((vw, "v"), (fw, "faces"), (cw, "centers")):
        w.check(n)
    _cmp(cw.cpu(), torch.from_numpy(mesh_ref.face_centers(v, f)), "centers")


# ------------------------------------------------------------------------------------------------
# mask lifting and the label map
# ------------------------------------------------------------------------------------------------
_LIFT = [(5, 100, 1000, 2, 3), (1, 37, 1, 0, 0), (3, 64, 33, 1, 1), (70, 4096, 100003, 0, 5), (2, 33, 4097, 3, 0), (0, 50, 70, 0, 0)]


def lift_id(K, S, M, dWs, dWm):
    Wm = _cdiv(M, 32) + dWm
    return _id("mask_lift_kernel", K=K, S=S, M=M, Ws=_cdiv(S, 32) + dWs, Wm=Wm, grid=_cdiv(_cdiv(Wm, 4), 8))


@pytest.mark.parametrize("K,S,M,dWs,dWm", _LIFT, ids=[lift_id(*c) for c in _LIFT])
def test_mask_lift(K, S, M, dWs, dWm):
    """bits_out [K, Wm] and area [K] bit for bit against oracle.mesh_ref.lift, padded with zero words to Wm.  Every bit
    past S of the source rows is set, and nearest holds S (that bit, when S % 32 != 0), -1, S + 31, 2^40 and S - 1, so an
    entry outside [0, S) that is read gives a wrong bit.  K = 0 writes nothing."""
    from oracle import mesh_ref

    nv = _nv()
    rng = np.random.default_rng(K * 7 + S + M)
    Ws, Wm = _cdiv(S, 32) + dWs, _cdiv(M, 32) + dWm
    m = rng.random((K, S)) < 0.5
    bits = _poison_tail(_pack(m, Ws), S)
    near = rng.integers(0, S, M).astype(np.int64)
    for j, val in enumerate([S, -1, S + 31, 2 ** 40, S - 1]):
        near[j::7 + 2 * j] = val
    bw, nw = Win(bits, fill=SENT), Win(torch.from_numpy(near), fill=0)
    ow, aw = Win(shape=(K, Wm), dtype=torch.int32, fill=SENT), Win(shape=(K,), dtype=torch.int32, fill=SENT)
    assert nv.lib().psam_mask_lift(bw.ptr, K, Ws, S, nw.ptr, M, Wm, ow.ptr, aw.ptr, nv.stream()) == 0
    for w, n in ((bw, "bits"), (nw, "nearest"), (ow, "bits_out"), (aw, "area")):
        w.check(n)
    if K == 0:
        _cmp(ow.cpu(), torch.zeros(0, Wm, dtype=torch.int32), "bits_out")
        return
    wb, wa = mesh_ref.lift(bits.numpy().view(np.uint32), near, S)
    want = torch.zeros(K, Wm, dtype=torch.int32)
    want[:, :wb.shape[1]] = torch.from_numpy(wb.view(np.int32))
    _cmp(ow.cpu(), want, "bits_out")
    _cmp(aw.cpu(), torch.from_numpy(wa), "area")


_LABEL = [(1025, 5000, 2, "ties"), (1025, 777, 0, "extremes"), (3000, 300, 1, "ties"), (1, 1, 0, "extremes"), (7, 4099, 4, "extremes"),
          (0, 100, 0, "ties")]


def label_id(K, N, dW, prio):
    return _id("mask_label_kernel", K=K, N=N, W=_cdiv(N, 32) + dW, tiles=_cdiv(K, 1024), grid=_cdiv(N, 256), prio=prio)


@pytest.mark.parametrize("K,N,dW,prio", _LABEL, ids=[label_id(*c) for c in _LABEL])
def test_mask_label_map(K, N, dW, prio):
    """labels [N] bit for bit against oracle.mesh_ref.label_map: the smallest (priority, row), ties to the lower row, -1
    where no row holds the point.  Every bit past N of every row is set (a row word stride above ceil(N/32) occurs in
    production); one row is empty; priorities tie within a handful of values, or include INT_MIN and INT_MAX; K = 1025 and
    3000 cross the 1024-row priority tile."""
    from oracle import mesh_ref

    nv = _nv()
    rng = np.random.default_rng(K + N + dW)
    W = _cdiv(N, 32) + dW
    m = rng.random((K, N)) < rng.uniform(0.001, 0.2, (K, 1))
    if K > 1:
        m[1] = False
    bits = _poison_tail(_pack(m, W), N)
    if prio == "ties":
        pr = rng.integers(-3, 3, K).astype(np.int32)
    else:
        pr = rng.choice(np.array([INT_MIN, INT_MAX, 0, -1, 1, INT_MIN + 1, INT_MAX - 1], np.int64), K).astype(np.int32)
    bw, pw = Win(bits, fill=SENT), Win(torch.from_numpy(pr), fill=INT_MIN)
    lw = Win(shape=(N,), dtype=torch.int32, fill=SENT)
    assert nv.lib().psam_mask_label_map(bw.ptr, K, W, pw.ptr, N, lw.ptr, nv.stream()) == 0
    for w, n in ((bw, "bits"), (pw, "priority"), (lw, "labels")):
        w.check(n)
    want = mesh_ref.label_map(bits.numpy().view(np.uint32), pr, N)
    _cmp(lw.cpu(), torch.from_numpy(want), "labels")


# ------------------------------------------------------------------------------------------------
# grid nearest search
# ------------------------------------------------------------------------------------------------
def _brute(qt, kt):
    nv = _nv()
    d = torch.empty(len(qt), dtype=torch.float32, device=_dev())
    i = torch.empty(len(qt), dtype=torch.int64, device=_dev())
    assert nv.lib().psam_nn_distance_f32(qt.data_ptr(), kt.data_ptr(), len(qt), len(kt), d.data_ptr(), i.data_ptr(), nv.stream()) == 0
    return d.cpu(), i.cpu()


def _grid_run(q, k, ws=None, with_idx=True):
    nv = _nv()
    L = nv.lib()
    n1, n2 = len(q), len(k)
    qw, kw = Win(torch.from_numpy(q)), Win(torch.from_numpy(k))
    dw = Win(shape=(n1,))
    iw = Win(shape=(n1,), dtype=torch.int64, fill=SENT) if with_idx else None
    nb = L.psam_nn_grid_workspace_bytes(n2)
    if ws is None:
        ws = _dirty(nb)
    assert ws.numel() >= nb
    rc = L.psam_nn_grid_f32(qw.ptr, n1, kw.ptr, n2, dw.ptr, iw.ptr if iw else None, ws.data_ptr(), nv.stream())
    assert rc == 0
    for w, n in ((qw, "query"), (kw, "key"), (dw, "dist"), (iw, "idx")):
        if w is not None:
            w.check(n)
    return qw, kw, dw, iw


def _fp64_margin(qt, kt, idx, rows):
    """Largest (chosen - nearest) / (REL * nearest) over the query rows `rows` (numpy), fp64 squared distances on the
    device in chunks (a non-finite key is never nearest).  <= 1 passes."""
    rows = torch.from_numpy(rows)
    q = qt[rows.to(_dev())].double()
    k = kt.double()
    kf = torch.isfinite(kt).all(1)
    best = torch.full((len(rows),), float("inf"), dtype=torch.float64, device=_dev())
    for s in range(0, len(k), 1 << 20):
        kc, fc = k[s:s + (1 << 20)], kf[s:s + (1 << 20)]
        for r in range(0, len(q), 128):
            d = ((q[r:r + 128, None, :] - kc[None]) ** 2).sum(-1)
            d[:, ~fc] = float("inf")
            best[r:r + 128] = torch.minimum(best[r:r + 128], d.min(1).values)
    ch = idx[rows].to(_dev())
    assert bool((ch >= 0).all())
    chosen = ((q - k[ch]) ** 2).sum(-1)
    excess = (chosen - best).clamp(min=0)
    return float((excess / (REL * best.clamp(min=2.0 ** -140))).max())


def _grid_keys(what, n2, rng):
    if what == "uniform":
        return rng.uniform(-1, 1, (n2, 3)).astype(F32)
    if what == "identical":
        return np.tile(F32([[0.25, -0.5, 0.125]]), (n2, 1))
    if what == "outliers":  # 1 % far outliers: the grid's box is the 5-95 % quantiles, they are clamped into border cells
        k = rng.normal(0, 0.2, (n2, 3)).astype(F32)
        o = rng.random(n2) < 0.01
        k[o] = (rng.normal(0, 1, (int(o.sum()), 3)) * 1e3).astype(F32)
        return k
    if what == "nonfinite":  # 30 % of the keys hold a NaN or an inf: fewer finite keys than cells
        k = rng.uniform(-1, 1, (n2, 3)).astype(F32)
        bad = rng.random(n2) < 0.3
        k[bad, rng.integers(0, 3, int(bad.sum()))] = rng.choice(F32([np.nan, np.inf, -np.inf]), int(bad.sum()))
        return k
    if what == "collinear":
        t = rng.uniform(-1, 1, n2).astype(F32)
        return np.stack([t, np.zeros_like(t), np.zeros_like(t)], 1)
    raise ValueError(what)


def _grid_queries(k, n1, rng, far=True):
    """A third uniform in a box 20 % larger than the keys', a third at keys plus a small jitter, a third exactly at keys;
    a few far away (unless not far) and a few non-finite."""
    fk = k[np.isfinite(k).all(1)]
    lo, hi = fk.min(0), fk.max(0)
    ext = np.maximum(hi - lo, 1e-3)
    a = n1 // 3
    q = np.empty((n1, 3), F32)
    q[:a] = rng.uniform(lo - 0.1 * ext, hi + 0.1 * ext, (a, 3))
    pick = fk[rng.integers(0, len(fk), n1 - a)]
    q[a:] = pick
    q[a:2 * a] += (rng.normal(0, 1e-4, (a, 3)) * ext).astype(F32)
    if far:
        q[5:8] = [[50, 50, 50], [-30, 0, 0], [0, 1e6, 0]]
    q[8] = [np.nan, 0, 0]
    q[9] = [0, np.inf, 0]
    return q


_GRID = [(700, 1001, "uniform"), (5000, 3333, "uniform"), ((1 << 22) + 5, 20037, "uniform"), (5000, 2999, "identical"),
         (200003, 10001, "outliers"), (300001, 9999, "nonfinite")]


@pytest.mark.parametrize("n2,n1,what", _GRID, ids=[grid_id(n2, n1, w) for n2, n1, w in _GRID])
def test_grid_nearest(n2, n1, what):
    """dist and idx bit for bit against the brute-force psam_nn_distance_f32 over the whole window, idx against the C
    oracle on 64 queries, and the fp64 check on up to 1024 queries.  n2 = 2^22 + 5 takes the cell cap and a looping scan
    of 4097 chunk totals; all keys identical give one cell of side 1 (ties to index 0); far outliers are clamped into the
    border cells; non-finite keys leave fewer finite keys than cells."""
    from oracle import tokenizer_ref

    rng = np.random.default_rng(n2 + n1)
    k = _grid_keys(what, n2, rng)
    q = _grid_queries(k, n1, rng)
    qw, kw, dw, iw = _grid_run(q, k)
    bd, bi = _brute(qw.t, kw.t)
    _cmp(iw.cpu(), bi, "idx")
    _cmp(dw.cpu(), bd, "dist", raw=True)
    sub = rng.choice(n1, 64, replace=False)
    w = tokenizer_ref.knn(q[sub][None], k[None], 1)[0][0, :, 0]
    fin = np.isfinite(q[sub]).all(1)
    assert np.array_equal(bi.numpy()[sub][fin], w[fin])
    rows = np.flatnonzero(np.isfinite(q).all(1) & (np.abs(q) < 1e5).all(1))[:1024]
    margin = _fp64_margin(qw.t, kw.t, iw.cpu(), rows)
    assert margin <= 1.0, margin
    if what == "identical":
        assert bool((bi[torch.from_numpy(np.isfinite(q).all(1))] == 0).all())
    print(f"[scan] grid {what} n2={n2} n1={n1}: fp64 margin {margin:.3f} of 10u")


def test_grid_nearest_no_idx_and_reuse():
    """idx_out = NULL: the distances alone, bit for bit; then a workspace left dirty by a 300001-key call serves a
    5000-key one."""
    rng = np.random.default_rng(4)
    k = _grid_keys("uniform", 300001, rng)
    q = _grid_queries(k, 4099, rng)
    qw, kw, dw, _ = _grid_run(q, k, with_idx=False)
    bd, _ = _brute(qw.t, kw.t)
    _cmp(dw.cpu(), bd, "dist", raw=True)
    ws = _dirty(_nv().lib().psam_nn_grid_workspace_bytes(300001))
    _grid_run(q, k, ws=ws)
    k2 = _grid_keys("outliers", 5000, rng)
    q2 = _grid_queries(k2, 1027, rng)
    qw, kw, dw, iw = _grid_run(q2, k2, ws=ws)
    bd, bi = _brute(qw.t, kw.t)
    _cmp(iw.cpu(), bi, "idx")
    _cmp(dw.cpu(), bd, "dist", raw=True)


def test_grid_nearest_collinear():
    """3 * 2^20 collinear keys: the dims clamp of 2^21 cells binds, and the last third of the line shares the last cell.
    Exact all the same; the query time is printed next to a uniform cloud of the same size (speed is not asserted).  The
    queries stay near the line: one far off it cannot meet the stopping bound before the last of the 2^21 rings, and
    every ring walks all the grid rows of its box, so it would take about 2^42 steps."""
    rng = np.random.default_rng(8)
    n2, n1 = 3 << 20, 1001
    times = {}
    for what in ("collinear", "uniform"):
        k = _grid_keys(what, n2, rng)
        q = _grid_queries(k, n1, rng, far=False)
        qw, kw, dw, iw = _grid_run(q, k)
        bd, bi = _brute(qw.t, kw.t)
        _cmp(iw.cpu(), bi, f"{what} idx")
        _cmp(dw.cpu(), bd, f"{what} dist", raw=True)
        nv = _nv()
        ws = _dirty(nv.lib().psam_nn_grid_workspace_bytes(n2))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        best = float("inf")
        for _ in range(3):
            e0.record()
            assert nv.lib().psam_nn_grid_f32(qw.ptr, n1, kw.ptr, n2, dw.ptr, iw.ptr, ws.data_ptr(), nv.stream()) == 0
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1))
        times[what] = best
    print(f"[scan] grid search n2={n2} n1={n1} (build and queries, best of 3): collinear {times['collinear']:.2f} ms, "
          f"uniform {times['uniform']:.2f} ms on {torch.cuda.get_device_name(0)}")


# ------------------------------------------------------------------------------------------------
# voxel subsample
# ------------------------------------------------------------------------------------------------
def _vox_run(xyz, S, seed, ws=None, name=""):
    from oracle import scan_ref

    nv = _nv()
    L = nv.lib()
    P = len(xyz)
    xw = Win(torch.from_numpy(np.ascontiguousarray(xyz, F32)))
    iw, sw = Win(shape=(S,), dtype=torch.int64, fill=SENT), Win(shape=(4,), dtype=torch.int64, fill=SENT)
    nb = L.psam_voxel_subsample_workspace_bytes(P)
    if ws is None:
        ws = _dirty(nb)
    assert ws.numel() >= nb
    assert L.psam_voxel_subsample_f32(xw.ptr, P, S, seed, iw.ptr, sw.ptr, ws.data_ptr(), nv.stream()) == 0
    for w, n in ((xw, "xyz"), (iw, "idx"), (sw, "stats")):
        w.check(n)
    want_i, want_s = scan_ref.subsample(xyz, S, seed)
    _cmp(sw.cpu(), torch.from_numpy(want_s), f"{name} stats")
    _cmp(iw.cpu(), torch.from_numpy(want_i), f"{name} idx")
    return want_s


def _vox_cloud(P, rng):
    """Clusters of different densities, a fifth of the points duplicated (ties on e, decided by the index)."""
    c = rng.uniform(-0.9, 0.9, (P, 3)) * rng.choice([1.0, 0.05, 0.002], (P, 1))
    x = c.astype(F32)
    d = rng.choice(P, P // 5, replace=False)
    x[d] = x[rng.choice(P, P // 5)]
    return x


def _level_sizes(xyz):
    """Two levels L with n_{L-1} < n_L - 1 < n_L < P, at about 100 and about 5000 cells."""
    from oracle import scan_ref

    n = scan_ref.level_counts(xyz)
    out = []
    for target in (100, 5000):
        L = next(L for L in range(1, 22) if n[L] >= target and n[L - 1] < n[L] - 1 and n[L] < len(xyz))
        out.append(int(n[L]))
    return out


@pytest.mark.parametrize("which", ["nL", "nL+1", "nL-1"])
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("seed", [0, 2 ** 64 - 1])
def test_voxel_subsample_levels(which, level, seed):
    """S exactly at a level count n_L (level L, nothing thinned), one above (the next level), one below (the radix select
    drops a single cell), at two levels and two seeds, against oracle.scan_ref bit for bit."""
    P = 50003
    xyz = _vox_cloud(P, np.random.default_rng(P))
    nL = _level_sizes(xyz)[level]
    S = nL + {"nL": 0, "nL+1": 1, "nL-1": -1}[which]
    st = _vox_run(xyz, S, seed, name=vox_id(P, which))
    assert st[3] == min(S, st[2])
    if which == "nL-1":
        assert st[2] == S + 1


_VOX = [(1, 1, "one"), (1, 3, "one"), (1003, 200, "far"), (1003, 2000, "far"), (4097, 64, "zeros"), (257, 10, "nonfinite")]


@pytest.mark.parametrize("P,S,kind", _VOX, ids=[vox_id(P, S) + f"-{k}" for P, S, k in _VOX])
def test_voxel_subsample_inputs(P, S, kind):
    """P = 1; P not a multiple of 256 or 1024; coordinates at +-5 (the quantiser's clamp) and exactly +-1; +-0.0
    coordinates (the same cell); rows with a NaN or an inf."""
    rng = np.random.default_rng(P + S)
    x = rng.uniform(-1, 1, (P, 3)).astype(F32)
    if kind == "far":
        x[::3] = rng.choice(F32([-5, 5, 1, -1, 0.999999, -0.9999999]), (len(x[::3]), 3))
    if kind == "zeros":
        x[::2] = np.where(rng.random((len(x[::2]), 3)) < 0.5, F32(-0.0), F32(0.0))
    if kind == "nonfinite":
        x[::4, 1] = np.nan
        x[1::9, 0] = -np.inf
    for seed in (0, 2 ** 64 - 1):
        _vox_run(x, S, seed, name=kind)


def test_voxel_subsample_reused_workspace():
    """A workspace full of a 50003-point call's leftovers serves a 1003-point call and then a 50003-point call again."""
    rng = np.random.default_rng(2)
    big = _vox_cloud(50003, rng)
    ws = _dirty(_nv().lib().psam_voxel_subsample_workspace_bytes(50003))
    _vox_run(big, 3000, 1, ws=ws, name="big")
    _vox_run(_vox_cloud(1003, rng), 100, 2, ws=ws, name="small after big")
    _vox_run(big, 2999, 3, ws=ws, name="big again")


# ------------------------------------------------------------------------------------------------
# crop layout, count and gather
# ------------------------------------------------------------------------------------------------
def _cloud(kind, N, rng):
    x = rng.uniform(-1, 1, (N, 3)).astype(F32) * F32(0.7)
    if kind == "flat0":  # z is +0.0 or -0.0
        x[:, 2] = np.where(rng.random(N) < 0.5, F32(-0.0), F32(0.0))
    if kind == "grid":  # coordinates on a lattice: many points exactly on crop faces
        x = (rng.integers(-8, 9, (N, 3)) / 8).astype(F32)
    return x


def _layout_single(x, layers, r):
    nv = _nv()
    N, T = len(x), nv.lib().psam_crop_total(layers)
    xw = Win(torch.from_numpy(x))
    bw, cw = Win(shape=(T, 6)), Win(shape=(T,), dtype=torch.int32, fill=SENT)
    assert nv.lib().psam_crop_layout_f32(xw.ptr, N, layers, r, bw.ptr, cw.ptr, nv.stream()) == 0
    for w, n in ((xw, "xyz"), (bw, "boxes"), (cw, "counts")):
        w.check(n)
    return bw.cpu(), cw.cpu()


_LAYOUT = [(1, 2, OVR, "uniform"), (300, 0, 0.0, "uniform"), (20000, 1, float(np.nextafter(F32(1), F32(0))), "uniform"),
           (20000, 3, OVR, "uniform"), (20000, 2, OVR, "flat0"), (20000, 1, OVR, "grid"), (262149, 1, OVR, "uniform")]


@pytest.mark.parametrize("N,layers,r,kind", _LAYOUT, ids=[layout_id(False, N, ly) + f"-r{r:.3g}-{k}" for N, ly, r, k in _LAYOUT])
def test_crop_layout(N, layers, r, kind):
    """boxes and counts bit for bit against oracle.amg_crops_ref.layout: n_layers 0 to 3 (585 crops in shared memory),
    overlap 0 and just below 1, a flat cloud of mixed +-0.0 (the box's sign of zero, duplicate boxes), a lattice with
    points on the closed upper faces, and a count grid capped at 512 CTAs."""
    from oracle import amg_crops_ref

    x = _cloud(kind, N, np.random.default_rng(N + layers))
    boxes, counts = _layout_single(x, layers, r)
    wb, wc, _ = amg_crops_ref.layout(x, layers, r)
    _cmp(boxes, torch.from_numpy(wb), "boxes")
    _cmp(counts, torch.from_numpy(wc.astype(np.int32)), "counts")


def _want_gather(x, c, boxes, crop, margin, n_out, width=None):
    """(idx, xyz, rgb, edge words) of one crop, the first n_out points, padded with zeros to `width` rows."""
    from oracle import amg_crops_ref

    idx, coords, rgb, edge = amg_crops_ref.crop_cloud(x, c, boxes, crop, margin)
    width = n_out if width is None else width
    We = _cdiv(width, 32)
    out_i = np.zeros(width, np.int32)
    out_x, out_c = np.zeros((width, 3), F32), np.zeros((width, 3), F32)
    e = np.zeros((1, We * 32), bool)
    out_i[:n_out], out_x[:n_out], out_c[:n_out], e[0, :n_out] = idx[:n_out], coords[:n_out], rgb[:n_out], edge[:n_out]
    return torch.from_numpy(out_i), torch.from_numpy(out_x), torch.from_numpy(out_c), _pack(e, We)[0]


def _gather_single(x, c, boxes, crop, margin, n_out, ws=None):
    nv = _nv()
    L = nv.lib()
    N, T = len(x), len(boxes)
    xw, cw, bw = Win(torch.from_numpy(x)), Win(torch.from_numpy(c)), Win(torch.from_numpy(np.ascontiguousarray(boxes)))
    outs = [Win(shape=(n_out,), dtype=torch.int32, fill=SENT), Win(shape=(n_out, 3)), Win(shape=(n_out, 3)),
            Win(shape=(_cdiv(n_out, 32),), dtype=torch.int32, fill=SENT)]
    if ws is None:
        ws = _dirty(L.psam_crop_gather_workspace_bytes(N))
    rc = L.psam_crop_gather_f32(xw.ptr, cw.ptr, N, bw.ptr, crop, T, margin, n_out, *[o.ptr for o in outs], ws.data_ptr(), nv.stream())
    assert rc == 0
    for w, n in zip([xw, cw, bw] + outs, ("xyz", "rgb", "boxes", "idx_out", "xyz_out", "rgb_out", "edge")):
        w.check(n)
    return [o.cpu() for o in outs]


_GATHER = [(20000, 1, 5, 0.02, "uniform"), (20000, 2, 30, 0.0, "uniform"), (20000, 1, 0, 0.02, "flat0"), (20000, 1, 3, 0.02, "flat0"),
           (20000, 1, 6, 0.1, "grid"), (1, 0, 0, 0.02, "uniform"), ((1 << 20) + 1025, 1, 0, 0.02, "uniform"),
           ((1 << 20) + 1025, 1, 8, 0.02, "uniform")]


@pytest.mark.parametrize("N,layers,crop,margin,kind", _GATHER, ids=[gather_id(False, N) + f"-crop{cr}-m{m}-{k}" for N, _, cr, m, k in _GATHER])
def test_crop_gather(N, layers, crop, margin, kind):
    """idx, renormalised xyz, rgb and edge words bit for bit against oracle.amg_crops_ref.crop_cloud: edge margins of 0,
    0.02 and 0.1; a flat cloud of mixed +-0.0 (the sign of a centred -0.0); lattice points on the faces; N = 2^20 + 1025
    points, whose 1026 chunks take the offset loop's second pass (crop 0: every point, so the last chunk's offset needs
    chunk 1024's count)."""
    from oracle import amg_crops_ref

    rng = np.random.default_rng(N + crop)
    x = _cloud(kind, N, rng)
    c = rng.uniform(0, 1, (N, 3)).astype(F32)
    boxes, counts, _ = amg_crops_ref.layout(x, layers, OVR)
    n_out = int(counts[crop])
    assert n_out >= 1
    got = _gather_single(x, c, boxes, crop, margin, n_out)
    for g, w, n in zip(got, _want_gather(x, c, boxes, crop, margin, n_out), ("idx_out", "xyz_out", "rgb_out", "edge")):
        _cmp(g, w, n, raw=True)
    if kind == "flat0" and crop == 0:
        zx = got[1][:, 2]
        assert bool(torch.signbit(zx).any()) and bool((~torch.signbit(zx)).any())
    print(f"[crops] gather N={N} crop {crop}: {n_out} points, {int(got[3].view(torch.int32).ne(0).sum())} nonzero edge words")


def _batch_inputs(rng, B, N_max, lengths, kind="uniform"):
    """xyz / rgb [B, N_max, 3]: each cloud's first clamp(lengths[b], 0, N_max) rows real, the rest poison - coordinates of
    +-1e30 that would win the bounding box and land in every crop if read, every fifth row NaN."""
    x = np.stack([_cloud(kind, N_max, rng) for _ in range(B)])
    c = rng.uniform(0, 1, (B, N_max, 3)).astype(F32)
    for b, n in enumerate(lengths):
        n = min(max(n, 0), N_max)
        x[b, n:] = rng.choice(F32([-1e30, 1e30]), (N_max - n, 3))
        x[b, n::5] = np.nan
        c[b, n:] = 9.0
    return x, c


def _layout_batched(x, lengths, layers, r):
    nv = _nv()
    B, N_max, _ = x.shape
    T = nv.lib().psam_crop_total(layers)
    xw, lw = Win(torch.from_numpy(x)), Win(torch.tensor(lengths, dtype=torch.int32), fill=N_max)
    bw, cw = Win(shape=(B, T, 6)), Win(shape=(B, T), dtype=torch.int32, fill=SENT)
    assert nv.lib().psam_crop_layout_batched_f32(xw.ptr, lw.ptr, B, N_max, layers, r, bw.ptr, cw.ptr, nv.stream()) == 0
    for w, n in ((xw, "xyz"), (lw, "lengths"), (bw, "boxes"), (cw, "counts")):
        w.check(n)
    return bw.cpu(), cw.cpu()


def _gather_batched(x, c, lengths, boxes, pairs, n_max, margin):
    nv = _nv()
    L = nv.lib()
    B, N_max, _ = x.shape
    P, T = pairs.shape[1], boxes.shape[1]
    ins = [Win(torch.from_numpy(x)), Win(torch.from_numpy(c)), Win(torch.tensor(lengths, dtype=torch.int32), fill=N_max),
           Win(torch.as_tensor(boxes)), Win(torch.from_numpy(pairs.astype(np.int32)), fill=0)]
    We = _cdiv(n_max, 32)
    outs = [Win(shape=(P, n_max), dtype=torch.int32, fill=SENT), Win(shape=(P, n_max, 3)), Win(shape=(P, n_max, 3)),
            Win(shape=(P, We), dtype=torch.int32, fill=SENT)]
    ws = _dirty(L.psam_crop_gather_batched_workspace_bytes(P, N_max))
    rc = L.psam_crop_gather_batched_f32(ins[0].ptr, ins[1].ptr, ins[2].ptr, B, N_max, ins[3].ptr, T, ins[4].ptr, P, n_max, margin,
                                        *[o.ptr for o in outs], ws.data_ptr(), nv.stream())
    assert rc == 0
    for w, n in zip(ins + outs, ("xyz", "rgb", "lengths", "boxes", "pairs", "idx_out", "xyz_out", "rgb_out", "edge")):
        w.check(n)
    return [o.cpu() for o in outs]


_BATCH = [(2, 2500, [2500, 1700], 1, "uniform"), (4, 5000, [5000, 3111, -4, 9000], 1, "uniform"), (3, 3000, [3000, 0, 2047], 2, "flat0"),
          (2, 1100, [1100, 1025], 3, "grid")]


@pytest.mark.parametrize("B,N_max,lengths,layers,kind", _BATCH,
                         ids=[layout_id(True, Nm, ly).replace("crop_count", "crop_gather_write") + f"-B{B}-len{'_'.join(map(str, ln))}-{k}"
                              for B, Nm, ln, ly, k in _BATCH])
def test_crop_batched(B, N_max, lengths, layers, kind):
    """The batched layout and gather: each cloud's boxes and counts, and each pair's rows, bit for bit against the oracle
    on that cloud's first clamp(length, 0, N_max) rows (lengths of 0, negative and above N_max), with padding rows built
    to win the bounding box and NaN rows.  Pairs outside their ranges (cloud -1 or B, crop T, count -1 or n_max + 1)
    gather nothing: all their rows 0; a count below the crop's size keeps its first points; rows past a count are 0."""
    from oracle import amg_crops_ref

    rng = np.random.default_rng(B + N_max)
    x, c = _batch_inputs(rng, B, N_max, lengths, kind)
    boxes, counts = _layout_batched(x, lengths, layers, OVR)
    T = boxes.shape[1]
    want_boxes = []
    for b, n in enumerate(lengths):
        n = min(max(n, 0), N_max)
        with np.errstate(all="ignore"):
            wb, wc, _ = amg_crops_ref.layout(x[b, :n], layers, OVR)
        _cmp(boxes[b], torch.from_numpy(wb), f"cloud {b} boxes")
        _cmp(counts[b], torch.from_numpy(wc.astype(np.int32)), f"cloud {b} counts")
        want_boxes.append(wb)
    pl = [(b, t, int(counts[b, t])) for b in range(B) for t in range(T) if int(counts[b, t]) > 0][:40]
    n_max = max(p[2] for p in pl)
    pl += [(0, 1, int(counts[0, 1]) // 2), (0, 0, 0), (-1, 0, 5), (B, 0, 5), (0, T, 5), (0, 0, -1), (0, 0, n_max + 1)]
    pairs = np.array(pl, np.int64).T.copy()
    got = _gather_batched(x, c, lengths, boxes, pairs, n_max, 0.02)
    want = [torch.zeros_like(g) for g in got]
    for p, (b, t, cnt) in enumerate(pl):
        if not (0 <= b < B and 0 <= t < T and 0 <= cnt <= n_max) or cnt == 0:
            continue
        n = min(max(lengths[b], 0), N_max)
        for w, part in zip(want, _want_gather(x[b, :n], c[b, :n], want_boxes[b], t, 0.02, cnt, n_max)):
            w[p] = part
    for g, w, n in zip(got, want, ("idx_out", "xyz_out", "rgb_out", "edge")):
        _cmp(g, w, f"batched {n}", raw=True)


def test_crop_batched_one_cloud_equals_single():
    """B = 1 through the batched entry points equals the single-cloud ones bit for bit: the layout, and a gather of each
    crop with its count."""
    rng = np.random.default_rng(12)
    N = 4099
    x, c = _cloud("flat0", N, rng), rng.uniform(0, 1, (N, 3)).astype(F32)
    boxes, counts = _layout_single(x, 1, OVR)
    bb, bc = _layout_batched(x[None], [N], 1, OVR)
    _cmp(bb[0], boxes, "boxes")
    _cmp(bc[0], counts, "counts")
    pl = [(0, t, int(counts[t])) for t in range(len(counts)) if int(counts[t]) > 0]
    n_max = max(p[2] for p in pl)
    got = _gather_batched(x[None], c[None], [N], bb, np.array(pl, np.int64).T.copy(), n_max, 0.02)
    for p, (_, t, cnt) in enumerate(pl):
        single = _gather_single(x, c, boxes.numpy(), t, 0.02, cnt)
        for g, s, n in zip(got, single, ("idx_out", "xyz_out", "rgb_out")):
            _cmp(g[p, :cnt], s, f"crop {t} {n}", raw=True)
        _cmp(got[3][p, :len(single[3])], single[3], f"crop {t} edge")


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def test_routing_guard():
    """One call per launch path - the mesh sampler with and without its add pass, face centres, the lift, the label map,
    the grid search with and without its chunk-sum passes, the voxel subsample, and the crop layout and gather in both
    BATCH forms - under the profiler: the kernels that ran must be the restated sequence, and each crop count grid the
    restated one.  It runs in a fresh interpreter, as the other routing guards do."""
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_mesh_scan_kernels as t; t._routing_guard()" % (
        here, repo, os.path.join(repo, "point-sam_b200"))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())


def _routing_guard():
    nv = _nv()
    L, d = nv.lib(), _dev()
    st = nv.stream()
    calls, keep = [], []  # (expected kernel names, (x, y) grid of the first one or None, fn)

    def t(a, dtype=None):
        x = torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(d)
        keep.append(x)
        return x

    def z(*shape, dtype=torch.int32):
        x = torch.zeros(shape, dtype=dtype, device=d)
        keep.append(x)
        return x

    rng = np.random.default_rng(0)
    for F in (100, 2000):
        v, f = t(rng.uniform(-1, 1, (50, 3)).astype(F32)), t(rng.integers(0, 50, (F, 3)).astype(np.int32))
        xo, ro, fo, so = z(64, 3, dtype=torch.float32), z(64, 3, dtype=torch.float32), z(64), z(3, dtype=torch.int64)
        ws = z(L.psam_mesh_sample_workspace_bytes(F) // 4 + 4)
        calls.append((mesh_kernels(F), None, lambda v=v, f=f, F=F, xo=xo, ro=ro, fo=fo, so=so, ws=ws: L.psam_mesh_sample_f32(
            v.data_ptr(), 50, f.data_ptr(), F, 64, 1, None, None, None, 0, 0, 0, xo.data_ptr(), ro.data_ptr(), fo.data_ptr(), so.data_ptr(),
            ws.data_ptr(), st)))
    cen = z(2000, 3, dtype=torch.float32)
    calls.append((["mesh_centers_kernel"], None, lambda: L.psam_mesh_face_centers_f32(v.data_ptr(), 50, f.data_ptr(), 2000, cen.data_ptr(), st)))
    lb, ln, lo, la = z(3, 4), z(100, dtype=torch.int64), z(3, 5), z(3)
    calls.append((["mask_lift_kernel", "mask_area_kernel"], None,
                  lambda: L.psam_mask_lift(lb.data_ptr(), 3, 4, 100, ln.data_ptr(), 100, 5, lo.data_ptr(), la.data_ptr(), st)))
    pr, lab = z(3), z(100)
    calls.append((["mask_label_kernel"], None, lambda: L.psam_mask_label_map(lb.data_ptr(), 3, 4, pr.data_ptr(), 100, lab.data_ptr(), st)))
    for n2 in (500, 5000):
        k, q = t(rng.uniform(-1, 1, (n2, 3)).astype(F32)), t(rng.uniform(-1, 1, (77, 3)).astype(F32))
        dd, ii = z(77, dtype=torch.float32), z(77, dtype=torch.int64)
        ws = z(L.psam_nn_grid_workspace_bytes(n2) // 4 + 4)
        calls.append((grid_kernels(n2), None, lambda k=k, q=q, n2=n2, dd=dd, ii=ii, ws=ws: L.psam_nn_grid_f32(
            q.data_ptr(), 77, k.data_ptr(), n2, dd.data_ptr(), ii.data_ptr(), ws.data_ptr(), st)))
    vx, vi, vs = t(rng.uniform(-1, 1, (3000, 3)).astype(F32)), z(100, dtype=torch.int64), z(4, dtype=torch.int64)
    vws = z(L.psam_voxel_subsample_workspace_bytes(3000) // 4 + 4)
    calls.append((VOX_KERNELS, None, lambda: L.psam_voxel_subsample_f32(vx.data_ptr(), 3000, 100, 5, vi.data_ptr(), vs.data_ptr(),
                                                                         vws.data_ptr(), st)))
    for N in (700, 200000):
        cx = t(rng.uniform(-1, 1, (N, 3)).astype(F32))
        cb, cc = z(9, 6, dtype=torch.float32), z(9)
        calls.append((["crop_layout_kernel<false>", "crop_count_kernel<false>"], ("crop_count_kernel<false>", count_grid(N), 1),
                      lambda cx=cx, N=N, cb=cb, cc=cc: L.psam_crop_layout_f32(cx.data_ptr(), N, 1, OVR, cb.data_ptr(), cc.data_ptr(), st)))
    B, Nm = 3, 5000
    bx, blen = t(rng.uniform(-1, 1, (B, Nm, 3)).astype(F32)), t(np.array([Nm, 100, 4000], np.int32))
    bb, bc = z(B, 9, 6, dtype=torch.float32), z(B, 9)
    calls.append((["crop_layout_kernel<true>", "crop_count_kernel<true>"], ("crop_count_kernel<true>", count_grid(Nm), B),
                  lambda: L.psam_crop_layout_batched_f32(bx.data_ptr(), blen.data_ptr(), B, Nm, 1, OVR, bb.data_ptr(), bc.data_ptr(), st)))
    gi, gx, gr, ge = z(64), z(64, 3, dtype=torch.float32), z(64, 3, dtype=torch.float32), z(2)
    gws = z(L.psam_crop_gather_workspace_bytes(700) // 4 + 4)
    cx7 = t(rng.uniform(-1, 1, (700, 3)).astype(F32))  # the single gather's boxes come from a layout run before the profiler
    cb7, cc7 = z(9, 6, dtype=torch.float32), z(9)
    assert L.psam_crop_layout_f32(cx7.data_ptr(), 700, 1, OVR, cb7.data_ptr(), cc7.data_ptr(), st) == 0
    calls.append((["crop_gather_count_kernel<false>", "crop_gather_write_kernel<false>"], None,
                  lambda: L.psam_crop_gather_f32(cx7.data_ptr(), cx7.data_ptr(), 700, cb7.data_ptr(), 0, 9, 0.02, 64, gi.data_ptr(),
                                                 gx.data_ptr(), gr.data_ptr(), ge.data_ptr(), gws.data_ptr(), st)))
    pairs = t(np.array([[0, 2], [1, 3], [10, 10]], np.int32))
    pi, px, pr3, pe = z(2, 64), z(2, 64, 3, dtype=torch.float32), z(2, 64, 3, dtype=torch.float32), z(2, 2)
    pws = z(L.psam_crop_gather_batched_workspace_bytes(2, Nm) // 4 + 4)
    calls.append((["crop_gather_count_kernel<true>", "crop_gather_write_kernel<true>"], None,
                  lambda: L.psam_crop_gather_batched_f32(bx.data_ptr(), bx.data_ptr(), blen.data_ptr(), B, Nm, bb.data_ptr(), 9, pairs.data_ptr(),
                                                         2, 64, 0.02, pi.data_ptr(), px.data_ptr(), pr3.data_ptr(), pe.data_ptr(),
                                                         pws.data_ptr(), st)))

    torch.cuda.synchronize()
    rcs = []
    got = _kernels_launched(lambda: rcs.extend(fn() for _, _, fn in calls))
    assert rcs == [0] * len(calls), f"return codes {rcs}"
    want = [n for names, _, _ in calls for n in names]
    assert len(got) == len(want), f"{len(want)} kernels expected, {len(got)} launched: {[n for n, _ in got]}"
    for w, (name, _) in zip(want, got):
        assert w in name and (w.endswith(">") or f"{w}<" not in name), f"expected {w}, ran {name}"
    grids, pos = 0, 0
    for names, g, _ in calls:
        if g is not None:
            gi_ = pos + names.index(g[0])
            grid = got[gi_][1]
            if grid is not None:
                assert (grid[0], grid[1]) == (g[1], g[2]), f"{g[0]}: grid {grid}, restated {g[1:]}"
                grids += 1
                print(f"[crops] {g[0]}: grid {grid[0]} x {grid[1]}, restated {g[1]} x {g[2]}")
        pos += len(names)
    print(f"[mesh/scan/crops] routing guard: {len(want)} kernels in {len(calls)} calls, each the one restated; {grids} count grids checked"
          f"{'' if got[0][1] is not None else ' (the trace has no grids)'}")
