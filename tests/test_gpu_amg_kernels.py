"""The discrete kernels of automatic mask generation - candidate extraction, the three-kernel mask NMS, the small-region
pass (csrc/mask_gen.cu), and the crop edge filter and uncrop (csrc/crops.cu) - through the C ABI, on every launch path of
their host functions.

Each kernel is compared bit for bit with a plain reference that shares no code with it: oracle.amg_ref (candidate rules,
greedy NMS as a loop over the sorted candidates), oracle.amg_regions_ref (scipy connected components), and a few lines of
numpy here for the edge filter and the uncrop.  These kernels compute on integer counts and state their fp32 arithmetic,
so every output must match exactly.

Every output sits inside a larger buffer prefilled with a sentinel (NaN for floats, 0x7f7f7f7f for ints and bits), with
guards on either side; every case compares the whole buffer, so nothing outside the header's write window may change: the
slots between clouds' blocks, keep entries past the count, ranks past the count, uncrop rows past the capacity.  Poison
inputs are in range but wrong (padding logits of +1e9, graph entries that point at padding rows, keep entries past the
count that name a different valid mask), so a kernel that read them gives a wrong answer, never a fault.

Every case id names the instantiation it reaches, from the host dispatch restated below; test_routing_guard checks those
names, and the small-region grid, under torch.profiler."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 64                # guard elements on either side of every window (256 bytes of fp32: alignment is kept)
SENT = 0x7F7F7F7F         # sentinel of int and bit windows
FSENT = 0x7FC0DEAD        # sentinel of float windows: a NaN whose payload no arithmetic produces
NAN = float("nan")
INF = float("inf")
SMS = 132                 # H100 SXM; the case ids use it, the runs use the device's own count


def _nv():
    from psam_b200 import native as nv

    return nv


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tf(b):
    return "true" if b else "false"


def _id(kernel, **kw):
    return kernel.replace(", ", ",") + "-" + "-".join(f"{k}{v}" for k, v in kw.items())


# ------------------------------------------------------------------------------------------------
# the host dispatch, restated (test_routing_guard checks it against the kernels that run)
# ------------------------------------------------------------------------------------------------
def cand_kernel(N, aligned=True, varlen=False):
    """mask_candidates_launch: 128-bit loads when N % 4 == 0 and the logits pointer is 16-byte aligned."""
    return f"mask_candidates_kernel<{_tf(N % 4 == 0 and aligned)}, {_tf(varlen)}>"


REGION_SMEM_MAX_N = 49152
REGION_L2_BYTES = 24 << 20
REGION_MAX_SLICES = 132


def region_slices(items, N):
    fit = min(max(REGION_L2_BYTES // (4 * N), 1), REGION_MAX_SLICES)
    return min(items, fit)


def region_grid(items, N, sms=SMS):
    """Persistent grid of mask_regions_launch: two CTAs per SM in the shared-memory form, one per label slice otherwise."""
    return min(items, 2 * sms) if N <= REGION_SMEM_MAX_N else min(region_slices(items, N), sms)


def region_kernel(N, varlen=False):
    return f"mask_regions_kernel<{_tf(N <= REGION_SMEM_MAX_N)}, {_tf(varlen)}>"


# ------------------------------------------------------------------------------------------------
# guarded device windows
# ------------------------------------------------------------------------------------------------
class Win:
    """A device tensor `t` inside a flat buffer with GUARD elements of `fill` on either side (`offset` more in front, to
    misalign it).  Without data the window itself is filled too.  check() asserts that the guards are untouched."""

    def __init__(self, data=None, shape=None, dtype=torch.float32, fill=None, offset=0):
        if data is not None:
            data = torch.as_tensor(data)
            shape, dtype = tuple(data.shape), data.dtype
        n = int(np.prod(shape)) if len(shape) else 1
        flat = _sentinel((GUARD + offset + n + GUARD,), dtype) if fill is None else torch.full((GUARD + offset + n + GUARD,), fill, dtype=dtype)
        if data is not None:
            flat[GUARD + offset:GUARD + offset + n] = data.reshape(-1)
        self.before = flat[:GUARD + offset].clone()
        self.after = flat[GUARD + offset + n:].clone()
        self.flat = flat.to(_dev())
        self.lo, self.n = GUARD + offset, n
        self.t = self.flat[self.lo:self.lo + n].view(shape)

    @property
    def ptr(self):  # from the buffer: an empty window still has an address
        return self.flat.data_ptr() + self.lo * self.flat.element_size()

    def check(self, name):
        torch.cuda.synchronize()
        f = self.flat.cpu()
        assert _same_bits(f[:self.lo], self.before) and _same_bits(f[self.lo + self.n:], self.after), f"{name}: wrote outside its buffer"

    def cpu(self):
        return self.t.cpu()


def _ints(t, raw=True):
    """The bit patterns of t; unless raw, every NaN but the sentinel becomes one pattern (x86 and the GPU give 0/0
    different payloads, and the header states only that it is NaN)."""
    t = torch.as_tensor(t).contiguous()
    if t.dtype != torch.float32:
        return t
    b = t.view(torch.int32).clone()
    if not raw:
        b[torch.isnan(t) & (b != FSENT)] = 0x7FC00000
    return b


def _same_bits(a, b):
    return torch.equal(_ints(a), _ints(b))


def _cmp(got, want, name, raw=False):
    """Bit-for-bit equality of two host tensors, sentinels included; computed NaNs compare as NaN unless raw."""
    g, w = _ints(got, raw), _ints(torch.as_tensor(want), raw)
    assert g.shape == w.shape, f"{name}: shape {tuple(g.shape)}, want {tuple(w.shape)}"
    bad = g != w
    if bool(bad.any()):
        at = bad.nonzero()[:4].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())} of {g.numel()} entries differ, first at {at}: got "
                             f"{[torch.as_tensor(got)[tuple(i)].item() for i in at]} want {[torch.as_tensor(want)[tuple(i)].item() for i in at]}")


def _sentinel(shape, dtype):
    if dtype == torch.float32:
        return torch.full(shape, FSENT, dtype=torch.int32).view(torch.float32)
    return torch.full(shape, SENT, dtype=dtype)


def _bits_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a).astype(np.uint32).view(np.int32))


def _f32(x):
    return float(np.float32(x))


def _next(x, d):
    return float(np.nextafter(np.float32(x), np.float32(d), dtype=np.float32))


# ------------------------------------------------------------------------------------------------
# candidates
# ------------------------------------------------------------------------------------------------
RULES = {  # (mask_threshold, stability_offset, pred_iou_thresh, stability_thresh, min_area)
    "plain": (0.0, 1.0, 0.0, 0.0, 0),
    "filters": (0.0, 1.0, 0.5, 0.4, 3),       # about half of the rows pass each filter
    "thr_rounds": (0.3, 1e-8, 0.0, 0.5, 1),    # 0.3f +- 1e-8f rounds back to 0.3f: hi == lo == thr
    "neg_offset": (0.25, -0.5, 0.0, 0.9, -3),  # hi < lo: stability > 1, or +inf where nothing exceeds lo
    "min_area_big": (0.0, 1.0, 0.0, 0.0, None),  # None: N + 1, so nothing survives
}


def _logits(Z, C, N, seed, thr=0.0, off=1.0, special=False):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((Z, C, N)) * 2 + thr).astype(np.float32)
    if special:
        hi, lo = np.float32(np.float32(thr) + np.float32(off)), np.float32(np.float32(thr) - np.float32(off))
        pool = np.array([NAN, INF, -INF, 0.0, -0.0, thr, _next(thr, INF), _next(thr, -INF), hi, lo, _next(hi, INF),
                         _next(lo, -INF), _next(hi, -INF), _next(lo, INF)], dtype=np.float32)
        at = g.random((Z, C, N)) < 0.35
        x[at] = pool[g.integers(0, len(pool), int(at.sum()))]
    return torch.from_numpy(x)


def _ious(Z, C, seed, special=False):
    g = np.random.default_rng(seed)
    x = g.random((Z, C)).astype(np.float32)
    if special:
        pool = np.array([NAN, INF, -INF, -0.0, 0.0, 0.5, _next(0.5, INF), 1e-45, -1e-45, 0.75], dtype=np.float32)
        at = g.random((Z, C)) < 0.5
        x[at] = pool[g.integers(0, len(pool), int(at.sum()))]
    return torch.from_numpy(x)


def _rules(name, N):
    thr, off, iou_t, stab_t, min_area = RULES[name]
    return thr, off, iou_t, stab_t, (N + 1 if min_area is None else min_area)


def _run_cand(logits, iou, B, W, base, stride, rules, *, lengths=None, P=0, misalign=False, single=False):
    """psam_mask_candidates_{f32, batched_f32, varlen_f32} on guarded windows of B * stride slots (one slot block of
    `stride` slots per cloud).  Returns (bits, area, stability, score) of the whole slot range on the host."""
    nv = _nv()
    Z, C, Ns = logits.shape
    Zc = Z // B
    thr, off, iou_t, stab_t, min_area = rules
    lg, io = Win(logits, offset=1 if misalign else 0), Win(iou)
    S = B * stride
    bits, area = Win(shape=(S, W), dtype=torch.int32, fill=SENT), Win(shape=(S,), dtype=torch.int32, fill=SENT)
    stab, score = Win(shape=(S,)), Win(shape=(S,))
    outs = (bits.ptr, area.ptr, stab.ptr, score.ptr, nv.stream())
    ins = [(lg, "logits"), (io, "iou_preds")]
    if lengths is not None:
        ln = Win(torch.tensor(lengths, dtype=torch.int32), fill=SENT)
        ins.append((ln, "lengths"))
        rc = nv.lib().psam_mask_candidates_varlen_f32(lg.ptr, io.ptr, ln.ptr, B, Zc, C, Ns, P, thr, off, iou_t, stab_t, min_area,
                                                      base, stride, W, *outs)
    elif single:
        assert B == 1
        rc = nv.lib().psam_mask_candidates_f32(lg.ptr, io.ptr, Z, C, Ns, thr, off, iou_t, stab_t, min_area, base, W, *outs)
    else:
        rc = nv.lib().psam_mask_candidates_batched_f32(lg.ptr, io.ptr, B, Zc, C, Ns, thr, off, iou_t, stab_t, min_area, base, stride,
                                                       W, *outs)
    assert rc == 0
    for w, name in ins + [(bits, "bits"), (area, "area"), (stab, "stability"), (score, "score")]:
        w.check(name)
    return bits.cpu(), area.cpu(), stab.cpu(), score.cpu()


def _want_cand(logits, iou, B, W, base, stride, rules, *, lengths=None, P=0):
    """amg_ref.candidates on every cloud's own (unpadded) rows, placed in the slot layout; sentinels everywhere else."""
    from oracle import amg_ref

    Z, C, Ns = logits.shape
    Zc = Z // B
    thr, off, iou_t, stab_t, min_area = rules
    S = B * stride
    bits, area = _sentinel((S, W), torch.int32), _sentinel((S,), torch.int32)
    stab, score = _sentinel((S,), torch.float32), _sentinel((S,), torch.float32)
    for b in range(B):
        N = Ns if lengths is None else min(max(lengths[b], 0), Ns)
        r = amg_ref.candidates(logits[b * Zc:(b + 1) * Zc, :, :N].numpy(), iou[b * Zc:(b + 1) * Zc].numpy(), thr, off, iou_t, stab_t,
                               min_area, W)
        sc = r["score"].copy()
        if lengths is not None:  # prompt j owns slots j*C .. j*C+C-1 of the block, counted from the block start, base included
            sc[(base + np.arange(Zc * C)) // C >= min(P, N)] = -np.inf
        s0 = b * stride + base
        bits[s0:s0 + Zc * C] = _bits_i32(r["bits"])
        area[s0:s0 + Zc * C] = torch.from_numpy(r["area"])
        stab[s0:s0 + Zc * C] = torch.from_numpy(r["stability"])
        score[s0:s0 + Zc * C] = torch.from_numpy(sc)
    return bits, area, stab, score


def _check_cand(got, want, name):
    for g, w, what in zip(got, want, ("bits", "area", "stability", "score")):
        _cmp(g, w, f"{name} {what}")


_CAND_SHAPES = [(N, dW, mis) for N in (1, 3, 4, 31, 32, 33, 127, 128, 129, 4100) for dW in (0, 1, 5)
                for mis in ((False, True) if N % 4 == 0 else (False,))]


@pytest.mark.parametrize("N,dW,misalign", _CAND_SHAPES,
                         ids=[_id(cand_kernel(N, not m), N=N, W=-(-N // 32) + d, ptr="+4B" if m else "16B") for N, d, m in _CAND_SHAPES])
def test_candidates_shapes(N, dW, misalign):
    """Two clouds of 3 x 3 rows in one launch, with base > 0 and cloud_stride > base + Zc*C (gaps that stay untouched), W
    up to five words past ceil(N/32) (written zero), and logits behind a pointer offset by one float where N % 4 == 0."""
    B, Zc, C, base = 2, 3, 3, 3
    W, stride = -(-N // 32) + dW, base + Zc * C + 5
    lg, io = _logits(B * Zc, C, N, N * 10 + dW), _ious(B * Zc, C, N)
    rules = _rules("filters", N)
    got = _run_cand(lg, io, B, W, base, stride, rules, misalign=misalign)
    _check_cand(got, _want_cand(lg, io, B, W, base, stride, rules), f"N={N} W={W}")
    print(f"[amg] candidates {cand_kernel(N, not misalign)} N={N} W={W}: {int((got[3] > -INF).sum())} of {B * Zc * C} survive")


_CAND_ROWS = [(1, 1, 128, False), (1, 1, 33, False), (22000, 3, 4, False), (22000, 3, 3, False), (16500, 4, 8, True)]


@pytest.mark.parametrize("Z,C,N,misalign", _CAND_ROWS,
                         ids=[_id(cand_kernel(N, not m), rows=Z * C, N=N) for Z, C, N, m in _CAND_ROWS])
def test_candidates_rows(Z, C, N, misalign):
    """One row, and more than 65535 rows (one CTA per row), through the single-cloud entry point."""
    W, base = -(-N // 32) + 1, 2
    lg, io = _logits(Z, C, N, Z + N, special=True), _ious(Z, C, Z, special=True)
    rules = _rules("plain", N)
    stride = base + Z * C + 3
    got = _run_cand(lg, io, 1, W, base, stride, rules, misalign=misalign, single=True)
    _check_cand(got, _want_cand(lg, io, 1, W, base, stride, rules), f"rows={Z * C} N={N}")


_CAND_SPECIAL = [(r, N, m) for r in RULES for N, m in ((128, False), (128, True), (33, False))]


@pytest.mark.parametrize("rule,N,misalign", _CAND_SPECIAL,
                         ids=[_id(cand_kernel(N, not m), rule=r, N=N, ptr="+4B" if m else "16B") for r, N, m in _CAND_SPECIAL])
def test_candidates_special(rule, N, misalign):
    """Logits that are NaN, +-inf, +-0 and one ulp either side of the threshold and of thr +- offset; a threshold where
    thr +- offset rounds back to thr; a negative offset (stability > 1 or +inf); predicted IoUs that are NaN, +-inf, -0.0,
    subnormal; min_area <= 0, 1 and N + 1.  Scores keep the IoU's bit pattern (-0.0 included)."""
    B, Zc, C, base = 2, 4, 3, 1
    W, stride = -(-N // 32) + 1, base + Zc * C + 2
    rules = _rules(rule, N)
    lg = _logits(B * Zc, C, N, list(RULES).index(rule) * 1000 + N, thr=rules[0], off=rules[1], special=True)
    io = _ious(B * Zc, C, N + 1, special=True)
    got = _run_cand(lg, io, B, W, base, stride, rules, misalign=misalign)
    _check_cand(got, _want_cand(lg, io, B, W, base, stride, rules), f"{rule} N={N}")
    st = got[2][got[2] == got[2]]
    print(f"[amg] candidates {rule} N={N}: stability in [{float(st.min()) if len(st) else NAN}, {float(st.max()) if len(st) else NAN}], "
          f"{int((got[3] > -INF).sum())} survive")


_CAND_VARLEN = [  # (N_max, lengths, Zc, C, P, base, misalign)
    (129, [1, 129, 64, 100], 4, 3, 3, 0, False),
    (128, [1, 128, 33, 127], 4, 3, 4, 5, False),
    (128, [1, 128, 33, 127], 4, 3, 4, 5, True),
    (4100, [4100, 1, 2049, 4097], 5, 3, 0, 0, False),
    (4100, [4100, 1, 2049, 4097], 5, 3, 2, 4, False),
    (33, [33, 2, 1], 6, 1, 4, 3, False),
]


@pytest.mark.parametrize("Nmax,lengths,Zc,C,P,base,misalign", _CAND_VARLEN,
                         ids=[_id(cand_kernel(n, not m, True), Nmax=n, B=len(l), P=p, base=b, ptr="+4B" if m else "16B")
                              for n, l, _, _, p, b, m in _CAND_VARLEN])
def test_candidates_varlen(Nmax, lengths, Zc, C, P, base, misalign):
    """Padded clouds of lengths 1, N_max and mixed, P = 0 and P < Zc, base > 0 (and not a multiple of C), so the prompt
    index of a slot is counted from the block start, base included.  Padding logits are +1e9: counted if read."""
    B = len(lengths)
    W, stride = -(-Nmax // 32) + 1, base + Zc * C + 4
    rules = _rules("plain", Nmax)  # every non-empty mask with a non-NaN IoU survives: the prompt cut decides
    lg, io = _logits(B * Zc, C, Nmax, Nmax + P, special=True), _ious(B * Zc, C, P + 7, special=True)
    for b, L in enumerate(lengths):
        lg[b * Zc:(b + 1) * Zc, :, L:] = 1e9
    got = _run_cand(lg, io, B, W, base, stride, rules, lengths=lengths, P=P, misalign=misalign)
    _check_cand(got, _want_cand(lg, io, B, W, base, stride, rules, lengths=lengths, P=P), f"varlen Nmax={Nmax} P={P}")
    print(f"[amg] candidates varlen Nmax={Nmax} lengths={lengths} P={P} base={base}: {int((got[3] > -INF).sum())} of {B * Zc * C} survive")


@pytest.mark.parametrize("Nmax", [128, 129], ids=[_id(cand_kernel(n, True, True), Nmax=n) for n in (128, 129)])
def test_candidates_varlen_out_of_range(Nmax):
    """Lengths of 0, negative and past N_max: their values are unspecified, but nothing outside the clouds' slot blocks
    may be written, and an in-range cloud of the same launch is exact."""
    lengths, Zc, C, base, P = [0, -3, Nmax + 5, 7], 3, 2, 2, 2
    B, W, stride = len(lengths), -(-Nmax // 32) + 2, base + Zc * C + 3
    rules = _rules("plain", Nmax)
    lg, io = _logits(B * Zc, C, Nmax, 5), _ious(B * Zc, C, 5)
    got = _run_cand(lg, io, B, W, base, stride, rules, lengths=lengths, P=P)
    want = _want_cand(lg, io, B, W, base, stride, rules, lengths=lengths, P=P)
    inside = torch.zeros(B * stride, dtype=torch.bool)
    for b in range(B):
        inside[b * stride + base:b * stride + base + Zc * C] = True
    for g, w, what in zip(got, want, ("bits", "area", "stability", "score")):
        _cmp(g[~inside], w[~inside], f"out-of-range lengths {what} outside the blocks")
        _cmp(g[3 * stride:4 * stride], w[3 * stride:4 * stride], f"in-range cloud {what}")


# ------------------------------------------------------------------------------------------------
# NMS
# ------------------------------------------------------------------------------------------------
def _nms_masks(B, K, N, seed, groups=64, empty=0):
    """bool [B, K, N]: noisy copies of `groups` prototypes (copies overlap above 0.7, prototypes below), `empty` empty
    masks per cloud."""
    g = np.random.default_rng(seed)
    proto = g.random((B, groups, N)) < g.uniform(0.2, 0.6, (B, groups, 1))
    m = proto[np.arange(B)[:, None], g.integers(0, groups, (B, K))] ^ (g.random((B, K, N)) < 0.03)
    for b in range(B):
        if K:
            m[b, g.choice(K, min(empty, K), replace=False)] = False
    return m


def _nms_scores(B, K, kind, seed, valid=None):
    g = np.random.default_rng(seed)
    if kind == "random":
        s = g.random((B, K)).astype(np.float32)
    elif kind == "ties":  # long runs of equal scores
        s = np.array([0.25, 0.5, 0.75], dtype=np.float32)[g.integers(0, 3, (B, K))]
    else:  # special values
        pool = np.array([NAN, INF, -INF, 0.0, -0.0, 1e-45, 2e-45, -1e-45, 1.17e-38, 1.0, 0.5], dtype=np.float32)
        s = pool[g.integers(0, len(pool), (B, K))]
    if kind != "special":
        s[g.random((B, K)) < 0.1] = -np.inf
    if valid is not None:  # exactly valid[b] candidates keep a score
        for b, v in enumerate(valid):
            s[b] = np.float32(g.random(K))
            s[b, g.permutation(K)[v:]] = -np.inf
    return s


def _run_nms(bits, area, score, thr):
    """psam_mask_nms_batched on guarded windows.  Returns (keep [B, K], keep_count [B]) on the host."""
    nv = _nv()
    B, K, W = bits.shape
    bw, aw, sw = Win(bits), Win(area), Win(score)
    keep, cnt = Win(shape=(B, K), dtype=torch.int32, fill=SENT), Win(shape=(B,), dtype=torch.int32, fill=SENT)
    nb = nv.lib().psam_mask_nms_batched_workspace_bytes(B, K, W)
    ws = Win(shape=(nb // 4,), dtype=torch.int32, fill=SENT)
    rc = nv.lib().psam_mask_nms_batched(bw.ptr, aw.ptr, sw.ptr, B, K, W, thr, keep.ptr, cnt.ptr, ws.ptr, nv.stream())
    assert rc == 0
    for w, name in ((bw, "bits"), (aw, "area"), (sw, "score"), (keep, "keep"), (cnt, "keep_count"), (ws, "workspace")):
        w.check(name)
    return keep.cpu(), cnt.cpu()


def _want_nms(bits, area, score, thr):
    from oracle import amg_ref

    B, K, _ = bits.shape
    keep, cnt = _sentinel((B, K), torch.int32), torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        k = amg_ref.nms(bits[b].numpy().view(np.uint32), area[b].numpy(), score[b].numpy(), np.float32(thr))
        keep[b, :len(k)] = torch.from_numpy(k.astype(np.int32))
        cnt[b] = len(k)
    return keep, cnt


def _nms_case(masks, score, thr, W=None, name=""):
    from oracle import amg_ref

    B, K, N = masks.shape
    W = W or max(-(-N // 32), 1)
    bits = torch.stack([_bits_i32(amg_ref.pack_bits(masks[b], W)) for b in range(B)]) if K else torch.zeros(B, 0, W, dtype=torch.int32)
    area = torch.from_numpy(masks.sum(-1).astype(np.int32))
    score = torch.from_numpy(np.asarray(score, dtype=np.float32))
    keep, cnt = _run_nms(bits, area, score, thr)
    wk, wc = _want_nms(bits, area, score, thr)
    _cmp(cnt, wc, f"{name} keep_count")
    _cmp(keep, wk, f"{name} keep")
    return keep, cnt


_NMS_K = [(K, kind) for K in (0, 1, 63, 64, 65, 4096, 4097, 16383, 16384) for kind in ("random", "ties")]
_NMS_K += [(200, "special"), (4097, "special")]


@pytest.mark.parametrize("K,kind", _NMS_K, ids=[f"nms-K{K}-{kind}" for K, kind in _NMS_K])
def test_nms_k(K, kind):
    """K around the 64-tiles, and 4096 / 4097 where nms_order_kernel's keys cross the 48 KB dynamic shared-memory
    attribute; ties, NaN, +inf, +-0.0, subnormals and empty masks (a 0/0 IoU) among the scores."""
    B = 2 if K <= 4097 else 1
    masks = _nms_masks(B, K, 200, K + len(kind), empty=3)
    keep, cnt = _nms_case(masks, _nms_scores(B, K, kind, K), 0.7, name=f"K={K} {kind}")
    print(f"[amg] nms K={K} {kind}: kept {cnt.tolist()}")


_NMS_VALID = [(300, [0, 64, 65, 128]), (300, [63, 1, 300, 129]), (4097, [4096, 4097]), (200, [192, 193])]


@pytest.mark.parametrize("K,valid", _NMS_VALID, ids=[f"nms-K{K}-valid{'_'.join(map(str, v))}" for K, v in _NMS_VALID])
def test_nms_valid_counts(K, valid):
    """Clouds of one launch with different valid counts, 0 included, ending on and just past a 64-tile."""
    B = len(valid)
    _nms_case(_nms_masks(B, K, 96, K, groups=24), _nms_scores(B, K, "random", K + 1, valid=valid), 0.5, W=4, name=f"valid={valid}")


@pytest.mark.parametrize("thr", [-1.0, 0.0, 1.0, NAN], ids=["nms-thr-1", "nms-thr0", "nms-thr1", "nms-thrNaN"])
def test_nms_thresholds(thr):
    """nms_thresh < 0 (every non-NaN IoU suppresses), 0, 1 (nothing suppresses) and NaN (nothing suppresses)."""
    masks = _nms_masks(2, 150, 64, 9, groups=10, empty=4)
    _, cnt = _nms_case(masks, _nms_scores(2, 150, "special", 3), thr, name=f"thr={thr}")
    print(f"[amg] nms thr={thr}: kept {cnt.tolist()}")


def test_nms_iou_equal_to_threshold():
    """Integer-built masks whose fp32 IoU equals nms_thresh exactly (2/4 = 0.5, 1/3 = fp32(1/3)): the comparison is strict,
    so neither suppresses; one point more of overlap does."""
    N = 64
    m = np.zeros((1, 6, N), dtype=bool)
    m[0, 0, [0, 1, 2]] = True          # area 3
    m[0, 1, [1, 2, 3]] = True          # inter 2, union 4 with 0: IoU 0.5
    m[0, 2, [10, 11]] = True           # area 2
    m[0, 3, [11, 12]] = True           # inter 1, union 3 with 2: IoU 1/3
    m[0, 4, [20, 21, 22, 23]] = True
    m[0, 5, [20, 21, 22, 24]] = True   # inter 3, union 5: 0.6
    score = np.array([[0.9, 0.8, 0.7, 0.6, 0.5, 0.4]], dtype=np.float32)
    keep, cnt = _nms_case(m, score, 0.5, name="IoU 0.5 at 0.5")
    assert keep[0, :int(cnt[0])].tolist() == [0, 1, 2, 3, 4]
    keep, cnt = _nms_case(m, score, _f32(1 / 3), name="IoU 1/3 at 1/3")
    assert keep[0, :int(cnt[0])].tolist() == [0, 2, 3, 4]


@pytest.mark.parametrize("slots", [(3, 7), (7, 3)], ids=["nms-zero-minus_first", "nms-zero-plus_first"])
def test_nms_signed_zero(slots):
    """-0.0 ranks equal to +0.0: the lower slot goes first, whichever zero it holds, and suppresses its identical twin."""
    lo, hi = slots
    m = np.zeros((1, 10, 64), dtype=bool)
    for k in range(10):
        m[0, k, 6 * k:6 * k + 5] = True
    m[0, hi] = m[0, lo]
    score = np.full((1, 10), -np.inf, dtype=np.float32)
    score[0, lo], score[0, hi] = -0.0, 0.0
    score[0, 0] = -1e-45  # below both zeros
    keep, cnt = _nms_case(m, score, 0.5, name=f"-0.0 at slot {lo}, +0.0 at slot {hi}")
    assert keep[0, :int(cnt[0])].tolist() == [min(lo, hi), 0]


# ------------------------------------------------------------------------------------------------
# small regions
# ------------------------------------------------------------------------------------------------
def _graph(kind, N, k1, rng, length=None):
    """int64 [N, k1] host-built graphs that stress a concurrent union-find.  With `length`, entries that would reach past
    the cloud point at padding rows length .. N-1 instead (present, but no edge)."""
    L = N if length is None else length
    i = np.arange(N)[:, None]
    if kind == "window":  # kNN-like: nearby indices in random order, some -1
        g = np.clip(i + rng.integers(-3, 4, (N, k1)), 0, L - 1)
        g[rng.random((N, k1)) < 0.05] = -1
    elif kind == "chain_up":  # each point lists the next one only: hooked from the top in the worst order
        g = np.repeat(i + 1, k1, 1)
    elif kind == "chain_down":
        g = np.repeat(i - 1, k1, 1)
    elif kind == "chain_perm":  # a chain over a random order of the points, each edge listed on one side
        p = rng.permutation(L)
        g = np.full((N, k1), -1)
        g[p[:-1]] = p[1:, None]
    elif kind == "star":  # every point lists point 0 (and itself)
        g = np.zeros((N, k1), dtype=np.int64)
        g[:, 1:] = i
    elif kind == "full":  # k1 = N: each row lists every point, in a row-specific order
        g = np.stack([rng.permutation(N) for _ in range(N)])
    elif kind == "messy":  # self-loops, repeated entries, -1, one-sided window edges
        g = np.clip(i + rng.integers(-4, 5, (N, k1)), 0, L - 1)
        g[:, 0] = i[:, 0]
        g[:, 1] = g[:, 2]
        g[rng.random((N, k1)) < 0.1] = -1
    else:
        raise ValueError(kind)
    g = np.where((g >= L) | (g < -1), -1, g)
    if length is not None and length < N:  # in-range poison: entries that point at padding rows, which exist
        pad = rng.random((N, k1)) < 0.2
        g[pad] = rng.integers(L, N, int(pad.sum()))
        g[L:] = rng.integers(0, N, (N - L, k1))  # padding rows: edges into the cloud
    return g.astype(np.int64)


def _runs_mask(N, rng, mean):
    """Alternating in / out runs of lengths around `mean`: components on both sides near min_area."""
    m = np.zeros(N, dtype=bool)
    pos, inside = 0, bool(rng.integers(2))
    while pos < N:
        r = int(rng.integers(1, 2 * mean + 2)) if rng.random() < 0.9 else int(rng.integers(1, 8 * mean))
        m[pos:pos + r] = inside
        pos, inside = pos + r, not inside
    return m


def _region_inputs(B, Kc, K, Ns, counts, lengths, rng, mean):
    """Candidate bits [B, Kc, W] with set bits past each cloud's N in its last word and set words past ceil(N/32), and keep
    [B, K] of distinct slots whose entries past the count name other valid slots."""
    from oracle import amg_ref

    W = -(-Ns // 32) + 2
    bits = np.zeros((B, Kc, W), dtype=np.uint32)
    for b in range(B):
        N = Ns if lengths is None else lengths[b]
        m = np.stack([_runs_mask(N, rng, mean) for _ in range(Kc)])
        bits[b, :, :-(-N // 32)] = amg_ref.pack_bits(m)
        if N % 32:
            bits[b, :, N // 32] |= np.uint32(0xFFFFFFFF << (N % 32) & 0xFFFFFFFF) & rng.integers(0, 2 ** 32, Kc, dtype=np.uint64).astype(np.uint32)
        bits[b, :, -(-N // 32):] = rng.integers(0, 2 ** 32, (Kc, W - (-(-N // 32))), dtype=np.uint64).astype(np.uint32)
    keep = np.stack([rng.permutation(Kc)[:K] for _ in range(B)]).astype(np.int32)
    return torch.from_numpy(bits.view(np.int32)), torch.from_numpy(keep)


def _run_regions(bits, keep, counts, nbr, min_area, lengths=None, single=False):
    """psam_mask_regions{, _batched, _varlen} on guarded windows.  Returns (bits_out [B, K, W], area_out, score_out)."""
    nv = _nv()
    B, Kc, W = bits.shape
    K, Ns, k1 = keep.shape[1], nbr.shape[1], nbr.shape[2]
    bw, kw = Win(bits, fill=SENT), Win(keep, fill=SENT)
    cw, gw = Win(torch.tensor(counts, dtype=torch.int32), fill=SENT), Win(torch.as_tensor(nbr), fill=SENT)
    bo, ao = Win(shape=(B, K, W), dtype=torch.int32, fill=SENT), Win(shape=(B, K), dtype=torch.int32, fill=SENT)
    so = Win(shape=(B, K))
    nb = nv.lib().psam_mask_regions_batched_workspace_bytes(B, K, Ns)
    ws = Win(shape=(nb // 4,), dtype=torch.int32, fill=SENT)
    ins = [(bw, "bits"), (kw, "keep"), (cw, "keep_count"), (gw, "nbr")]
    outs = (bo.ptr, ao.ptr, so.ptr, ws.ptr, nv.stream())
    if lengths is not None:
        lw = Win(torch.tensor(lengths, dtype=torch.int32), fill=SENT)
        ins.append((lw, "lengths"))
        rc = nv.lib().psam_mask_regions_varlen(bw.ptr, Kc, lw.ptr, B, K, W, Ns, kw.ptr, cw.ptr, gw.ptr, k1, min_area, *outs)
    elif single:
        assert B == 1
        rc = nv.lib().psam_mask_regions(bw.ptr, K, W, Ns, kw.ptr, cw.ptr, gw.ptr, k1, min_area, *outs)
    else:
        rc = nv.lib().psam_mask_regions_batched(bw.ptr, Kc, B, K, W, Ns, kw.ptr, cw.ptr, gw.ptr, k1, min_area, *outs)
    assert rc == 0
    for w, name in ins + [(bo, "bits_out"), (ao, "area_out"), (so, "score_out"), (ws, "workspace")]:
        w.check(name)
    return bo.cpu(), ao.cpu(), so.cpu()


def _want_regions(bits, keep, counts, nbr, min_area, lengths=None):
    """amg_regions_ref.remove_small_regions (holes, then islands) on every kept rank of every cloud's own points and graph;
    ranks past the count: score -inf and nothing else."""
    from oracle import amg_ref, amg_regions_ref

    B, Kc, W = bits.shape
    K, Ns = keep.shape[1], nbr.shape[1]
    bo, ao, so = _sentinel((B, K, W), torch.int32), _sentinel((B, K), torch.int32), _sentinel((B, K), torch.float32)
    ub = bits.numpy().view(np.uint32)
    for b in range(B):
        N = Ns if lengths is None else min(max(lengths[b], 0), Ns)
        g = np.asarray(nbr[b, :N])
        for p in range(K):
            if p >= counts[b]:
                so[b, p] = -INF
                continue
            m = amg_ref.unpack_bits(ub[b, int(keep[b, p])][None], N)[0]
            m, ch = amg_regions_ref.remove_small_regions(m, g, min_area, "holes")
            m, ci = amg_regions_ref.remove_small_regions(m, g, min_area, "islands")
            bo[b, p] = _bits_i32(amg_ref.pack_bits(m[None], W)[0])
            ao[b, p] = int(m.sum())
            so[b, p] = 0.0 if (ch or ci) else 1.0
    return bo, ao, so


def _check_regions(got, want, name):
    for g, w, what in zip(got, want, ("bits_out", "area_out", "score_out")):
        _cmp(g, w, f"{name} {what}")


_REGIONS = [  # (Ns, lengths, B, K, counts, k1, graph, min_area, mean)
    (1, None, 1, 2, [1], 1, "window", 1, 1),
    (31, None, 2, 4, [4, 3], 31, "full", 3, 3),
    (32, None, 2, 5, [5, 2], 1, "chain_up", 4, 3),
    (33, None, 1, 6, [6], 2, "chain_down", 3, 3),
    (129, None, 1, 6, [6], 3, "star", 1, 5),
    (129, None, 1, 6, [6], 3, "chain_perm", 500, 5),
    (1024, None, 3, 100, [100, 99, 97], 9, "messy", 12, 10),
    (49152, None, 1, 6, [6], 9, "window", 40, 30),
    (49153, None, 1, 6, [5], 5, "window", 40, 30),
    (200003, None, 2, 24, [24, 21], 4, "window", 30, 25),
    (1024, [1024, 1, 500, 33], 4, 8, [8, 1, 7, 8], 9, "messy", 10, 8),
    (49153, [49153, 40000, 2], 3, 4, [4, 4, 4], 5, "chain_perm", 20, 15),
    (200003, [200003, 70001], 2, 20, [20, 20], 4, "window", 30, 25),
]


def _regions_id(Ns, lengths, B, K, counts, k1, graph, min_area, mean):
    items = B * K
    return _id(region_kernel(Ns, lengths is not None), N=Ns, B=B, items=items, grid=region_grid(items, Ns), k1=k1, g=graph,
               min=min_area)


@pytest.mark.parametrize("Ns,lengths,B,K,counts,k1,graph,min_area,mean", _REGIONS, ids=[_regions_id(*c) for c in _REGIONS])
def test_regions(Ns, lengths, B, K, counts, k1, graph, min_area, mean):
    """Every instantiation on host-built graphs (kNN-like windows, chains hooked in the worst order, stars, one-sided
    edges, self-loops, repeated and -1 entries, k1 of 1 and of N), with set bits past N and set words past ceil(N/32) in
    the candidates, min_area of 1 and more than N, and more items than CTAs in both forms: B*K > 2*SMs with counts close
    to K in shared memory, and about 31 label slices for 40-48 items at N ~ 200000.  In the padded batches a slice first
    serves a long cloud and then a short one, and graph entries past a cloud's length point at padding rows."""
    rng = np.random.default_rng(Ns + B * K + k1)
    Kc = K + 3
    bits, keep = _region_inputs(B, Kc, K, Ns, counts, lengths, rng, mean)
    nbr = torch.from_numpy(np.stack([_graph(graph, Ns, k1, rng, None if lengths is None else lengths[b]) for b in range(B)]))
    single = B == 1 and lengths is None and Ns < 100
    got = _run_regions(bits, keep, counts, nbr, min_area, lengths, single=single)
    _check_regions(got, _want_regions(bits, keep, counts, nbr, min_area, lengths), f"N={Ns} {graph}")
    grid = region_grid(B * K, Ns, _sms())
    reuse = ""
    if Ns > REGION_SMEM_MAX_N and lengths is not None:
        later = [i for i in range(grid, B * K) if i % K < counts[i // K]]  # items a CTA serves after its first one
        longer = sum(lengths[i // K] < lengths[(i % grid) // K] for i in later)
        reuse = f", {longer} items reuse a slice a longer cloud used before"
    print(f"[amg] regions {region_kernel(Ns, lengths is not None)} N={Ns}: {B * K} items on {grid} CTAs{reuse}; "
          f"changed {int((got[2] == 0).sum())}, unchanged {int((got[2] == 1).sum())}")


def _hand_masks(N):
    """Masks on the chain 0-1-...-N-1 (chain_up) with min_area 5: equal largest islands below min_area (10..13 has the
    smallest root), islands of exactly min_area and min_area - 1, holes of both sizes, an empty and a full mask."""
    m = np.zeros((6, N), dtype=bool)
    for a in (40, 10, 25):
        m[0, a:a + 4] = True
    m[1, 0:5] = True
    m[1, 20:24] = True
    m[2, 0:30] = True
    m[2, 10:14] = False
    m[2, 20:25] = False
    m[4, :] = True
    m[5, 50:54] = True
    m[5, 2:6] = True
    return m


@pytest.mark.parametrize("N,min_area", [(64, 5), (64, 65), (49153, 5)],
                         ids=[_id(region_kernel(n), N=n, min=a) for n, a in ((64, 5), (64, 65), (49153, 5))])
def test_regions_hand(N, min_area):
    """Hand-built masks on a chain: ties for the largest component below min_area (the smallest root wins), components of
    exactly min_area and min_area - 1, an empty kept mask, and min_area > N (the empty mask fills up)."""
    from oracle import amg_ref

    m = _hand_masks(N)
    K, W = len(m), -(-N // 32) + 1
    bits = _bits_i32(amg_ref.pack_bits(m, W))[None]
    keep = torch.arange(K, dtype=torch.int32)[None]
    nbr = torch.from_numpy(_graph("chain_up", N, 1, np.random.default_rng(0))[None])
    got = _run_regions(bits, keep, [K], nbr, min_area)
    want = _want_regions(bits, keep, [K], nbr, min_area)
    _check_regions(got, want, f"hand N={N} min_area={min_area}")
    if min_area == 5:
        kept = np.nonzero(amg_ref.unpack_bits(got[0][0, 0:1].numpy().view(np.uint32), N)[0])[0]
        assert kept.tolist() == [10, 11, 12, 13]


# ------------------------------------------------------------------------------------------------
# crop edge filter and uncrop
# ------------------------------------------------------------------------------------------------
def _edge_inputs(T, K, W, rng):
    bits = (rng.random((T, K, W * 32)) < 0.004)
    edge = (rng.random((T, W * 32)) < 0.05)
    if W > 32:  # rows whose only hit is in a word a lane reaches on its second pass
        edge[:, 33 * 32 + 5] = True
        bits[:, ::5] = False
        bits[:, ::5, 33 * 32 + 5] = True
    pool = np.array([0xFFC0BEEF, 0x80000000, 0, 0x7F800000, 0xFF800000, 0x3F000000, 1], dtype=np.uint32)  # -NaN with a
    score = pool[rng.integers(0, len(pool), (T, K))].view(np.float32)  # payload, -0.0, +0.0, +inf, -inf, 0.5, a subnormal
    pb = np.packbits(bits, axis=-1, bitorder="little").view("<u4")
    pe = np.packbits(edge, axis=-1, bitorder="little").view("<u4")
    return torch.from_numpy(pb.view(np.int32).copy()), torch.from_numpy(pe.view(np.int32).copy()), torch.from_numpy(score)


_EDGE = [(False, 1, 5, 1), (False, 1, 9000, 40), (False, 1, 0, 3), (True, 3, 9000, 40), (True, 2, 7, 3), (True, 2, 0, 3)]


@pytest.mark.parametrize("batch,T,K,W", _EDGE, ids=[_id(f"crop_edge_filter_kernel<{_tf(b)}>", T=t, K=k, W=w) for b, t, k, w in _EDGE])
def test_crop_edge_filter(batch, T, K, W):
    """Only the scores of rows that hit the edge bitset become -inf; the others keep their bit patterns (NaN and -0.0
    included).  K = 9000 crosses the grid stride of 1024 CTAs x 8 warps, and W = 40 > 32 takes the lane loop twice."""
    nv = _nv()
    rng = np.random.default_rng(K + W + T)
    bits, edge, score = _edge_inputs(T, K, W, rng)
    bw, ew, sw = Win(bits, fill=SENT), Win(edge, fill=SENT), Win(score)
    if batch:
        rc = nv.lib().psam_crop_edge_filter_batched(bw.ptr, T, K, W, ew.ptr, sw.ptr, nv.stream())
    else:
        rc = nv.lib().psam_crop_edge_filter(bw.ptr, K, W, ew.ptr, sw.ptr, nv.stream())
    assert rc == 0
    for w, name in ((bw, "bits"), (ew, "edge"), (sw, "score")):
        w.check(name)
    hit = ((bits.numpy().view(np.uint32) & edge.numpy().view(np.uint32)[:, None, :]) != 0).any(-1)
    want = score.clone()
    want[torch.from_numpy(hit)] = -INF
    _cmp(sw.cpu(), want, "edge filter score", raw=True)
    _cmp(bw.cpu(), bits, "edge filter bits")
    print(f"[amg] edge filter batch={batch} T={T} K={K} W={W}: {int(hit.sum())} rows hit")


def _uncrop_run(rng, n, N, Z, slots, K, count, W_extra=1):
    """One crop's inputs: candidates of n local points (bits set past n), idx [n] distinct global points, prompt indices,
    a keep list of K distinct slots (entries past the count name other valid slots)."""
    from oracle import amg_ref

    Kc = Z * slots
    W = -(-n // 32) + W_extra
    m = rng.random((Kc, n)) < rng.uniform(0.05, 0.5, (Kc, 1))
    bits = np.zeros((Kc, W), dtype=np.uint32)
    bits[:, :-(-n // 32)] = amg_ref.pack_bits(m)
    if n % 32:
        bits[:, n // 32] |= np.uint32((0xFFFFFFFF << (n % 32)) & 0xFFFFFFFF)
    bits[:, -(-n // 32):] = 0xFFFFFFFF
    return dict(bits=torch.from_numpy(bits.view(np.int32)), m=m, area=torch.from_numpy(rng.integers(0, 1000, Kc).astype(np.int32)),
                score=torch.from_numpy(rng.random(Kc).astype(np.float32)), stab=torch.from_numpy(rng.random(Kc).astype(np.float32)),
                keep=torch.from_numpy(rng.permutation(Kc)[:K].astype(np.int32)), count=count,
                idx=torch.from_numpy(np.sort(rng.choice(N - 1, n, replace=False)).astype(np.int32)),  # never N - 1
                prompt=torch.from_numpy(rng.integers(0, n, Z).astype(np.int64)), slots=slots, n=n, W=W)


def _want_uncrop_rows(run, N, Wg, crop, layer_score, base, cap, outs):
    """Write run's rows base + p < cap into the host arrays outs = (gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore)."""
    from oracle import amg_ref

    for p in range(run["count"]):
        d = base + p
        if d >= cap:
            break
        s = int(run["keep"][p])
        z = s // run["slots"]
        g = np.zeros(N, dtype=bool)
        g[run["idx"].numpy()[run["m"][s]]] = True
        outs[0][d] = _bits_i32(amg_ref.pack_bits(g[None], Wg)[0])
        outs[1][d], outs[2][d], outs[3][d] = run["area"][s], run["score"][s], run["stab"][s]
        outs[4][d] = int(run["idx"][int(run["prompt"][z])])
        outs[5][d], outs[6][d], outs[7][d] = s - z * run["slots"], crop, _f32(layer_score)


def _out_windows(shape_rows, Wg):
    return [Win(shape=shape_rows + (Wg,), dtype=torch.int32, fill=SENT), Win(shape=shape_rows, dtype=torch.int32, fill=SENT),
            Win(shape=shape_rows), Win(shape=shape_rows), Win(shape=shape_rows, dtype=torch.int64, fill=SENT),
            Win(shape=shape_rows, dtype=torch.int32, fill=SENT), Win(shape=shape_rows, dtype=torch.int32, fill=SENT), Win(shape=shape_rows)]


_OUT_NAMES = ("gbits", "garea", "giou", "gstab", "gprompt", "gslot", "gcrop", "gscore")

_UNCROP = [(0, 40, 500), (3, 37, 40), (5, 40, 40), (40, 3, 40), (100, 550, 1000), (16000, 600, 16384)]


@pytest.mark.parametrize("off,count,cap", _UNCROP, ids=[_id("crop_uncrop_kernel<false>", off=o, count=c, cap=p) for o, c, p in _UNCROP])
def test_crop_uncrop(off, count, cap):
    """Uncrop writes rows [off, min(off + count, cap)), its offset and, past the capacity, the overflow flag - nothing
    else: not the rows before the offset, not those past the capacity, and not the flag when the set fits.  Local bits past
    n are ignored (the idx buffer's guards hold a valid point, so reading them would set a wrong bit); ranks past the
    grid of 264 CTAs loop."""
    nv = _nv()
    N, n, Z, slots = 5000, 1000, 300, 3
    K = max(count + 10, 1)
    rng = np.random.default_rng(off + count + cap)
    run = _uncrop_run(rng, n, N, Z, slots, K, count)
    Wg = -(-N // 32) + 1
    crop, layer_score = 7, 0.375
    ins = dict(bits=Win(run["bits"], fill=SENT), area=Win(run["area"], fill=SENT), score=Win(run["score"]), stab=Win(run["stab"]),
               keep=Win(run["keep"], fill=SENT), cnt=Win(torch.tensor([count], dtype=torch.int32), fill=SENT),
               idx=Win(run["idx"], fill=N - 1), prompt=Win(run["prompt"], fill=0), off=Win(torch.tensor([off], dtype=torch.int32), fill=SENT))
    offo, ovf = Win(shape=(1,), dtype=torch.int32, fill=SENT), Win(shape=(1,), dtype=torch.int32, fill=SENT)
    outs = _out_windows((cap,), Wg)
    rc = nv.lib().psam_crop_uncrop(ins["bits"].ptr, ins["area"].ptr, ins["score"].ptr, ins["stab"].ptr, K, run["W"], ins["keep"].ptr,
                                   ins["cnt"].ptr, ins["idx"].ptr, n, ins["prompt"].ptr, slots, crop, layer_score, N, Wg, cap,
                                   ins["off"].ptr, offo.ptr, *[o.ptr for o in outs], ovf.ptr, nv.stream())
    assert rc == 0
    for name, w in list(ins.items()) + [("offset_out", offo), ("overflow", ovf)] + list(zip(_OUT_NAMES, outs)):
        w.check(name)
    want = [_sentinel(tuple(o.t.shape), o.t.dtype) for o in outs]
    _want_uncrop_rows(run, N, Wg, crop, layer_score, off, cap, want)
    for o, w, name in zip(outs, want, _OUT_NAMES):
        _cmp(o.cpu(), w, f"uncrop {name}", raw=True)
    _cmp(offo.cpu(), torch.tensor([off + count], dtype=torch.int32), "offset_out")
    _cmp(ovf.cpu(), torch.tensor([1 if off + count > cap else SENT], dtype=torch.int32), "overflow")


def test_crop_uncrop_batched():
    """Six crop runs of three clouds in one launch: each cloud's rows start at the prefix of its earlier runs' kept counts;
    one cloud fits, one reaches its capacity exactly and one overflows; rows past a cloud's capacity (which is below
    cloud_rows) stay untouched, and only lifted / overflow of each cloud are written besides the rows."""
    from psam_b200 import ops

    kernel = "crop_uncrop_kernel<true>"
    nv = _nv()
    assert nv.lib().psam_crop_run_bytes() == ops.CROP_RUN.itemsize
    B, N_max, cloud_rows = 3, 3000, 300
    Wg = -(-N_max // 32) + 1
    rng = np.random.default_rng(17)
    plan = [  # (cloud, n, count, K, crop, layer score, capacity)
        (0, 700, 30, 40, 0, 0.0, 250), (0, 400, 200, 210, 3, 1.0, 250),
        (1, 1000, 100, 110, 1, 0.0, 100),
        (2, 333, 120, 125, 2, 1.0, 200), (2, 97, 50, 60, 5, 2.0, 200), (2, 1500, 90, 100, 9, 2.0, 200),
    ]
    runs, keepalive = [], []
    table = np.zeros(len(plan), dtype=ops.CROP_RUN)
    for r, (c, n, count, K, crop, ls, capacity) in enumerate(plan):
        run = _uncrop_run(rng, n, N_max, 60, 4, K, count)
        dev = {k: Win(run[k], fill=SENT) for k in ("bits", "area", "keep")}
        dev.update(score=Win(run["score"]), stab=Win(run["stab"]), idx=Win(run["idx"], fill=N_max - 1), prompt=Win(run["prompt"], fill=0),
                   cnt=Win(torch.tensor([count], dtype=torch.int32), fill=SENT))
        keepalive.append(dev)
        first = next(i for i, p in enumerate(plan) if p[0] == c)
        last = r + 1 == len(plan) or plan[r + 1][0] != c
        table[r] = (dev["bits"].ptr, dev["area"].ptr, dev["score"].ptr, dev["stab"].ptr, dev["keep"].ptr, dev["cnt"].ptr, dev["idx"].ptr,
                    dev["prompt"].ptr, K, run["W"], n, 4, crop, c, first, int(last), ls, capacity)
        runs.append((run, c, crop, ls, capacity))
    tw = torch.from_numpy(table.view(np.uint8).copy()).to(_dev())
    outs = _out_windows((B, cloud_rows), Wg)
    lifted, ovf = Win(shape=(B,), dtype=torch.int32, fill=SENT), Win(shape=(B,), dtype=torch.int32, fill=SENT)
    K_max = max(p[3] for p in plan)
    rc = nv.lib().psam_crop_uncrop_batched(tw.data_ptr(), len(plan), K_max, B, N_max, Wg, cloud_rows, *[o.ptr for o in outs], lifted.ptr,
                                           ovf.ptr, nv.stream())
    assert rc == 0
    for name, w in list(zip(_OUT_NAMES, outs)) + [("lifted", lifted), ("overflow", ovf)]:
        w.check(name)
    for dev in keepalive:
        for name, w in dev.items():
            w.check(f"run {name}")
    want = [_sentinel(tuple(o.t.shape), o.t.dtype) for o in outs]
    base = [0] * B
    for run, c, crop, ls, capacity in runs:
        _want_uncrop_rows(run, N_max, Wg, crop, ls, base[c], min(capacity, cloud_rows), [w[c] for w in want])
        base[c] += run["count"]
    for o, w, name in zip(outs, want, _OUT_NAMES):
        _cmp(o.cpu(), w, f"batched uncrop {name}", raw=True)
    caps = [250, 100, 200]
    _cmp(lifted.cpu(), torch.tensor(base, dtype=torch.int32), "lifted")
    _cmp(ovf.cpu(), torch.tensor([int(t > cp) for t, cp in zip(base, caps)], dtype=torch.int32), "overflow")
    print(f"[amg] {kernel}: lifted {base} against capacities {caps}, grid {min(K_max, max(16, 2 * 264 // len(plan)))} x {len(plan)}")


# ------------------------------------------------------------------------------------------------
# the references and guards have teeth (host only: no kernel runs)
# ------------------------------------------------------------------------------------------------
def test_checks_have_teeth():
    """Each comparison rejects a wrong answer: an NMS keep list with two ranks swapped, a regions result that keeps one
    island of min_area - 1 points, and a candidates result with one slot written just past its cloud's block."""
    from oracle import amg_ref

    masks = _nms_masks(1, 300, 96, 5, groups=30)
    bits = torch.stack([_bits_i32(amg_ref.pack_bits(masks[0], 3))])
    area = torch.from_numpy(masks.sum(-1).astype(np.int32))
    score = torch.from_numpy(_nms_scores(1, 300, "random", 5))
    keep, cnt = _want_nms(bits, area, score, 0.7)
    assert int(cnt[0]) >= 2
    _cmp(keep, _want_nms(bits, area, score, 0.7)[0], "nms")
    swapped = keep.clone()
    swapped[0, 0], swapped[0, 1] = keep[0, 1], keep[0, 0]
    with pytest.raises(AssertionError, match="keep"):
        _cmp(swapped, keep, "nms keep")

    N, min_area = 64, 5
    m = np.zeros((1, N), dtype=bool)
    m[0, 0:20] = True
    m[0, 40:44] = True  # an island of min_area - 1 points: removed
    rb = _bits_i32(amg_ref.pack_bits(m, 3))[None]
    keep1 = torch.zeros(1, 1, dtype=torch.int32)
    nbr = torch.from_numpy(_graph("chain_up", N, 1, np.random.default_rng(0))[None])
    want = _want_regions(rb, keep1, [1], nbr, min_area)
    assert int(want[1][0, 0]) == 20 and float(want[2][0, 0]) == 0.0
    wrong = (rb[:, :1].clone(), torch.tensor([[24]], dtype=torch.int32), want[2].clone())  # the input mask, island kept
    with pytest.raises(AssertionError, match="bits_out"):
        _check_regions(wrong, want, "regions")

    B, Zc, C, base, Nc = 2, 2, 3, 1, 40
    W, stride = 2, base + Zc * C + 2
    lg, io = _logits(B * Zc, C, Nc, 3), _ious(B * Zc, C, 3)
    rules = _rules("plain", Nc)
    want = _want_cand(lg, io, B, W, base, stride, rules)
    got = [t.clone() for t in want]
    got[3][base + Zc * C] = 0.5  # one slot past cloud 0's block
    with pytest.raises(AssertionError, match="score"):
        _check_cand(got, want, "candidates")


# ------------------------------------------------------------------------------------------------
# routing guard
# ------------------------------------------------------------------------------------------------
def test_routing_guard():
    """One call per instantiation - mask_candidates_kernel<VEC, VARLEN> x4, the three NMS kernels, mask_regions_kernel
    <SMEM, VARLEN> x4, crop_edge_filter_kernel<BATCH> x2 and crop_uncrop_kernel<BATCH> x2 - under the profiler; the kernel
    that ran must be the one the case ids name, and the small-region grid the restated one.  It runs in a fresh
    interpreter, as the other routing guards do: what the profiler records must not depend on what ran before it."""
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    code = "import sys; sys.path[:0] = [%r, %r, %r]; import test_gpu_amg_kernels as t; t._routing_guard()" % (
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
    L, d = nv.lib(), _dev()
    calls, keep = [], []
    st = nv.stream()

    def z(*shape, dtype=torch.int32):
        t = torch.zeros(shape, dtype=dtype, device=d)
        keep.append(t)
        return t

    def cand_call(N, aligned, varlen):
        lg = z(4 * N + 4, dtype=torch.float32)
        p = lg.data_ptr() + (0 if aligned else 4)
        io, ln = z(4, dtype=torch.float32), torch.full((1,), N, dtype=torch.int32, device=d)
        bits, area, stab, score = z(4, 8), z(4), z(4, dtype=torch.float32), z(4, dtype=torch.float32)
        keep.append(ln)
        outs = (bits.data_ptr(), area.data_ptr(), stab.data_ptr(), score.data_ptr(), st)
        if varlen:
            return lambda: L.psam_mask_candidates_varlen_f32(p, io.data_ptr(), ln.data_ptr(), 1, 2, 2, N, 2, 0.0, 1.0, 0.0, 0.0, 0, 0, 4, 8,
                                                             *outs)
        return lambda: L.psam_mask_candidates_batched_f32(p, io.data_ptr(), 1, 2, 2, N, 0.0, 1.0, 0.0, 0.0, 0, 0, 4, 8, *outs)

    for varlen in (False, True):
        for N, aligned in ((128, True), (128, False)):
            calls.append((cand_kernel(N, aligned, varlen), None, cand_call(N, aligned, varlen)))

    K, W = 70, 2
    nbits, narea = z(K, W), z(K)
    nscore = torch.rand(K, device=d)
    nkeep, ncnt = z(K), z(1)
    nws = z(L.psam_mask_nms_workspace_bytes(K, W) // 4 + 4)
    keep.append(nscore)
    calls.append(("nms_order_kernel", None, lambda: L.psam_mask_nms(nbits.data_ptr(), narea.data_ptr(), nscore.data_ptr(), K, W, 0.5,
                                                                     nkeep.data_ptr(), ncnt.data_ptr(), nws.data_ptr(), st)))
    calls.append(("nms_pairs_kernel", None, None))
    calls.append(("nms_scan_kernel", None, None))

    def regions_call(N, varlen, B, K):
        Wn = -(-N // 32)
        bits, kp, cnt = z(B, K, Wn), z(B, K), torch.full((B,), K, dtype=torch.int32, device=d)
        nbr = torch.full((B, N, 1), -1, dtype=torch.int64, device=d)
        ln = torch.full((B,), N, dtype=torch.int32, device=d)
        bo, ao, so = z(B, K, Wn), z(B, K), z(B, K, dtype=torch.float32)
        ws = z(L.psam_mask_regions_batched_workspace_bytes(B, K, N) // 4 + 4)
        keep.extend([cnt, nbr, ln])
        args = (kp.data_ptr(), cnt.data_ptr(), nbr.data_ptr(), 1, 1, bo.data_ptr(), ao.data_ptr(), so.data_ptr(), ws.data_ptr(), st)
        if varlen:
            return lambda: L.psam_mask_regions_varlen(bits.data_ptr(), K, ln.data_ptr(), B, K, Wn, N, *args)
        return lambda: L.psam_mask_regions_batched(bits.data_ptr(), K, B, K, Wn, N, *args)

    for varlen in (False, True):
        for N, B, K in ((1000, 3, 100), (60000, 2, 3)):
            calls.append((region_kernel(N, varlen), (B * K, N), regions_call(N, varlen, B, K)))

    eb, ee, es = z(2, 9, 3), z(2, 3), z(2, 9, dtype=torch.float32)
    calls.append(("crop_edge_filter_kernel<false>", None, lambda: L.psam_crop_edge_filter(eb.data_ptr(), 9, 3, ee.data_ptr(), es.data_ptr(), st)))
    calls.append(("crop_edge_filter_kernel<true>", None,
                  lambda: L.psam_crop_edge_filter_batched(eb.data_ptr(), 2, 9, 3, ee.data_ptr(), es.data_ptr(), st)))

    ub, ua, us, ut = z(4, 1), z(4), z(4, dtype=torch.float32), z(4, dtype=torch.float32)
    uk, uc, ui, up = z(2), torch.full((1,), 2, dtype=torch.int32, device=d), z(8), z(2, dtype=torch.int64)
    uoff, uoo, uovf = z(1), z(1), z(1)
    gouts = [z(16, 2), z(16), z(16, dtype=torch.float32), z(16, dtype=torch.float32), z(16, dtype=torch.int64), z(16), z(16),
             z(16, dtype=torch.float32)]
    keep.append(uc)
    calls.append(("crop_uncrop_kernel<false>", None,
                  lambda: L.psam_crop_uncrop(ub.data_ptr(), ua.data_ptr(), us.data_ptr(), ut.data_ptr(), 2, 1, uk.data_ptr(), uc.data_ptr(),
                                             ui.data_ptr(), 8, up.data_ptr(), 2, 0, 0.0, 40, 2, 16, uoff.data_ptr(), uoo.data_ptr(),
                                             *[o.data_ptr() for o in gouts], uovf.data_ptr(), st)))
    from psam_b200 import ops

    table = np.zeros(1, dtype=ops.CROP_RUN)
    table[0] = (ub.data_ptr(), ua.data_ptr(), us.data_ptr(), ut.data_ptr(), uk.data_ptr(), uc.data_ptr(), ui.data_ptr(), up.data_ptr(),
                2, 1, 8, 2, 0, 0, 0, 1, 0.0, 16)
    tw = torch.from_numpy(table.view(np.uint8).copy()).to(d)
    bouts = [z(1, 16, 2), z(1, 16), z(1, 16, dtype=torch.float32), z(1, 16, dtype=torch.float32), z(1, 16, dtype=torch.int64), z(1, 16),
             z(1, 16), z(1, 16, dtype=torch.float32)]
    lifted, bovf = z(1), z(1)
    keep.append(tw)
    calls.append(("crop_uncrop_kernel<true>", None,
                  lambda: L.psam_crop_uncrop_batched(tw.data_ptr(), 1, 2, 1, 40, 2, 16, *[o.data_ptr() for o in bouts], lifted.data_ptr(),
                                                     bovf.data_ptr(), st)))

    torch.cuda.synchronize()
    rcs = []
    fns = [fn for _, _, fn in calls if fn is not None]
    got = _kernels_launched(lambda: rcs.extend(fn() for fn in fns))
    assert rcs == [0] * len(fns), f"return codes {rcs}"
    assert len(got) == len(calls), f"{len(calls)} kernels expected, {len(got)} launched: {[n for n, _ in got]}"
    sms = _sms()
    for (want, what, _), (name, grid) in zip(calls, got):
        assert want in name, f"expected {want}, ran {name}"
        if what is not None and grid is not None:
            items, N = what
            assert grid[0] == region_grid(items, N, sms), f"{want} N={N}: grid {grid}, restated {region_grid(items, N, sms)}"
            print(f"[amg] {want} N={N}: {items} items on grid {grid[0]}")
    print(f"[amg] routing guard: {len(calls)} kernels, each the one its case id names"
          f"{'' if got[0][1] is not None else ' (the trace has no grids)'}")
