"""The paths bench.py times, in the configuration it runs them, against the fp64 oracle.

c2 is PipelinedPredictor at depth 8 with CUDA graphs and host result slots (enable_host_results(3)) on a perturbed ViT-L at
N = 32768, G = 512, K = 64.  It is the only caller where the LayerNorm-free ViT blocks (BLOCK_LN_POLICY "auto" resolved by
the predictor's block_ln_fold scope) and the throughput tile policy (ops.GEMM_TILE_HINT = 1, which the LayerNorm kernel's
policy field reads too) are baked into captured graphs.  c3 is the evaluation loop: 4 lanes of make_iterative_predictor with
throughput tiles, chunks of clouds round-robin over the lanes, 3 GT-driven prompt iterations.

The benchmark itself cannot see a lane that ignores its new inputs or returns another ticket's result: it rotates 4 inputs
over 8 lanes, so lane i always holds cloud i mod 4.  Here 9 clouds (coprime with the 8 lanes) rotate instead: ticket t takes
cloud t mod 9, so every lane gets a cloud it has not held on every round and no two lanes share one within a round.  The
weights are perturbed like a trained checkpoint's (oracle/params_ref.py): with gamma = 1 and beta = 0 a fold that lost its
gamma or beta term would still give the right answer.

Bounds: masks and IoU 1e-3 abs + 1e-2 rel (the north-star bound, pr.ratio <= 1).  Lanes are never compared with each other
or with eager runs bit for bit: the encoder's split-K GEMMs add partial sums with float atomics.

The last part pins psam_posenc_f32, the kernel that raises the serving tickets' ValueError, through the C ABI.  It
establishes that the range flag is set exactly when the reference's fp32 predicate (c < -1 - 1e-6) | (c > 1 + 1e-6) holds:
fp32(1 + 1e-6) itself passes and the next float flags, +-inf flag and NaN does not (as in the reference, whose comparisons
are false for NaN).  Labels other than 0 and 1 add no embedding, a NULL flag pointer writes nothing, and the kernel never
clears the flag word."""
import math
import time
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import params_ref as pr  # noqa: E402
from oracle import torch_ref  # noqa: E402

ENC, N, G, K = "eva02_large_patch14_448", 32768, 512, 64
DEPTH, HOST_C = 8, 3   # bench.py: make_pipelined_predictor(..., depth=8), enable_host_results(3)
CLOUDS = 9             # coprime with DEPTH
C3_TOTAL, C3_LANES, C3_CHUNK, C3_ITERS = 32, 4, 4, 3

# the engine switches as bench.py runs them (no PSAM_* variable set)
SWITCHES = dict(FUSED_ATTENTION=True, FUSED_ATTENTION_LONG=True, ATTENTION_TWOPASS=False, FUSED_ATTENTION_DH88=True,
                FUSED_INNER_LN=True, FUSED_BLOCK_LN=True, BLOCK_LN_POLICY="auto", FUSED_ROW_LN=True, DECODER_TC=True,
                FUSED_MASK_DOT=True)
OPS = dict(GEMM_TILE_HINT=0, GEMM_TILE_BN=0, GEMM_VARIANT=0)


def _dev():
    return torch.device("cuda:0")


class _Worst:
    """Largest err/bound of the masks and the IoU seen by one arm."""

    def __init__(self, name):
        self.name, self.masks, self.iou, self.n = name, 0.0, 0.0, 0

    def check(self, what, got_m, got_i, want_m, want_i):
        rm, ri = pr.ratio(got_m, want_m, "masks"), pr.ratio(got_i, want_i, "iou")
        self.masks, self.iou, self.n = max(self.masks, rm), max(self.iou, ri), self.n + 1
        assert rm <= 1.0 and ri <= 1.0, f"{self.name}: {what}: err/bound masks {rm:.3f}, iou {ri:.3f}"

    def report(self):
        print(f"[serving] {self.name}: {self.n} results, worst err/bound masks {self.masks:.3f} iou {self.iou:.3f}")


class _Spy:
    """Per pass of a predictor's _run: every GEMM (its tile hint as gemm_raw resolved it, and whether a LayerNorm over the
    ViT width is folded into it) and every LayerNorm launch (rows, width, and the tile policy its kernel reads)."""

    def __init__(self, mp, predictor_cls=None):
        from psam_b200 import ops

        self.passes = [dict(owner=None, gemm=[], ln=[])]
        gemm_raw, layernorm = ops.gemm_raw, ops.layernorm
        spy = self

        def gemm(a, w, out, *args, **kw):
            gemm_raw(a, w, out, *args, **kw)
            spy.passes[-1]["gemm"].append((out.tile_hint, bool(out.ln_stats) and out.ln_h == 1024))

        def ln(x, *args, **kw):
            D = kw.get("D") or x.shape[-1]
            rows = kw.get("rows") or x.numel() // x.shape[-1]
            spy.passes[-1]["ln"].append((rows, D, ops.GEMM_TILE_HINT))
            return layernorm(x, *args, **kw)

        mp.setattr(ops, "gemm_raw", gemm)
        mp.setattr(ops, "layernorm", ln)
        if predictor_cls is not None:
            run = predictor_cls._run

            def run_pass(self_, *a, **k):
                spy.begin(self_)
                return run(self_, *a, **k)

            mp.setattr(predictor_cls, "_run", run_pass)

    def begin(self, owner):
        self.passes.append(dict(owner=owner, gemm=[], ln=[]))

    def runs(self):
        return [p for p in self.passes if p["owner"] is not None]


def _summary(p, rows):
    """(GEMMs, block GEMMs with a folded LayerNorm, block LayerNorm launches of `rows` x 1024, LayerNorm launches),
    the set of GEMM tile hints, the set of LayerNorm policies."""
    fold = sum(f for _, f in p["gemm"])
    block_ln = sum((r, d) == (rows, 1024) for r, d, _ in p["ln"])
    return (len(p["gemm"]), fold, block_ln, len(p["ln"])), {h for h, _ in p["gemm"]}, {pol for *_, pol in p["ln"]}


# ------------------------------------------------------------------------------------------------
# model, c2 reference
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def served():
    """The perturbed ViT-L (CUDA model and the fp64 oracle on the GPU) and the oracle's outputs for CLOUDS clouds of one
    1-point prompt set each, computed before any predictor exists.  The engine switches, the tile switches and
    PSAM_THROUGHPUT_TILES stay at bench.py's defaults for the whole module."""
    from pc_sam.model import build_point_sam
    from pc_sam.model.pc_encoder import PatchEmbed
    from pc_sam.model.transformer import TwoWayTransformer
    from psam_b200 import engine, ops

    with pytest.MonkeyPatch.context() as mp:
        for k, v in SWITCHES.items():
            mp.setattr(engine, k, v)
        for k, v in OPS.items():
            mp.setattr(ops, k, v)
        mp.setenv("PSAM_THROUGHPUT_TILES", "1")
        mp.delenv("PSAM_PROFILE_STAGE", raising=False)
        s = pr.spec(enc=ENC, G=G, K=K, N=N, seed=151, eps=1e-6)
        oracle = pr.build_oracle(s)
        model = build_point_sam(ENC, G, K)
        pr.restructure(model, s, types.SimpleNamespace(TwoWayTransformer=TwoWayTransformer, PatchEmbed=PatchEmbed))
        pr.copy_to(oracle, model)  # before the CUDA model's first call
        model = model.cuda().eval()
        x, f, c, l = pr.inputs(s, B=CLOUDS, M=1, P=1)
        t0 = time.perf_counter()
        want = pr.reference(oracle.cuda(), x, f, c, l)
        torch.cuda.synchronize()
        secs = time.perf_counter() - t0
        print(f"\n[serving] fp64 c2 reference, {CLOUDS} clouds: {secs:.1f} s")
        clouds = [(x[i:i + 1], f[i:i + 1], c[i:i + 1], l[i:i + 1]) for i in range(CLOUDS)]
        yield types.SimpleNamespace(
            model=model, oracle=oracle, ref_secs=secs, host=clouds,
            pinned=[tuple(t.pin_memory() for t in cl) for cl in clouds],
            dev=[tuple(t.to(_dev()) for t in cl) for cl in clouds],
            want_m=want["masks"].cpu(), want_i=want["iou"].cpu())


@pytest.fixture(scope="module")
def c2(served):
    """PipelinedPredictor(depth=8) as bench.py builds it: warmup on cloud 0 (with the spy), then enable_host_results(3)."""
    from psam_b200.predictor import GraphPredictor

    pp = served.model.make_pipelined_predictor(1, N, 1, depth=DEPTH)
    assert pp.throughput_tiles and pp.ln_fold
    with pytest.MonkeyPatch.context() as mp:
        spy = _Spy(mp, GraphPredictor)
        pp.warmup(*served.dev[0])
    pp.enable_host_results(HOST_C)
    assert pp.slots == 2 * DEPTH
    held = {i: {0} for i in range(DEPTH)}  # clouds each lane's buffers have held
    return types.SimpleNamespace(pp=pp, spy=spy, held=held)


def _submit(c2, cloud, inputs, to_host=False):
    t = c2.pp.submit(*inputs, to_host=to_host)
    c2.held[t % DEPTH].add(cloud)
    return t


def test_c2_capture_routing(served, c2, monkeypatch):
    """Every pass of every lane's warmup (two eager passes and the capture) runs each GEMM with tile hint 1 and each
    LayerNorm with policy 1, and has 2 x 24 + 1 block GEMMs with a folded LayerNorm and no block LayerNorm (the
    block_folded form of test_gpu_model_params.py at depth 24).  Afterwards the switch is 0 again and an eager call takes
    the LayerNorm form."""
    from psam_b200 import ops

    depth = len(served.model.pc_encoder.transformer.blocks)
    runs = c2.spy.runs()
    assert len(runs) == 3 * DEPTH, f"{len(runs)} passes for {DEPTH} lanes"
    assert [sum(p["owner"] is ln for p in runs) for ln in c2.pp.lanes] == [3] * DEPTH
    counts = set()
    for i, p in enumerate(runs):
        n, hints, policies = _summary(p, G)
        assert hints == {1}, f"pass {i}: GEMM tile hints {hints}"
        assert policies == {1}, f"pass {i}: LayerNorm policies {policies}"
        assert n[1] == 2 * depth + 1 and n[2] == 0, f"pass {i}: {n[1]} folded block GEMMs, {n[2]} block LayerNorms"
        counts.add(n)
    assert len(counts) == 1, f"the lanes' passes differ: {counts}"
    print(f"[serving] c2 capture: {len(runs)} passes, each (GEMMs, folded, block LN, LN) = {counts.pop()}")

    assert ops.GEMM_TILE_HINT == 0
    spy = _Spy(monkeypatch)
    spy.begin("eager")
    with torch.no_grad():
        served.model.predict_masks(*served.dev[1], None, True)
    n, hints, policies = _summary(spy.passes[-1], G)
    assert hints == {0} and policies == {0}, (hints, policies)
    assert n[1] == 0 and n[2] == 2 * depth + 1, f"eager: {n[1]} folded block GEMMs, {n[2]} block LayerNorms"


def test_c2_device_arm(served, c2, tmp_path):
    """Tickets with device inputs, cloud t mod 9: each result is read back before its lane takes the next ticket, and
    bench.dump_outputs writes exactly the last 8 tickets' results."""
    import bench

    pp, worst = c2.pp, _Worst("c2 device arm")
    t0, got = pp.count, {}
    for t in range(t0, t0 + 4 * DEPTH):
        if t - DEPTH >= t0:
            m, i = pp.result(t - DEPTH)
            got[t - DEPTH] = (m.cpu(), i.cpu())  # synchronous copies, before ticket t overwrites the lane
        _submit(c2, t % CLOUDS, served.dev[t % CLOUDS])
    for t in range(pp.count - DEPTH, pp.count):
        m, i = pp.result(t)
        got[t] = (m.cpu(), i.cpu())
    for t, (m, i) in sorted(got.items()):
        worst.check(f"ticket {t} (cloud {t % CLOUDS})", m, i, served.want_m[t % CLOUDS:t % CLOUDS + 1],
                    served.want_i[t % CLOUDS:t % CLOUDS + 1])
    worst.report()
    info = bench.dump_outputs(pp, 2 * DEPTH, str(tmp_path))
    assert info["tickets"] == [pp.count - DEPTH, pp.count]
    dm, di = np.load(tmp_path / "masks.npy"), np.load(tmp_path / "iou.npy")
    assert dm.shape == (DEPTH, 1, 3, N) and di.shape == (DEPTH, 1, 3)
    for j, t in enumerate(range(pp.count - DEPTH, pp.count)):
        assert np.array_equal(dm[j], got[t][0].numpy()) and np.array_equal(di[j], got[t][1].numpy()), f"dumped ticket {t}"


def test_c2_single_stream_arm(served, c2):
    """bench.py's latency arm calls lane 0 directly; the pipelined tickets that follow must still be right."""
    pp, worst = c2.pp, _Worst("c2 single-stream arm")
    lane = pp.lanes[0]
    cloud = min(set(range(CLOUDS)) - c2.held[0])
    m, i = lane(*served.dev[cloud])
    lane.check()
    c2.held[0].add(cloud)
    worst.check(f"lane 0 called directly (cloud {cloud})", m.cpu(), i.cpu(), served.want_m[cloud:cloud + 1],
                served.want_i[cloud:cloud + 1])
    t0 = pp.count
    for t in range(t0, t0 + 2 * DEPTH):
        if t - DEPTH >= t0:
            m, i = pp.result(t - DEPTH)
            worst.check(f"ticket {t - DEPTH}", m.cpu(), i.cpu(), served.want_m[(t - DEPTH) % CLOUDS][None],
                        served.want_i[(t - DEPTH) % CLOUDS][None])
        _submit(c2, t % CLOUDS, served.dev[t % CLOUDS])
    for t in range(pp.count - DEPTH, pp.count):
        m, i = pp.result(t)
        worst.check(f"ticket {t}", m.cpu(), i.cpu(), served.want_m[t % CLOUDS][None], served.want_i[t % CLOUDS][None])
    worst.report()


def test_c2_end_to_end_arm(served, c2):
    """Pinned host inputs and host results, in bench.py's loop: before ticket t is submitted the host reads ticket
    t - slots, whose host slot t reuses.  One ticket's cloud is x3 and another's prompt alone is out of range: exactly
    those two raise ValueError, and the tickets that reuse their lane (+8) and their host slot (+16) are right."""
    pp, worst = c2.pp, _Worst("c2 end-to-end arm")
    slots = pp.slots
    t0 = pp.count
    x, f, c, l = served.host[4]
    bad = {t0 + 3: tuple(t.pin_memory() for t in (x * 3, f, c * 3, l)),
           t0 + 13: tuple(t.pin_memory() for t in (x, f, c + 5, l))}
    assert bool((bad[t0 + 3][0].abs() > 1.5).any()) and bool((bad[t0 + 13][2] > 1.5).all())
    checked, raised = set(), set()

    def read(t):
        if t in bad:
            with pytest.raises(ValueError):
                pp.result(t, to_host=True)
            raised.add(t)
            return
        m, i = pp.result(t, to_host=True)
        worst.check(f"ticket {t} (cloud {t % CLOUDS}, slot {t % slots})", m, i, served.want_m[t % CLOUDS][None],
                    served.want_i[t % CLOUDS][None])
        checked.add(t)

    end = t0 + 2 * slots + 8
    for t in range(t0, end):
        if t - slots >= t0:
            read(t - slots)
        assert pp.count == t
        if t in bad:
            pp.submit(*bad[t], to_host=True)
        else:
            _submit(c2, t % CLOUDS, served.pinned[t % CLOUDS], to_host=True)
    for t in range(end - slots, end):
        read(t)
    worst.report()
    assert raised == set(bad)
    for tb in bad:
        assert {tb + DEPTH, tb + slots} <= checked
    assert len(checked) + len(raised) == end - t0


# ------------------------------------------------------------------------------------------------
# c3: the evaluation-loop lanes, built while the c2 predictor is alive (as bench.py does)
# ------------------------------------------------------------------------------------------------
def test_c3_evaluation_lanes(served, c2, monkeypatch):
    """4 lanes of make_iterative_predictor(chunk, 1, N, throughput_tiles=True), chunks round-robin with check=False and the
    IoU rows written on the lane streams (bench.py's one_step).  Each iteration's new prompt is the reference sampler's
    choice from the lane's own previous prompt mask (iteration 0: from the ground truth), bit for bit; the masks and IoU
    of every iteration are within the bound of the fp64 oracle replaying those prompts; the captures use tile hint 1 and
    the LayerNorm form of the blocks; no lane raises."""
    from pc_sam.model.loss import compute_iou
    from psam_b200 import synth
    from psam_b200.parallel import plan_graph_chunks
    from psam_b200.predictor import IterativeGraphPredictor

    model = served.model
    chunk, n_chunks = plan_graph_chunks(C3_TOTAL, C3_LANES, C3_CHUNK)
    print(f"\n[serving] c3: {n_chunks} chunks of {chunk} clouds over {C3_LANES} lanes, {C3_ITERS} iterations")
    monkeypatch.setattr(model, "prompt_iters", C3_ITERS)
    host = []
    for ci in range(n_chunks):
        made = [synth.make_batch(1, N, 5000 + ci * chunk + b, "ball") for b in range(chunk)]
        xyz, feats = torch.cat([m[0] for m in made]), torch.cat([m[1] for m in made])
        host.append((xyz, feats, synth.make_region_masks(xyz, 1)))
    devin = [tuple(t.to(_dev()) for t in h) for h in host]
    with pytest.MonkeyPatch.context() as mp:
        spy = _Spy(mp, IterativeGraphPredictor)
        lanes = [model.make_iterative_predictor(chunk, 1, N, throughput_tiles=True) for _ in range(C3_LANES)]
        for ln in lanes:
            ln.warmup(*devin[0])
    depth = len(model.pc_encoder.transformer.blocks)
    runs = spy.runs()
    assert len(runs) == 3 * C3_LANES
    for i, p in enumerate(runs):
        n, hints, policies = _summary(p, chunk * G)
        assert hints == {1} and policies == {1}, f"c3 pass {i}: tile hints {hints}, LayerNorm policies {policies}"
        assert n[1] == 0 and n[2] == 2 * depth + 1, f"c3 pass {i}: {n[1]} folded block GEMMs, {n[2]} block LayerNorms"

    keys = ("prompt_coords", "prompt_labels", "masks", "iou_preds", "prompt_masks")
    main = torch.cuda.current_stream()
    rows = torch.zeros((n_chunks * chunk, C3_ITERS), dtype=torch.float32, device=_dev())
    start = torch.cuda.Event()
    start.record(main)
    saved = []
    for ln in lanes:
        ln.stream.wait_event(start)
    for ci in range(n_chunks):
        ln = lanes[ci % len(lanes)]
        outs = ln(*devin[ci], check=False)
        with torch.no_grad(), torch.cuda.stream(ln.stream):
            gtf = ln.gt.flatten(0, 1)
            for t, o in enumerate(outs):
                rows[ci * chunk:(ci + 1) * chunk, t] = compute_iou(o["prompt_masks"], gtf).view(chunk, 1).mean(dim=1)
            saved.append([{k: o[k].clone() for k in keys} for o in outs])  # before the lane's next chunk
    for ln in lanes:
        ln.check()
    torch.cuda.synchronize()
    saved = [[{k: v.cpu() for k, v in o.items()} for o in outs] for outs in saved]

    t_sampler = t_ref = 0.0
    worst = [[0.0, 0.0] for _ in range(C3_ITERS)]
    oracle = served.oracle
    for ci, ((xyz, feats, gt), outs) in enumerate(zip(host, saved)):
        assert len(outs) == C3_ITERS
        for t, o in enumerate(outs):
            want_rows = compute_iou(o["prompt_masks"], gt.flatten(0, 1)).view(chunk, 1).mean(dim=1)
            assert torch.equal(rows[ci * chunk:(ci + 1) * chunk, t].cpu(), want_rows), f"chunk {ci} iteration {t}: IoU rows"
        s0 = time.perf_counter()
        for t in range(C3_ITERS):
            c, l = torch_ref.sample_prompts_eval(xyz, gt, outs[t - 1]["prompt_masks"] if t else None)
            got_c, got_l = outs[t]["prompt_coords"][:, t:t + 1], outs[t]["prompt_labels"][:, t:t + 1]
            assert torch.equal(c, got_c) and torch.equal(l, got_l.bool()), f"chunk {ci} iteration {t}: sampled prompt"
        s1 = time.perf_counter()
        pcs = [outs[t]["prompt_coords"][:, t:t + 1].to(_dev(), torch.float64) for t in range(C3_ITERS)]
        pls = [outs[t]["prompt_labels"][:, t:t + 1].to(_dev()) for t in range(C3_ITERS)]
        with torch.no_grad(), pr.fp32_neighbours():
            want = oracle.predict_iterative(xyz.to(_dev(), torch.float64), feats.to(_dev(), torch.float64), pcs, pls)
        torch.cuda.synchronize()
        t_sampler, t_ref = t_sampler + s1 - s0, t_ref + time.perf_counter() - s1
        for t in range(C3_ITERS):
            rm = pr.ratio(outs[t]["masks"], want[t]["masks"].cpu(), "masks")
            ri = pr.ratio(outs[t]["iou_preds"], want[t]["iou_preds"].cpu(), "iou")
            worst[t] = [max(worst[t][0], rm), max(worst[t][1], ri)]
            assert rm <= 1.0 and ri <= 1.0, f"chunk {ci} iteration {t}: err/bound masks {rm:.3f}, iou {ri:.3f}"
    del oracle
    served.oracle = None
    torch.cuda.empty_cache()
    print(f"[serving] c3: reference sampler {t_sampler:.1f} s, fp64 oracle replay {t_ref:.1f} s (c2 reference "
          f"{served.ref_secs:.1f} s)")
    for t, (wm, wi) in enumerate(worst):
        print(f"[serving] c3 iteration {t}: worst err/bound masks {wm:.3f} iou {wi:.3f}")


# ------------------------------------------------------------------------------------------------
# psam_posenc_f32 through the C ABI
# ------------------------------------------------------------------------------------------------
U = 2.0 ** -24
PAD = 37            # sentinel floats on each side of the output window
SENTINEL = -777.25
FLAG_LO = torch.tensor(-1 - 1e-6, dtype=torch.float32)
FLAG_HI = torch.tensor(1 + 1e-6, dtype=torch.float32)


def _posenc(coords, gauss, labels, emb0, emb1, flag):
    """Launch into the middle of a sentinel-filled buffer; returns (whole buffer, return code)."""
    from psam_b200 import native as nv

    rows, F = coords.shape[0], gauss.shape[1]
    buf = torch.full((2 * PAD + rows * 2 * F,), SENTINEL, dtype=torch.float32, device=_dev())
    rc = nv.lib().psam_posenc_f32(nv.ptr(coords), rows, nv.ptr(gauss), F, nv.ptr(labels), nv.ptr(emb0), nv.ptr(emb1),
                                  buf.data_ptr() + 4 * PAD, nv.ptr(flag), nv.stream())
    torch.cuda.synchronize()
    return buf, rc


def _posenc64(coords, gauss, labels, emb0, emb1):
    """fp64 restatement: [sin(2 pi c @ G), cos(2 pi c @ G)] per row, plus emb0 / emb1 for labels 0 / 1 only; and the
    error bound of the kernel's fp32 arithmetic.  The kernel forms s = fma(z, g2, fma(y, g1, x g0)): three roundings, each
    at most u times a partial sum bounded by S = |x g0| + |y g1| + |z g2|, so |s - c @ G| <= 3 u S (1 + 2u).  Multiplying by
    fp32(2 pi) (relative error 0.47 u) and rounding adds 2 u S (2 pi) more: the argument is within 2 pi 5.01 u S of the
    exact one, and sin / cos have slope at most 1.  sincosf (no fast math) is within 2 ulp of its fp32 argument's sine:
    2^-23 for results below 1 in magnitude.  Adding the embedding rounds once more, u |out|."""
    c, g = coords.double(), gauss.double()
    terms = c[:, :, None] * g[None]
    s = 2 * math.pi * terms.sum(1)
    out = torch.cat([torch.sin(s), torch.cos(s)], -1)
    if labels is not None:
        out = out + (labels == 0)[:, None].double() * emb0.double()[None] + (labels == 1)[:, None].double() * emb1.double()[None]
    S = terms.abs().sum(1)
    arg = 2 * math.pi * 5.01 * U * S
    bound = torch.cat([arg, arg], -1) + 2.0 ** -23 + U * out.abs()
    return out, bound


def _check_window(name, buf, want, bound):
    pads = torch.cat([buf[:PAD], buf[-PAD:]])
    assert bool((pads == SENTINEL).all()), f"{name}: written outside the output window"
    got = buf[PAD:-PAD].view(want.shape).double()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{name}: NaN positions differ"
    ratio = float(((got - want).abs() / bound)[~nan].max()) if bool((~nan).any()) else 0.0
    print(f"[serving] posenc {name}: worst err/bound {ratio:.3f}")
    assert ratio <= 1.0, f"{name}: error {ratio:.2f}x its bound"


def _inputs(rows, F, seed):
    g = torch.Generator().manual_seed(seed)
    coords = torch.rand((rows, 3), generator=g) * 2 - 1
    coords[0, 0] = 1.0
    if rows > 1:
        coords[1, 2] = -1.0
    gauss = torch.randn((3, F), generator=g)
    emb0, emb1 = torch.randn(2 * F, generator=g), torch.randn(2 * F, generator=g)
    return [t.to(_dev()) for t in (coords, gauss, emb0, emb1)]


@pytest.mark.parametrize("labels", ["null", "mixed"])
@pytest.mark.parametrize("rows", [1, G, 70001], ids=["rows1", "rowsG", "rows70001"])
@pytest.mark.parametrize("F", [1, 31, 128, 129, 256])
def test_posenc_values(F, rows, labels):
    """F beyond the 128-thread block loops; more than 65535 rows; labels 2, 0, 1, -1 in rotation (a single row gets 2),
    where only 0 and 1 add an embedding.  In-range coordinates: the flag word stays 0."""
    coords, gauss, emb0, emb1 = _inputs(rows, F, 1000 * F + rows)
    lab = None
    if labels == "mixed":
        lab = torch.tensor([2, 0, 1, -1], dtype=torch.int32).repeat(rows // 4 + 1)[:rows].contiguous().to(_dev())
    flag = torch.zeros(3, dtype=torch.int32, device=_dev())
    flag[0], flag[2] = -5, -5
    buf, rc = _posenc(coords, gauss, lab, emb0 if lab is not None else None, emb1 if lab is not None else None, flag[1:])
    assert rc == 0
    want, bound = _posenc64(coords, gauss, lab, emb0, emb1)
    _check_window(f"F {F} rows {rows} labels {labels}", buf, want, bound)
    assert flag.tolist() == [-5, 0, -5]


_NEXT_UP = float(torch.nextafter(FLAG_HI, torch.tensor(math.inf)))
_NEXT_DOWN = float(torch.nextafter(FLAG_LO, torch.tensor(-math.inf)))
FLAG_CASES = [
    ("at_plus_bound", float(FLAG_HI), False),
    ("ulp_above_plus_bound", _NEXT_UP, True),
    ("at_minus_bound", float(FLAG_LO), False),
    ("ulp_below_minus_bound", _NEXT_DOWN, True),
    ("plus_one", 1.0, False),
    ("minus_one", -1.0, False),
    ("plus_inf", math.inf, True),
    ("minus_inf", -math.inf, True),
    ("nan", math.nan, False),
]


@pytest.mark.parametrize("axis", [0, 1, 2], ids=["x", "y", "z"])
@pytest.mark.parametrize("name,value,flagged", FLAG_CASES, ids=[c[0] for c in FLAG_CASES])
def test_posenc_range_flag(name, value, flagged, axis):
    """One coordinate of one row of 8 set to `value`: the flag is set exactly when the reference's predicate, evaluated on
    the fp32 coordinates, holds.  A flag word that is already set stays set, and a NULL flag pointer writes nothing."""
    F, rows = 128, 8
    coords, gauss, emb0, emb1 = _inputs(rows, F, 7 + axis)
    coords[5, axis] = value
    c32 = coords.cpu()
    predicate = bool((c32 < -1 - 1e-6).any() or (c32 > 1 + 1e-6).any())
    assert predicate == flagged, f"{name}: the reference predicate gives {predicate}"
    lab = torch.tensor([0, 1, 2, -1, 0, 1, 0, 1], dtype=torch.int32, device=_dev())
    want, bound = _posenc64(coords, gauss, lab, emb0, emb1)
    for start in (0, 7):
        flag = torch.tensor([-5, start, -5], dtype=torch.int32, device=_dev())
        buf, rc = _posenc(coords, gauss, lab, emb0, emb1, flag[1:])
        assert rc == 0
        _check_window(f"{name} axis {axis}", buf, want, bound)
        assert flag.tolist() == [-5, 1 if predicate else start, -5], f"{name}: flag word {flag.tolist()[1]} from {start}"
    buf, rc = _posenc(coords, gauss, lab, emb0, emb1, None)
    assert rc == 0
    _check_window(f"{name} axis {axis}, NULL flag", buf, want, bound)
