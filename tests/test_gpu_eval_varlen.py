"""GPU tests of the evaluation loop on clouds of different sizes: psam_border_prompt_varlen_f32 equals the single-cloud
sampler on every cut cloud bit for bit whatever the padding holds; forward_varlen matches the reference sampler and the
fp32 oracles per cloud and is forward for one cloud; the varlen graph predictor serves batches of other sizes than it was
captured with; the evaluation driver reproduces the per-crop rows; and ViT-L runs once at full size."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hier_ref, synth, torch_ref  # noqa: E402

DEV = torch.device("cuda:0")
ATOL, RTOL = 1e-3, 1e-2  # test_gpu_model.py's
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------
# 1. the sampler kernel
# ------------------------------------------------------------------------------------------------
SIZES = [1, 255, 256, 257, 511, 513, 2047, 2049, 5000]  # compaction (256), foreground (512) and chunk (2048) boundaries


def _sampler_batch(sizes, M, seed, gt_rule=None):
    """Padded coords [B, N_max, 3], gt [B, M, N_max], logits [B*M, N_max] and lengths, with padding built to win if read:
    even padded rows are far points (distance ~100) with gt 1 and logit +1e9 (the farthest foreground), odd ones are
    copies of the cloud's foreground nudged by 1e-6 with gt 0 and logit -1e9 (the nearest background)."""
    rng = np.random.default_rng(seed)
    B, n_max = len(sizes), max(sizes)
    xyz = np.zeros((B, n_max, 3), np.float32)
    gt = np.zeros((B, M, n_max), bool)
    lg = np.zeros((B, M, n_max), np.float32)
    for b, n in enumerate(sizes):
        x = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
        xyz[b, :n] = x
        for m in range(M):
            c = x[rng.integers(0, n)]
            g = ((x - c) ** 2).sum(1) < rng.uniform(0.2, 0.8) ** 2
            if gt_rule is not None:
                g = gt_rule(b, m, n, g)
            gt[b, m, :n] = g
            v = rng.normal(0, 1, n).astype(np.float32) + np.where(g, 0.5, -0.5).astype(np.float32)
            k = rng.random(n)
            v[k < 0.05] = 0.0
            v[(k >= 0.05) & (k < 0.1)] = -0.0
            lg[b, m, :n] = v
            fg = np.nonzero(g)[0]
            for j in range(n, n_max):
                if (j - n) % 2 == 0 or not len(fg):
                    xyz[b, j] = (100.0 + 1e-3 * (j - n), 50.0, -75.0)
                    gt[b, m, j], lg[b, m, j] = True, 1e9
                else:
                    xyz[b, j] = x[fg[(j - n) % len(fg)]] + np.float32(1e-6)
                    gt[b, m, j], lg[b, m, j] = False, -1e9
    lengths = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    return (torch.from_numpy(xyz).to(DEV), torch.from_numpy(gt).to(DEV), torch.from_numpy(lg).reshape(B * M, n_max).to(DEV),
            lengths)


def _compare_sampler(sizes, M, seed, gt_rule=None):
    from psam_b200 import ops

    xyz, gt, lg, lengths = _sampler_batch(sizes, M, seed, gt_rule)
    n_max = xyz.shape[1]
    statuses = {}
    for form in ("none", "logits", "masks"):
        for err in (True, False):
            if form == "none" and not err:
                continue  # the first iteration samples from the error region (adapter: pred_logits is None)
            kw = dict(pred_logits=lg if form == "logits" else None, pred_masks=(lg > 0) if form == "masks" else None)
            bx, bl, bs = ops.border_prompt(xyz, gt, from_error_region=err, lengths=lengths, **kw)
            want_status = 0
            for b, n in enumerate(sizes):
                rows = slice(b * M, (b + 1) * M)
                one = {k: (v.reshape(-1, M, n_max)[b, :, :n] if v is not None else None) for k, v in kw.items()}
                sx, sl, ss = ops.border_prompt(xyz[b:b + 1, :n], gt[b:b + 1, :, :n], from_error_region=err, **one)
                assert torch.equal(bx[rows].view(torch.int32), sx.view(torch.int32)), (form, err, b, n)
                assert torch.equal(bl[rows], sl), (form, err, b, n)
                want_status |= int(ss.item())
            assert int(bs.item()) == want_status, (form, err)
            statuses[(form, err)] = want_status
    return statuses


def test_border_prompt_varlen_equals_single_cloud():
    st = _compare_sampler(SIZES, 2, 1)
    assert st[("none", True)] == 1  # the one-point cloud has no border
    st = _compare_sampler(SIZES[1:], 3, 2)  # every cloud has a border: nothing may be flagged
    assert not any(st.values()), st
    _compare_sampler([5000, 4999, 2], 1, 3)  # N_b == N_max, and a tiny cloud next to it


@pytest.mark.parametrize("real", ["empty", "full", "border"])
def test_border_prompt_varlen_status(real):
    """The status follows the real rows: a cloud whose real gt is empty or full is flagged although its padding has a
    border; a cloud with a border is not flagged although its padding is all foreground."""
    from psam_b200 import ops

    def rule(b, m, n, g):
        if b != 1:
            return g
        return np.zeros(n, bool) if real == "empty" else np.ones(n, bool) if real == "full" else g

    sizes = [700, 300, 1000]
    st = _compare_sampler(sizes, 2, 4, rule)
    assert st[("none", True)] == (0 if real == "border" else 1)
    xyz, gt, lg, lengths = _sampler_batch(sizes, 1, 5)
    gt[1, 0, 300:] = True  # cloud 1: a border inside, padding all foreground
    _, _, s = ops.border_prompt(xyz, gt, lengths=lengths, from_error_region=True)
    assert int(s.item()) == 0


# ------------------------------------------------------------------------------------------------
# 2.-3. forward_varlen
# ------------------------------------------------------------------------------------------------
def _models(kind, seed):
    from pc_sam.model import build_point_sam, build_point_sam_hier

    if kind == "base":
        oracle = torch_ref.build_model("eva02_test_tiny", 64, 32, seed=seed)
        model = build_point_sam("eva02_test_tiny", 64, 32)
    else:
        oracle = hier_ref.build_hier_model("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3, seed=seed)
        model = build_point_sam_hier("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3)
    model.load_state_dict(oracle.state_dict(), strict=True)
    model.prompt_iters = oracle.prompt_iters = 3
    return model.cuda().eval(), oracle


def _clouds(sizes, M, seed):
    xs, fs, gs = [], [], []
    for b, n in enumerate(sizes):
        x, f = synth.make_batch(1, n, seed + b)
        xs.append(x[0])
        fs.append(f[0])
        gs.append(synth.make_region_masks(x, M)[0])
    return xs, fs, gs


def _prompt_seq(outs):
    T = len(outs)
    return ([outs[0]["prompt_coords"].cpu()] + [outs[t]["prompt_coords"][:, t:t + 1].cpu() for t in range(1, T)],
            [outs[0]["prompt_labels"].cpu()] + [outs[t]["prompt_labels"][:, t:t + 1].cpu() for t in range(1, T)])


@pytest.mark.parametrize("kind", ["base", "hier"])
def test_forward_varlen_matches_references_per_cloud(kind):
    model, oracle = _models(kind, 21)
    sizes, M = [2048, 3000, 4100], 2
    xs, fs, gs = _clouds(sizes, M, 30)
    with torch.no_grad():
        got = model.forward_varlen([x.to(DEV) for x in xs], [f.to(DEV) for f in fs], [g.to(DEV) for g in gs])
    assert len(got) == len(sizes)
    for b, n in enumerate(sizes):
        outs = got[b]
        assert len(outs) == 3
        for t, o in enumerate(outs):
            C = 3 if t == 0 else 1
            assert o["masks"].shape == (M, C, n) and o["iou_preds"].shape == (M, C)
            assert o["prompt_masks"].shape == (M, n) and o["prompt_coords"].shape == (M, t + 1, 3)
            assert o["prompt_labels"].shape == (M, t + 1)
            # the prompt is the reference sampler's on this cloud alone, given this cloud's previous prompt masks
            prev = outs[t - 1]["prompt_masks"].cpu() if t else None
            wc, wl = torch_ref.sample_prompts_eval(xs[b][None], gs[b][None], prev)
            assert torch.equal(o["prompt_coords"][:, t:t + 1].cpu(), wc), (kind, b, t)
            assert torch.equal(o["prompt_labels"][:, t:t + 1].cpu(), wl.bool()), (kind, b, t)
        pcs, pls = _prompt_seq(outs)
        with torch.no_grad():
            want = oracle.predict_iterative(xs[b][None], fs[b][None], pcs, pls)
        for t in range(3):
            np.testing.assert_allclose(outs[t]["masks"].cpu().numpy(), want[t]["masks"].numpy(), atol=ATOL, rtol=RTOL)


def test_one_cloud_forward_varlen_is_forward():
    """forward_varlen([x], [f], [g])[0] equals forward(x[None], f[None], g[None]) in every field, bit for bit, with
    forward's encode and decode outputs replayed to forward_varlen (the encoder's split-K reductions may round
    differently between two runs): the sampler, the loop and the per-cloud views are what is compared."""
    model, _ = _models("base", 22)
    xs, fs, gs = _clouds([2500], 2, 40)
    x, f, g = xs[0].to(DEV), fs[0].to(DEV), gs[0].to(DEV)
    with torch.no_grad():
        model(x[None], f[None], g[None], is_eval=True)  # packs the weights
    enc_fn, dec_fn, log = model._encode, model._decode_unchecked, []

    def record_encode(*a):
        log.append(("enc", [t.clone() for t in a[:2]], enc_fn(*a)))
        return log[-1][2]

    def record_decode(enc, pc, pl, pm, multi, center_idx=None):
        log.append(("dec", [pc.clone(), pl.clone(), None if pm is None else pm.clone()],
                    dec_fn(enc, pc, pl, pm, multi, center_idx)))
        return log[-1][2]

    replay = iter(())

    def replay_call(kind):
        def fn(*a, **kw):
            k, args, out = next(replay)
            assert k == kind
            mine = [a[0], a[1]] if kind == "enc" else [a[1], a[2], a[3]]
            for u, v in zip(mine, args):
                assert (u is None and v is None) or torch.equal(u, v)
            return out
        return fn

    try:
        model._encode, model._decode_unchecked = record_encode, record_decode
        with torch.no_grad():
            one = model(x[None], f[None], g[None], is_eval=True)
        replay = iter(log)
        model._encode, model._decode_unchecked = replay_call("enc"), replay_call("dec")
        with torch.no_grad():
            (bat,) = model.forward_varlen([x], [f], [g])
        assert next(replay, None) is None
    finally:
        del model._encode, model._decode_unchecked
    assert len(one) == len(bat) == 3
    for o, v in zip(one, bat):
        assert list(o) == list(v)
        for k in o:
            if torch.is_tensor(o[k]):
                assert o[k].dtype == v[k].dtype and torch.equal(o[k], v[k]), k
            else:
                assert o[k] == v[k], k


# ------------------------------------------------------------------------------------------------
# 4. the varlen graph predictor
# ------------------------------------------------------------------------------------------------
def test_varlen_graph_predictor_serves_other_sizes():
    model, oracle = _models("base", 23)
    B, M, n_max = 3, 2, 3000
    pred = model.make_iterative_predictor_varlen(B, M, n_max)
    pred.warmup(*_clouds([2000, 2500, 1800], M, 50))
    assert pred.graph is not None and pred.launches_per_step > 0
    for sizes, seed in (([1500, 2900], 60), ([3000, 700, 2222], 70)):
        xs, fs, gs = _clouds(sizes, M, seed)
        args = ([x.to(DEV) for x in xs], [f.to(DEV) for f in fs], [g.to(DEV) for g in gs])
        with torch.no_grad():
            want = model.forward_varlen(*args)
        got = pred(*args)
        assert len(got) == len(sizes)
        for b, n in enumerate(sizes):
            for t in range(3):
                assert torch.equal(got[b][t]["prompt_coords"], want[b][t]["prompt_coords"]), (sizes, b, t)
                assert torch.equal(got[b][t]["prompt_labels"], want[b][t]["prompt_labels"]), (sizes, b, t)
                assert got[b][t]["masks"].shape == (M, 3 if t == 0 else 1, n)
                torch.testing.assert_close(got[b][t]["masks"], want[b][t]["masks"], atol=2e-4, rtol=1e-4)
                torch.testing.assert_close(got[b][t]["prompt_masks"], want[b][t]["prompt_masks"], atol=2e-4, rtol=1e-4)
    # the last replay against the oracle, cloud by cloud
    for b in range(len(sizes)):
        pcs, pls = _prompt_seq(got[b])
        with torch.no_grad():
            ow = oracle.predict_iterative(xs[b][None], fs[b][None], pcs, pls)
        for t in range(3):
            np.testing.assert_allclose(got[b][t]["masks"].cpu().numpy(), ow[t]["masks"].numpy(), atol=ATOL, rtol=RTOL)
    for fill in (True, False):  # a full or an empty ground truth is reported after the replay
        bad = [g.clone() for g in args[2]]
        bad[1][0] = fill
        with pytest.raises(RuntimeError):
            pred(args[0], args[1], bad)
    got = pred(*args)  # the flag was reset
    assert len(got) == 3


# ------------------------------------------------------------------------------------------------
# 5. the evaluation driver
# ------------------------------------------------------------------------------------------------
DRIVER_SIZES = [180, 240, 700, 2048, 2600, 5000, 9000, 31000]


def _write_crops(tmp_path):
    from pc_sam.utils import ply

    files = []
    for i, n in enumerate(DRIVER_SIZES):
        xyz, feats = synth.make_batch(1, n, 80 + i, "kitti")
        raw = xyz[0].numpy() * 7.5 + np.array([3.0, -2.0, 1.0], dtype=np.float32)
        rgb = ((feats[0].numpy() * 0.5 + 0.5) * 255).astype(np.uint8)
        label = (xyz[0, :, i % 3] > 0.05 * (i % 4)).numpy().astype(np.int32)
        f = str(tmp_path / f"c{i}_{i:04d}.ply")  # one object name per crop: per_object holds the crop's row
        ply.write_ply(f, {"x": raw[:, 0].copy(), "y": raw[:, 1].copy(), "z": raw[:, 2].copy(), "R": rgb[:, 0].copy(),
                          "G": rgb[:, 1].copy(), "B": rgb[:, 2].copy(), "label": label})
        files.append(f)
    return files


def _flips(ref, got, n, eps=1e-3):
    """None if the two runs' loops agree in sign on every real point in every iteration; 'margin' if the first
    difference is a logit within eps of 0 (or a near-tie of the first iteration's best mask); raises otherwise."""
    for t, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r["prompt_coords"], g["prompt_coords"]), t
        if t == 0 and not torch.equal(r["max_iou_pred_ind"], g["max_iou_pred_ind"]):
            top = torch.topk(r["iou_preds"].float(), 2, dim=1).values
            assert float((top[:, 0] - top[:, 1]).min()) < eps, "best mask differs without a near-tie"
            return "margin"
        a, b = r["prompt_masks"][:, :n], g["prompt_masks"][:, :n]
        diff = (a > 0) != (b > 0)
        if diff.any():
            assert float(a[diff].abs().max()) < eps, f"iteration {t}: a logit of |{float(a[diff].abs().max())}| flipped"
            return "margin"
    return None


def test_eval_driver_batches_reproduce_the_per_crop_rows(tmp_path, monkeypatch):
    """evaluate(batch_size=1) and evaluate(batch_size=4) against the parent's per-crop computation, one
    model(**data, is_eval=True) per crop.  The encoder's float atomics make even two forward calls on one crop differ by
    ~1e-5, so a logit that close to 0 may change sign between any two runs: a crop is compared, exactly, where no real
    point's logit changed sign in any iteration; a sign change of a logit within 1e-3 of 0 is printed and the crop
    skipped, and one farther from 0 fails."""
    sys.path.insert(0, os.path.join(ROOT, "point-sam_b200"))
    from evaluation import eval_kitti
    from pc_sam.model.loss import compute_iou

    model, _ = _models("base", 24)
    model.prompt_iters = 3
    files = _write_crops(tmp_path)
    rot = eval_kitti.parse_rotation(None)
    ref_rows, ref_outs = {}, {}
    with torch.no_grad():
        for f in files:
            data = eval_kitti.transform_fn(eval_kitti.load_crop(f, rot), device=DEV)
            eval_kitti.set_group_shape(model, data["coords"].shape[1])
            outs = model(**data, is_eval=True)
            gt = data["gt_masks"].flatten(0, 1)
            k = os.path.basename(f).split("_")[0]
            ref_rows[k] = np.array([compute_iou(o["prompt_masks"], gt).detach().cpu().numpy().mean() for o in outs])
            ref_outs[k] = outs
    seen, fv = [], model.forward_varlen

    def recording(coords, features, gt_masks, is_eval=True):
        out = fv(coords, features, gt_masks, is_eval)
        seen.append(([int(c.shape[0]) for c in coords], out))
        return out

    monkeypatch.setattr(model, "forward_varlen", recording)
    for bs in (1, 4):
        seen.clear()
        got = eval_kitti.evaluate(model, files, rotation=rot, log=None, batch_size=bs)
        assert list(got["per_object"]) == list(ref_rows)
        assert sorted(n for b, _ in seen for n in b) == sorted(DRIVER_SIZES)
        assert max(len(b) for b, _ in seen) == min(bs, 4)
        by_size = {n: o for b, out in seen for n, o in zip(b, out)}
        compared = 0
        for f, n in zip(files, DRIVER_SIZES):
            k = os.path.basename(f).split("_")[0]
            why = _flips(ref_outs[k], by_size[n], n)
            print(f"[eval varlen] batch {bs} crop {k} (N={n}): "
                  f"{'skipped, a logit within 1e-3 of 0 changed sign' if why else 'compared'}")
            if why:
                continue
            assert np.array_equal(got["per_object"][k], ref_rows[k]), (bs, k, got["per_object"][k], ref_rows[k])
            compared += 1
        assert compared > len(files) // 2, (bs, compared)


# ------------------------------------------------------------------------------------------------
# 6. full size, once
# ------------------------------------------------------------------------------------------------
def test_forward_varlen_full_size_vit_l():
    """ViT-L, 8 clouds of 2048 .. 30000 points with the evaluation's 2048 groups of 256: the first prompts are the
    reference sampler's on each cloud, and each cloud's first-iteration masks agree with its own forward."""
    from pc_sam.model import build_point_sam

    torch.manual_seed(0)
    model = build_point_sam("eva02_large_patch14_448", 2048, 256, prompt_iters=5).to(DEV).eval()
    sizes = [2048, 30000, 4096, 17000, 9000, 2500, 24576, 12000]
    xs, fs, gs = _clouds(sizes, 1, 90)
    with torch.no_grad():
        got = model.forward_varlen([x.to(DEV) for x in xs], [f.to(DEV) for f in fs], [g.to(DEV) for g in gs])
    for b, n in enumerate(sizes):
        assert len(got[b]) == 5 and got[b][4]["prompt_coords"].shape == (1, 5, 3)
        wc, wl = torch_ref.sample_prompts_eval(xs[b][None], gs[b][None], None)
        assert torch.equal(got[b][0]["prompt_coords"].cpu(), wc) and torch.equal(got[b][0]["prompt_labels"].cpu(), wl.bool())
        with torch.no_grad():
            m, _ = model.predict_masks(xs[b][None].to(DEV), fs[b][None].to(DEV), got[b][0]["prompt_coords"],
                                       got[b][0]["prompt_labels"].long(), None, True)
        np.testing.assert_allclose(got[b][0]["masks"].cpu().numpy(), m.cpu().numpy(), atol=ATOL, rtol=RTOL)
        assert torch.isfinite(got[b][4]["masks"]).all()
