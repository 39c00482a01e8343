"""GPU parity of the hierarchical model (PointCloudSAMHier: PatchEmbedHier, MaskEncoderHier, MaskDecoderHier) against the
fixture minted by the reference's own modules and against the fp32 oracle, plus its serving and caller paths.

Tolerance on mask logits is the north-star bound: 1e-3 abs + 1e-2 rel (fp32); FPS and kNN indices exact."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hier_ref, synth  # noqa: E402
from oracle.make_golden import state_checksum  # noqa: E402

ATOL, RTOL = 1e-3, 1e-2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(encoder, G, K, radius, prompt_iters=3, seed=1234):
    from pc_sam.model import build_point_sam_hier

    oracle = hier_ref.build_hier_model(encoder, G, K, radius, prompt_iters=prompt_iters, seed=seed)
    model = build_point_sam_hier(encoder, G, K, radius, prompt_iters)
    model.load_state_dict(oracle.state_dict(), strict=True)
    return model.cuda().eval(), oracle


def _report(name, got, want):
    err = (got - want).abs()
    print(f"[parity] {name}: max|err|={float(err.max()):.3e} mean|err|={float(err.mean()):.3e} "
          f"range=[{float(want.min()):.3f},{float(want.max()):.3f}]")


def test_hier_golden_predict_iterative_and_predict_masks(golden_dir):
    g = np.load(os.path.join(golden_dir, "hier.npz"))
    B, M, N, G1, G2, K1, K2, R, seed = [int(v) for v in g["meta"]]
    model, oracle = _build(str(g["encoder"]), (G1, G2), (K1, K2), tuple(float(r) for r in g["radius"]), R, 1234 + seed)
    assert state_checksum(oracle.state_dict()) == str(g["weights_checksum"])
    d = torch.device("cuda:0")
    xyz, feats = torch.from_numpy(g["xyz"]).to(d), torch.from_numpy(g["feats"]).to(d)
    seq_c = [torch.from_numpy(g[f"prompt_coords{t}"]).to(d) for t in range(R)]
    seq_l = [torch.from_numpy(g[f"prompt_labels{t}"]).to(d) for t in range(R)]
    with torch.no_grad():
        emb, (p1, p2) = model.pc_encoder(xyz, feats)
        outs = model.predict_iterative(xyz, feats, seq_c, seq_l)
    assert np.array_equal(p1["fps_idx"].cpu().numpy(), g["fps_idx1"])
    assert np.array_equal(p1["centers"].cpu().numpy(), g["centers1"])
    assert np.array_equal(p2["centers"].cpu().numpy(), g["centers2"])
    assert np.array_equal(np.sort(p1["knn_idx"].cpu().numpy(), -1), g["knn1_sorted"])
    assert np.array_equal(np.sort(p2["knn_idx"].cpu().numpy(), -1), g["knn2_sorted"])
    np.testing.assert_allclose(p1["embeddings"].cpu().numpy(), g["emb1"], atol=2e-4, rtol=1e-3)
    np.testing.assert_allclose(p2["embeddings"].cpu().numpy(), g["emb2"], atol=2e-4, rtol=1e-3)
    np.testing.assert_allclose(emb.cpu().numpy(), g["pc_embeddings"], atol=2e-4, rtol=1e-3)
    for t, o in enumerate(outs):
        _report(f"hier golden round {t}", o["masks"].cpu(), torch.from_numpy(g[f"masks{t}"]))
        np.testing.assert_allclose(o["masks"].cpu().numpy(), g[f"masks{t}"], atol=ATOL, rtol=RTOL)
        np.testing.assert_allclose(o["iou_preds"].cpu().numpy(), g[f"iou{t}"], atol=ATOL, rtol=RTOL)
    # predict_masks, reference form: one round of the loop body with the given prompts and prompt mask
    pm0 = torch.from_numpy(g["prompt_masks0"]).to(d)
    pc1, pl1 = torch.cat(seq_c[:2], 1), torch.cat(seq_l[:2], 1)
    with torch.no_grad():
        m0, i0 = model.predict_masks(xyz, feats, seq_c[0], seq_l[0], None, True)
        m1, i1 = model.predict_masks(xyz, feats, pc1, pl1, pm0, False)
    np.testing.assert_allclose(m0.cpu().numpy(), g["masks0"], atol=ATOL, rtol=RTOL)
    np.testing.assert_allclose(i0.cpu().numpy(), g["iou0"], atol=ATOL, rtol=RTOL)
    np.testing.assert_allclose(m1.cpu().numpy(), g["masks1"], atol=ATOL, rtol=RTOL)
    np.testing.assert_allclose(i1.cpu().numpy(), g["iou1"], atol=ATOL, rtol=RTOL)
    # demo form after set_pointcloud (one cloud)
    model.set_pointcloud(xyz[:1], feats[:1])
    _, scores, logits = model.predict_masks(seq_c[0][:1], seq_l[0][:1], None, True)
    np.testing.assert_allclose(logits.cpu().numpy(), g["masks0"][:1], atol=ATOL, rtol=RTOL)
    np.testing.assert_allclose(scores.cpu().numpy(), g["iou0"][:1], atol=ATOL, rtol=RTOL)


@pytest.mark.parametrize("tc", [True, False])
def test_hier_full_size_vs_fp32_oracle_on_gpu(tc, monkeypatch):
    """hier.yaml shapes: N = 32768, G = (2048, 512), K = (32, 32), radius (0.05, 0.1), ViT-L; B = 2 clouds x M = 2 masks,
    3 rounds with mask feedback; the decoder's patch-row projections on the tensor cores and on the SIMT linear."""
    from psam_b200 import engine

    monkeypatch.setattr(engine, "DECODER_TC", tc)
    model, oracle = _build("eva02_large_patch14_448", (2048, 512), (32, 32), (0.05, 0.1), 3, 77)
    d = torch.device("cuda:0")
    oracle = oracle.to(d)
    B, M, N = 2, 2, 32768
    xyz, feats = synth.make_batch(B, N, 21)
    seq_c = [synth.make_prompts(xyz, M, s)[0].reshape(B * M, 1, 3) for s in (1, 2, 3)]
    seq_l = [synth.make_prompts(xyz, M, s)[1].reshape(B * M, 1) for s in (1, 2, 3)]
    xyz, feats = xyz.to(d), feats.to(d)
    seq_c, seq_l = [c.to(d) for c in seq_c], [l.to(d) for l in seq_l]
    with torch.no_grad():
        want = oracle.predict_iterative(xyz, feats, seq_c, seq_l)
        got = model.predict_iterative(xyz, feats, seq_c, seq_l)
    for t, (a, b) in enumerate(zip(got, want)):
        _report(f"hier full size tc={tc} round {t} masks", a["masks"].cpu(), b["masks"].cpu())
        np.testing.assert_allclose(a["masks"].cpu().numpy(), b["masks"].cpu().numpy(), atol=ATOL, rtol=RTOL)
        np.testing.assert_allclose(a["iou_preds"].cpu().numpy(), b["iou_preds"].cpu().numpy(), atol=ATOL, rtol=RTOL)


@pytest.mark.parametrize("D", [256, 128])
def test_interp_add_ln_gelu_vs_fp64(D):
    """y[z*N+n] = GELU(LN(sum_k w f[z, idx] + addend[z / rep, n])), split-bf16 out; Z = 4, rep = 2, ragged N."""
    from psam_b200 import native as nv, ops

    d = torch.device("cuda:0")
    g = torch.Generator().manual_seed(D)
    B, rep, G, N = 2, 2, 37, 1001
    Z = B * rep
    f = torch.randn(Z * G, D, generator=g)
    idx = torch.randint(0, G, (B, N, 3), generator=g)
    w = torch.rand(B, N, 3, generator=g)
    w = w / w.sum(-1, keepdim=True)
    add = torch.randn(B * N, D, generator=g)
    gamma, beta = torch.rand(D, generator=g) + 0.5, torch.randn(D, generator=g)
    out = ops.Split(Z * N, D, d)
    fd, idxd, wd, addd, gd, bd = (t.to(d) for t in (f, idx, w, add, gamma, beta))  # alive until the kernel has run
    nv.check(nv.lib().psam_interp_add_ln_gelu(nv.ptr(fd), Z, rep, G, D, nv.ptr(idxd), nv.ptr(wd), N, nv.ptr(addd), nv.ptr(gd),
                                              nv.ptr(bd), 1e-5, out.ptr(), out.plane, out.pitch, nv.stream()), "interp_add_ln_gelu")
    torch.cuda.synchronize()
    fz = f.double().view(Z, G, D)
    zb = torch.arange(Z) // rep
    gath = fz[torch.arange(Z)[:, None, None], idx[zb]]                   # [Z, N, 3, D]
    x = (gath * w[zb].double()[..., None]).sum(2) + add.double().view(B, N, D)[zb]
    want = torch.nn.functional.gelu(torch.nn.functional.layer_norm(x, (D,), gamma.double(), beta.double(), 1e-5))
    err = float((out.float().cpu().double() - want.reshape(Z * N, D)).abs().max())
    print(f"[kernel] interp_add_ln_gelu D={D}: max|err| vs fp64 {err:.2e}")
    assert err < 1e-4  # split-bf16 output: residual <= 2^-17 relative


def _tiny():
    return _build("eva02_test_tiny", (128, 32), (32, 16), (0.2, 0.4), 3, 5)


def test_hier_graph_predictors_replay_eager_outputs():
    model, _ = _tiny()
    d = torch.device("cuda:0")
    clouds = [synth.make_batch(1, 2048, s) for s in (1, 2, 3)]
    prompts = [synth.make_prompts(c[0], 1, s) for s, c in enumerate(clouds)]
    want = []
    with torch.no_grad():
        for (xyz, feats), (pc, pl) in zip(clouds, prompts):
            m, i = model.predict_masks(xyz.to(d), feats.to(d), pc.to(d), pl.to(d), None, True)
            want.append((m.cpu(), i.cpu()))
    args = [[t.to(d) for t in (*c, *p)] for c, p in zip(clouds, prompts)]
    gp = model.make_predictor(1, 2048, 1)
    gp.warmup(*args[0])
    assert gp.graph is not None and gp.launches_per_step > 0
    for a, (wm, wi) in zip(args, want):
        m, i = gp(*a)
        gp.check()
        torch.testing.assert_close(m.cpu(), wm, atol=2e-5, rtol=1e-4)
        torch.testing.assert_close(i.cpu(), wi, atol=2e-5, rtol=1e-4)
    pp = model.make_pipelined_predictor(1, 2048, 1, depth=2)
    pp.warmup(*args[0])
    tickets = [pp.submit(*a) for a in args[:2]]
    for t in tickets:
        m, i = pp.result(t)
        torch.testing.assert_close(m.cpu(), want[t][0], atol=2e-5, rtol=1e-4)
        torch.testing.assert_close(i.cpu(), want[t][1], atol=2e-5, rtol=1e-4)
    # the evaluation loop (GT border sampler, is_eval=True) as one graph
    B, M, N = 2, 2, 1500
    it = model.make_iterative_predictor(B, M, N)
    cl = []
    for s_ in (0, 1):
        xyz, feats = synth.make_batch(B, N, 90 + s_)
        gt = torch.stack([torch.stack([xyz[b, :, (m + s_) % 3] > 0.1 * m for m in range(M)]) for b in range(B)])
        cl.append((xyz.to(d), feats.to(d), gt.to(d)))
    it.warmup(*cl[0])
    assert it.graph is not None
    for c in (cl[1], cl[0]):
        with torch.no_grad():
            want_it = model(*c, is_eval=True)
        got = it(*c)
        assert len(got) == 3
        for t in range(3):
            assert torch.equal(got[t]["prompt_coords"], want_it[t]["prompt_coords"])
            torch.testing.assert_close(got[t]["masks"], want_it[t]["masks"], atol=2e-5, rtol=1e-4)
            torch.testing.assert_close(got[t]["iou_preds"], want_it[t]["iou_preds"], atol=2e-5, rtol=1e-4)


def test_hier_random_sampler_forward_and_demo_session(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "point-sam_b200"))
    from demo.app import SegmentSession
    from pc_sam.utils import ply

    model, oracle = _tiny()
    d = torch.device("cuda:0")
    # forward(is_eval=False): the reference's random sampler every round; prompts lie in the cloud, masks are shaped
    B, M, N = 2, 2, 1500
    xyz, feats = synth.make_batch(B, N, 31)
    gt = torch.stack([torch.stack([xyz[b, :, m] > 0.0 for m in range(M)]) for b in range(B)]).to(d)
    with torch.no_grad():
        outs = model(xyz.to(d), feats.to(d), gt)
    assert [tuple(o["masks"].shape) for o in outs] == [(4, 3, N), (4, 1, N), (4, 1, N)]
    assert outs[-1]["prompt_coords"].shape == (4, 3, 3)
    # the sampled prompts replayed through the oracle give the same masks
    pcs = [outs[0]["prompt_coords"].cpu()] + [outs[t]["prompt_coords"][:, t:t + 1].cpu() for t in (1, 2)]
    pls = [outs[0]["prompt_labels"].cpu()] + [outs[t]["prompt_labels"][:, t:t + 1].cpu() for t in (1, 2)]
    with torch.no_grad():
        want = oracle.predict_iterative(xyz, feats, pcs, pls)
    for t in range(3):
        np.testing.assert_allclose(outs[t]["masks"].cpu().numpy(), want[t]["masks"].numpy(), atol=ATOL, rtol=RTOL)
    # demo session: two clicks on one cloud, encoded once
    pts = np.concatenate([xyz[0].numpy() * 4 + 1, np.round((feats[0].numpy() * 0.5 + 0.5) * 255)], axis=1)
    scene = tmp_path / "scene.ply"
    scene.write_text(f"ply\nformat ascii 1.0\nelement vertex {N}\nproperty float x\nproperty float y\nproperty float z\n"
                     "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n" +
                     "\n".join("%f %f %f %d %d %d" % tuple(r) for r in pts) + "\n")
    encodes = []
    enc = model._encode
    model._encode = lambda *a: encodes.append(1) or enc(*a)
    sess = SegmentSession(model, device=d, output_dir=str(tmp_path / "results"))
    resp = sess.pointcloud(str(scene))
    nxyz = np.array(resp["xyz"], dtype=np.float64).reshape(-1, 3)
    r1 = sess.segment({"prompt_point": nxyz[10].tolist(), "prompt_label": 1})
    r2 = sess.segment({"prompt_point": nxyz[200].tolist(), "prompt_label": 0})
    assert len(r1["seg"]) == N and len(r2["seg"]) == N and len(encodes) == 1
    cx = torch.from_numpy(nxyz).float()[None]
    cf = torch.from_numpy(np.array(resp["rgb"]).reshape(-1, 3)).float()[None]
    with torch.no_grad():
        m, s = oracle.predict_masks(cx, cf, cx[:, 10:11], torch.ones(1, 1, dtype=torch.long), None, True)
        m2, _ = oracle.predict_masks(cx, cf, torch.cat([cx[:, 10:11], cx[:, 200:201]], 1), torch.tensor([[1, 0]]),
                                     m[:, int(torch.argmax(s[0]))], False)
    np.testing.assert_allclose(sess.prompt_mask.cpu().numpy()[0], m2[0, 0].numpy(), atol=ATOL, rtol=RTOL)


def test_hier_eval_driver(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "point-sam_b200"))
    from evaluation import eval_kitti
    from pc_sam.utils import ply

    model, _ = _tiny()
    files = []
    for i, n in enumerate((900, 600)):
        xyz, feats = synth.make_batch(1, n, 50 + i, "kitti")
        raw = xyz[0].numpy() * 7.5 + np.array([3.0, -2.0, 1.0], dtype=np.float32)
        rgb = ((feats[0].numpy() * 0.5 + 0.5) * 255).astype(np.uint8)
        label = (xyz[0, :, 0] > 0.05).numpy().astype(np.int32)
        f = str(tmp_path / f"car_{i:04d}.ply")
        ply.write_ply(f, {"x": raw[:, 0].copy(), "y": raw[:, 1].copy(), "z": raw[:, 2].copy(), "R": rgb[:, 0].copy(),
                          "G": rgb[:, 1].copy(), "B": rgb[:, 2].copy(), "label": label})
        files.append(f)
    res = eval_kitti.evaluate(model, files, log=None)
    assert res["total"].shape == (model.prompt_iters,) and list(res["per_object"]) == ["car"]
    assert np.all((res["total"] >= 0) & (res["total"] <= 1))
