"""Where the time of the split-bf16 GEMM goes, in the regime of the timed benchmark (8 streams in flight).

Prints one JSON object:
  shapes   - the four ViT-L block GEMMs of a c2 cloud (M = 512 rows) with the epilogues the engine gives them, under the
             throughput tile policy (tile_hint = 1): us per launch (machine time: 8 streams share the GPU) and executed
             TFLOP/s (3 bf16 passes), next to torch/cuBLAS bf16 [M, 3K] x [3K, N] - the same executed work - on 8 streams
  square   - one large square bf16 cuBLAS GEMM: what this card sustains under its power limit
  k_sweep  - M = 512, N = 3072, K in {256, 1024, 2752, 8192} at BN = 256 and BN = 128, fitted as
             time = fixed + kb * t_kb with kb = K / 64; t_kb against the ideal time of a 64-wide k-slice at the sampled SM clock
  device   - name, power limit and clocks (nvidia-smi queries only; no setting is changed)
usage: python tools/gemm_regime.py [--streams 8] [--launches 40]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "point-sam_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from psam_b200 import ops  # noqa: E402

FLOP_PER_CLK_SM = 4096  # dense bf16 tensor-core flops per SM per clock on H100 (989 TFLOP/s = 132 SMs x 4096 x 1830 MHz)


def smi(fields):
    r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    return [c.strip() for c in r.stdout.strip().split(",")]


class Clocks:
    def __init__(self):
        self.rows, self.proc = [], None

    def __enter__(self):
        self.proc = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits",
                                      "-lms", "50"], stdout=subprocess.PIPE, text=True)
        threading.Thread(target=lambda: [self.rows.append(line) for line in self.proc.stdout], daemon=True).start()
        return self

    def __exit__(self, *exc):
        self.proc.terminate()
        self.proc.wait()

    def sm_mhz(self):
        v = sorted(float(r.split(",")[0]) for r in self.rows if r.split(",")[0].strip().replace(".", "").isdigit())
        return v[len(v) // 2] if v else None


def regime(fns, launches):
    """Machine time per launch (ms) of fns[i] replayed `launches` times on stream i, all streams at once."""
    streams = [torch.cuda.Stream() for _ in fns]
    main = torch.cuda.current_stream()

    def run(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(main)
        for s, fn in zip(streams, fns):
            s.wait_event(e0)
            with torch.cuda.stream(s):
                for _ in range(n):
                    fn()
            d = torch.cuda.Event()
            d.record(s)
            main.wait_event(d)
        e1.record(main)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    run(3)
    return min(run(launches) for _ in range(3)) / (launches * len(fns))


def block_gemm(name, M, dev, bn):
    """One of the LayerNorm-free block GEMMs with the engine's epilogue; returns (N, K, launch)."""
    D, Hf = 1024, 2752
    N, K = {"qkv": (3 * D, D), "proj": (D, D), "fc1": (2 * Hf, D), "fc2": (D, Hf)}[name]
    a, w = ops.Split(M, K, dev), ops.Split(N, K, dev)
    a.t.normal_()
    w.t.normal_().mul_(K ** -0.5)
    bias = torch.randn(N, device=dev)
    stats_in = torch.stack([torch.zeros(M, device=dev), torch.full((M,), float(K), device=dev)], 1).contiguous()
    ln = (stats_in, torch.randn(N, device=dev), K, 1e-6)
    stats = torch.zeros(M, 2, device=dev)
    if name == "qkv":
        out = ops.Split(M, N, dev)
        fn = lambda: ops.gemm(a, w, bias=bias, out_split=out, ln_fold=ln)
    elif name == "fc1":
        out = ops.Split(M, N // 2, dev)
        fn = lambda: ops.gemm(a, w, bias=bias, out_split=out, swiglu=True, stats_out=stats, ln_fold=ln)
    else:
        x = torch.randn(M, N, device=dev)
        out = ops.Split(M, N, dev)
        fn = lambda: ops.gemm(a, w, bias=bias, out_f32=x, resid=x, out_split=out, stats_out=stats,
                              ln_fold=ln if name == "fc2" else None)

    def launch():
        prev, ops.GEMM_TILE_BN, ops.GEMM_TILE_HINT = (ops.GEMM_TILE_BN, ops.GEMM_TILE_HINT), bn, 1
        try:
            fn()
        finally:
            ops.GEMM_TILE_BN, ops.GEMM_TILE_HINT = prev
    return N, K, launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--launches", type=int, default=40)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_regime: no CUDA device")
    dev = torch.device("cuda:0")
    S, L, M = args.streams, args.launches, 512
    name, plimit, max_sm = smi("name,power.limit,clocks.max.sm")
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    res = {"device": {"name": name, "power_limit_w": plimit, "sm_max_mhz": max_sm, "sms": nsm}, "streams": S, "m_rows": M}
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False

    with Clocks() as clk:
        shapes = {}
        for nm in ("qkv", "proj", "fc1", "fc2"):
            fns = [block_gemm(nm, M, dev, 0) for _ in range(S)]
            N, K = fns[0][0], fns[0][1]
            ms = regime([f[2] for f in fns], L)
            ex = 3 * 2.0 * M * N * K
            a3 = [torch.randn(M, 3 * K, device=dev, dtype=torch.bfloat16) for _ in range(S)]
            w3 = torch.randn(N, 3 * K, device=dev, dtype=torch.bfloat16)
            c3 = [torch.empty(M, N, device=dev, dtype=torch.bfloat16) for _ in range(S)]
            ms_cb = regime([(lambda i=i: torch.mm(a3[i], w3.t(), out=c3[i])) for i in range(S)], L)
            shapes[nm] = {"N": N, "K": K, "us_per_launch": ms * 1e3, "executed_tflops": ex / (ms / 1e3) / 1e12,
                          "cublas_3k_us": ms_cb * 1e3, "cublas_3k_tflops": ex / (ms_cb / 1e3) / 1e12,
                          "vs_cublas": ms_cb / ms}
        res["shapes"] = shapes
        q = 8192
        a = torch.randn(q, q, device=dev, dtype=torch.bfloat16)
        b = torch.randn(q, q, device=dev, dtype=torch.bfloat16)
        ms_sq = regime([lambda: torch.mm(a, b)], 20)
        res["square"] = {"size": q, "tflops": 2.0 * q ** 3 / (ms_sq / 1e3) / 1e12}
        del a, b

        sweep = {}
        for bn in (256, 128):
            pts = []
            for K in (256, 1024, 2752, 8192):
                aa, ww = ops.Split(M, K, dev), ops.Split(3072, K, dev)
                aa.t.normal_()
                ww.t.normal_()
                bias = torch.randn(3072, device=dev)
                outs = [ops.Split(M, 3072, dev) for _ in range(S)]

                def mk(o):
                    def f():
                        prev, ops.GEMM_TILE_BN = ops.GEMM_TILE_BN, bn
                        try:
                            ops.gemm(aa, ww, bias=bias, out_split=o)
                        finally:
                            ops.GEMM_TILE_BN = prev
                    return f
                pts.append((K / 64, regime([mk(o) for o in outs], L) * 1e3))
            kb, us = np.array([p[0] for p in pts]), np.array([p[1] for p in pts])
            t_kb, fixed = np.polyfit(kb, us, 1)
            sweep[f"bn{bn}"] = {"points_us": {str(int(k * 64)): u for k, u in pts}, "fixed_us": float(fixed), "t_kb_us": float(t_kb),
                                "fixed_share_k1024": float(fixed / us[1])}
    sm = clk.sm_mhz()
    res["device"]["sm_mhz_sampled"] = sm
    if sm:
        ideal = 3 * 2.0 * M * 3072 * 64 / (nsm * FLOP_PER_CLK_SM * sm * 1e6) * 1e6  # us per 64-wide k-slice of the launch
        for v in sweep.values():
            v["ideal_t_kb_us"] = ideal
            v["t_kb_efficiency"] = ideal / v["t_kb_us"]
    res["k_sweep"] = sweep
    print(json.dumps(res))


if __name__ == "__main__":
    main()
