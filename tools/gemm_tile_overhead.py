"""Fixed per-launch cost of the GEMM outside its main loop: time ops.gemm and the fused entry points at the cfg-3 generator
widths (M = 4608) over K = 1024 .. 8192, and fit time = intercept + slope * K. The slope is the k-loop, the intercept what
every launch pays regardless of K: tile epilogues, the first TMA round trip of every tile, launch and tail effects.

CUDA events over a window of more than a second per point; operands rotate over enough sets that L2 does not hold them
(as tools/bench_gemm_r2.py does). One JSON line per point and one per fit.

    python tools/gemm_tile_overhead.py [--ks 1024,2048,4096,8192] [--window 1.0]
"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from dalm_b200 import ops

dev = torch.device("cuda:0")
bf16, f32 = torch.bfloat16, torch.float32
M = 18 * 256                                                    # cfg-3: bs 18 x 256 generator tokens


def timeit(fn, window):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fn(); e.record(); torch.cuda.synchronize()
    iters = max(10, int(window / max(s.elapsed_time(e) * 1e-3, 1e-6)) + 1)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e-3 / iters, iters


def operands(N, K, nbuf):
    As = [(torch.randn(M, K, device=dev) * 0.1).to(bf16) for _ in range(nbuf)]
    Bs = [(torch.randn(N, K, device=dev) * 0.1).to(bf16) for _ in range(nbuf)]
    return As, Bs


def make_case(kind, K):
    """-> (N, fn) for one entry point at its cfg-3 width"""
    if kind == "bf16":
        N = 4096
    elif kind == "f32+resid":
        N = 4096
    elif kind == "swiglu":
        N = 22016
    else:
        N = 12288
    nbuf = max(2, int(-(-4 * 50e6 // (2 * (M + N) * K))) + 1)  # >= 4 x the 50 MB L2 in rotation
    As, Bs = operands(N, K, nbuf)
    i = [0]
    if kind == "bf16":
        out = torch.empty(M, N, device=dev, dtype=bf16)
        call = lambda a, b: ops.gemm(a, b, out=out)
    elif kind == "f32+resid":
        out = torch.empty(M, N, device=dev, dtype=f32)
        r = torch.randn(M, N, device=dev)
        call = lambda a, b: ops.gemm(a, b, out=out, resid=r)
    elif kind == "swiglu":
        gu = torch.empty(M, N, device=dev, dtype=bf16); act = torch.empty(M, N // 2, device=dev, dtype=bf16)
        call = lambda a, b: ops.gemm_swiglu(a, b, gu, act)
    else:
        L = 256
        out = torch.empty(M, N, device=dev, dtype=bf16)
        cos_t, sin_t = torch.randn(L, 64, device=dev), torch.randn(L, 64, device=dev)
        call = lambda a, b: ops.gemm_rope(a, b, cos_t, sin_t, L, 8192, out=out)

    def fn():
        j = i[0] % nbuf; i[0] += 1
        call(As[j], Bs[j])
    return N, fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1024,2048,4096,8192")
    ap.add_argument("--kinds", default="bf16,f32+resid,swiglu,rope")
    ap.add_argument("--window", type=float, default=1.0, help="seconds of timed launches per point")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    ks = [int(k) for k in args.ks.split(",")]
    for kind in args.kinds.split(","):
        ts = []
        for K in ks:
            N, fn = make_case(kind, K)
            t, iters = timeit(fn, args.window)
            ts.append(t)
            print(json.dumps({"kind": kind, "M": M, "N": N, "K": K, "us": round(t * 1e6, 1), "iters": iters,
                              "tflops": round(2.0 * M * N * K / t / 1e12, 1)}), flush=True)
            del fn
            torch.cuda.empty_cache()
        slope, icpt = np.polyfit(np.array(ks, dtype=float), np.array(ts), 1)
        t4096 = icpt + slope * 4096
        tiles = -(-M // 128) * -(-N // 256)
        per_cta = -(-tiles // torch.cuda.get_device_properties(0).multi_processor_count)
        print(json.dumps({"kind": kind, "fit": "t = a + b K", "intercept_us": round(icpt * 1e6, 1),
                          "us_per_k1024": round(slope * 1024 * 1e6, 1), "intercept_share_at_k4096": round(icpt / t4096, 4),
                          "tiles": tiles, "tiles_per_cta": per_cta,
                          "intercept_us_per_tile_of_a_cta": round(icpt * 1e6 / per_cta, 2)}), flush=True)


if __name__ == "__main__":
    main()
