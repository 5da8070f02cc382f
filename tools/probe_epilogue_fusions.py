"""Fused-epilogue GEMMs against the launch pairs they replace (CUDA events, rotating operand sets): GELU forward / backward at the
BERT (K = 1024) and Falcon (K = 4544) MLP shapes. One JSON line per case.
    python tools/probe_epilogue_fusions.py"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dalm_b200 import ops

dev = torch.device("cuda:0")
bf16 = torch.bfloat16


def timeit(fn, iters=8, warmup=3):
    for _ in range(warmup): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3


def rnd(*shape, s=0.1):
    return (torch.randn(*shape, device=dev) * s).to(bf16)


def gelu_case(name, M, H, F, nbuf=3):
    xs = [rnd(M, H) for _ in range(nbuf)]
    w1, w2T = rnd(F, H), rnd(F, H)                       # W1 [F,H]; W2^T [F,H] (dgrad of y = act W2^T against the transposed copy)
    b = torch.randn(F, device=dev)
    pre, act = torch.empty(M, F, device=dev, dtype=bf16), torch.empty(M, F, device=dev, dtype=bf16)
    i = [0]
    def nxt():
        i[0] += 1
        return xs[i[0] % nbuf]
    t_two = timeit(lambda: ops.gelu_fwd(ops.gemm(nxt(), w1, bias=b, out=pre), act))
    t_one = timeit(lambda: ops.gemm_gelu(nxt(), w1, bias=b, pre=pre, act=act))
    t_gemm = timeit(lambda: ops.gemm(nxt(), w1, bias=b, out=pre))
    print(json.dumps({"case": name + " fwd", "M": M, "N": F, "K": H, "gemm_us": round(t_gemm, 1), "gemm+gelu_fwd_us": round(t_two, 1),
                      "fused_us": round(t_one, 1)}), flush=True)
    dact = torch.empty(M, F, device=dev, dtype=bf16)
    t_two = timeit(lambda: ops.gelu_bwd_(pre, ops.gemm(nxt(), w2T, out=dact)))
    t_one = timeit(lambda: ops.gemm(nxt(), w2T, out=dact, act=2, resid=pre))
    t_gemm = timeit(lambda: ops.gemm(nxt(), w2T, out=dact))
    print(json.dumps({"case": name + " bwd", "M": M, "N": F, "K": H, "gemm_us": round(t_gemm, 1), "gemm+gelu_bwd_us": round(t_two, 1),
                      "fused_us": round(t_one, 1)}), flush=True)


if __name__ == "__main__":
    gelu_case("bge-large cfg-2 (26700 rows)", 26700, 1024, 4096)
    gelu_case("bge-large cfg-3 (3204 rows)", 3204, 1024, 4096)
    gelu_case("falcon-7b (4096 rows)", 4096, 4544, 18176)
    gelu_case("falcon-7b cfg-5 (36864 rows)", 36864, 4544, 18176, nbuf=2)
