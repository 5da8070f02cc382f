"""Cost of sampling (temperature -> top-k -> top-p -> draw, `sample_step`) against greedy argmax (`greedy_step`), with CUDA events:
  * the kernels alone, for B in {1, 16}, V in {32000 (Llama-2), 65024 (Falcon)}, (top_k, top_p) in {(50, 0.9), (0, 0.9), (0, 1)};
  * the per-token decode step of a Llama-2-7B-shaped generator (random bf16 weights) at B = 16, greedy vs Llama-2's sampling
    config (T 0.6, top-k 50, top-p 0.9), as the difference of two generation lengths so the prefill cancels.
Prints one JSON object with the card's name and power limit.
    python tools/bench_sampling.py [--skip-model]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from dalm_b200 import ops, synthetic
from dalm_b200.engine import params

dev = torch.device("cuda:0")
bf16 = torch.bfloat16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def events_us(fn, n):
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def kernels():
    out = []
    g = torch.Generator().manual_seed(0)
    for B in (1, 16):
        for V in (32000, 65024):
            logits = (torch.randn(B, V, generator=g) * 3).to(bf16).to(dev)
            T = 2
            st = lambda: [torch.ones(B, dtype=torch.int32, device=dev), torch.zeros(B, T, dtype=torch.int64, device=dev),
                          torch.zeros(B, T, dtype=torch.int64, device=dev), torch.zeros(B, dtype=torch.int64, device=dev),
                          torch.zeros(B, dtype=torch.int64, device=dev), torch.zeros(T, dtype=torch.int32, device=dev)]
            u, t, m, nx, p, a = st()
            greedy = events_us(lambda: ops.greedy_step_(logits, V, None, 0, u, t, m, 1, nx, p, a), 500)
            for k, tp in ((50, 0.9), (0, 0.9), (0, 1.0)):
                samp = events_us(lambda: ops.sample_step_(logits, V, None, 0, u, t, m, 1, nx, p, a, temperature=0.6, top_k=k,
                                                          top_p=tp, seed=1), 500)
                out.append({"B": B, "V": V, "top_k": k, "top_p": tp, "greedy_us": round(greedy, 2), "sample_us": round(samp, 2)})
    return out


def model_step(B=16, L0=64):
    cfg = synthetic.llama_config("Llama-2-7b-hf")
    from dalm_b200.engine.llama import LlamaDecoder
    dec = LlamaDecoder(cfg, params.random_state_dict("llama", cfg, seed=0, dtype=bf16, device=dev), device=dev)
    torch.cuda.empty_cache()
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(3, cfg["vocab_size"], (B, L0), generator=g).to(dev)
    mask = torch.ones_like(ids)
    os.environ["DALM_B200_DECODE_GRAPH"] = "1"
    modes = {"greedy": dict(do_sample=False), "sampling": dict(do_sample=True, temperature=0.6, top_k=50, top_p=0.9)}

    def run(n, kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        dec.generate(input_ids=ids, attention_mask=mask, max_new_tokens=n, eos_token_id=[], pad_token_id=0, **kw)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    n1, n2 = 8, 136
    for kw in modes.values():
        run(n1, kw); run(n2, kw)                                       # warm-up: tensor maps, allocator, graph pools
    res = {k: [] for k in modes}
    for _ in range(3):                                                 # alternate the two modes
        for name, kw in modes.items():
            res[name].append((run(n2, kw) - run(n1, kw)) / (n2 - n1))
    step = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    return {"model": "Llama-2-7b-hf shape, random bf16 weights", "batch": B, "prompt_len": L0,
            "ms_per_token_step": {k: round(v, 4) for k, v in step.items()},
            "all_ms_per_token_step": {k: [round(x, 4) for x in v] for k, v in res.items()},
            "sampling_overhead_pct": round(100 * (step["sampling"] / step["greedy"] - 1), 3)}


if __name__ == "__main__":
    out = {"card": card(), "kernels": kernels()}
    if "--skip-model" not in sys.argv:
        out["decode_step"] = model_step()
    print(json.dumps(out))
