"""Qwen2.5-7B-shaped measurements on one GPU, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * `gemm_rope` (training QKV + RoPE, M = 18 x 256 rows) and `decode_gemm` (B = 8 rows) at the 7B q|k|v shape [4608, 3584],
    bias=None against bias, alternated, CUDA events;
  * greedy decode tokens/s (prompt 256, 256 new tokens, no EOS) at B = 8 (decode_gemm path) and B = 64 (wgmma path), next to
    transformers' `generate` on the same random bf16 weights on the same GPU.
The cfg-3-shaped LoRA training step is not part of this script; its entry says so.
    python tools/bench_qwen2.py [--skip-hf]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.llama import LlamaDecoder  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else (torch.cuda.get_device_name(), "unknown", "unknown")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def time_pair(fa, fb, reps=200, rounds=5):
    """median over `rounds` of the per-call time of fa and fb, alternated round by round (us)"""
    res = {"a": [], "b": []}
    for f in (fa, fb):
        for _ in range(10):
            f()
    for _ in range(rounds):
        for key, f in (("a", fa), ("b", fb)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                f()
            e1.record()
            torch.cuda.synchronize()
            res[key].append(e0.elapsed_time(e1) * 1e3 / reps)
    med = lambda v: sorted(v)[len(v) // 2]
    return med(res["a"]), med(res["b"])


def kernel_bias_cost(dev, cfg):
    H, hd = cfg["hidden_size"], cfg["hidden_size"] // cfg["num_attention_heads"]
    nq, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
    N = (nq + 2 * nkv) * hd
    g = torch.Generator(device=dev).manual_seed(0)
    w = (torch.randn(N, H, device=dev, generator=g) * 0.02).to(bf16)
    bias = torch.randn(N, device=dev, generator=g) * 0.5
    L = 256
    a = torch.randn(18 * L, H, device=dev, generator=g).to(bf16)
    inv = 1.0 / (1e6 ** (torch.arange(0, 128, 2, dtype=f32, device=dev) / 128))
    fr = torch.outer(torch.arange(L, dtype=f32, device=dev), inv)
    cos_t, sin_t = fr.cos().contiguous(), fr.sin().contiguous()
    out = torch.empty(18 * L, N, dtype=bf16, device=dev)
    rc = (nq + nkv) * hd
    t0, t1 = time_pair(lambda: ops.gemm_rope(a, w, cos_t, sin_t, L, rc, out=out),
                       lambda: ops.gemm_rope(a, w, cos_t, sin_t, L, rc, out=out, bias=bias))
    a8 = torch.randn(8, H, device=dev, generator=g).to(bf16)
    o8 = torch.empty(8, N, dtype=bf16, device=dev)
    d0, d1 = time_pair(lambda: ops.decode_gemm(a8, w, out=o8), lambda: ops.decode_gemm(a8, w, out=o8, bias=bias))
    return {"shape_NxK": [N, H], "gemm_rope_M": 18 * L, "gemm_rope_us": {"no_bias": t0, "bias": t1},
            "decode_gemm_M": 8, "decode_gemm_us": {"no_bias": d0, "bias": d1}}


def hf_model(cfg, sd, dev):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    from transformers.initialization import no_init_weights
    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
    with no_init_weights(), torch.device(dev):
        m = Qwen2ForCausalLM(Qwen2Config(**keep)).to(bf16)
    m.load_state_dict(sd, strict=False)
    return m.eval()


def decode_rates(dec, hf, cfg, dev, B, L0=256, new=256):
    g = torch.Generator().manual_seed(B)
    ids = torch.randint(3, cfg["vocab_size"], (B, L0), generator=g).to(dev)
    mask = torch.ones_like(ids)

    def run(f):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = f()
        e1.record()
        torch.cuda.synchronize()
        assert out.shape == (B, L0 + new), out.shape
        return e0.elapsed_time(e1) / 1e3

    ours = lambda: dec.generate(input_ids=ids, attention_mask=mask, max_new_tokens=new, eos_token_id=[], pad_token_id=0)
    dec.generate(input_ids=ids, attention_mask=mask, max_new_tokens=8, eos_token_id=[], pad_token_id=0)   # warm-up
    s = run(ours)
    res = {"B": B, "prompt": L0, "new_tokens": new, "dalm_s": s, "dalm_tokens_per_s": B * new / s}
    if hf is not None:
        with torch.no_grad():
            theirs = lambda: hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=new, min_new_tokens=new,
                                         do_sample=False, pad_token_id=0, eos_token_id=None)
            hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=8, do_sample=False, pad_token_id=0)
            h = run(theirs)
        res.update(hf_s=h, hf_tokens_per_s=B * new / h)
    else:
        res.update(hf_tokens_per_s="not measured")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qwen2: needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = synthetic.qwen2_config("qwen2.5-7b")
    res = {"what": "Qwen2.5-7B shape", **card(), "torch": torch.__version__}
    res["bias_cost"] = kernel_bias_cost(dev, cfg)
    sd = params.random_state_dict("qwen2", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev)
    dec = LlamaDecoder(cfg, sd, device=dev)
    hf = None if args.skip_hf else hf_model(cfg, sd, dev)
    del sd
    torch.cuda.empty_cache()
    res["greedy_decode"] = [decode_rates(dec, hf, cfg, dev, B) for B in (8, 64)]
    res["cfg3_lora_step"] = "not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
