"""Mistral-7B-shaped measurements on one GPU, on random weights, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * wgmma attention forward + backward at B 1, Hq 32 / Hkv 8, head_dim 128, L 4096 / 8192 / 16384: sliding window 4096
    (Mistral-7B-v0.1) against plain causal, alternated in one call, with the 64 x 64 KV tiles each visits (from the shapes);
  * the cfg-3-shaped LoRA training step with Mistral-7B-v0.1 as the generator: bge-large + Mistral-7B, LoRA on both, bs 18,
    lengths 50 / 128 / 256 (the window never applies at 256), the step replayed as one CUDA graph: samples/s and peak memory;
  * greedy decode tokens/s, prompt 256 + 256 new tokens at B = 8 and 64, next to transformers' `generate` on the same bf16
    weights; and prompt 4096 + 1024 new tokens at B = 8 with the window on and off.
    python tools/bench_mistral.py [--steps K] [--warmup W] [--skip-hf] [--skip-step]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_llama3 import lora_step  # noqa: E402
from bench_qwen2 import card, decode_rates, time_pair  # noqa: E402
from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.llama import LlamaDecoder  # noqa: E402

bf16 = torch.bfloat16
BQ = BKV = 64


def kv_tiles(L, window):
    """KV tiles the forward visits per (sample, head): for each 64-query tile, from the tile holding its first visible key
    (q0 - window + 1) to the diagonal"""
    n = 0
    for q0 in range(0, L, BQ):
        first = max(0, q0 - window + 1) // BKV if window else 0
        n += (min(L, q0 + BQ) - 1) // BKV - first + 1
    return n


def attention_sweep(dev, window=4096, Hq=32, Hkv=8, D=128):
    out = []
    for L in (4096, 8192, 16384):
        g = torch.Generator(device=dev).manual_seed(L)
        q = torch.randn(L, Hq * D, device=dev, generator=g).to(bf16)
        k = torch.randn(L, Hkv * D, device=dev, generator=g).to(bf16)
        v = torch.randn(L, Hkv * D, device=dev, generator=g).to(bf16)
        do = torch.randn(L, Hq * D, device=dev, generator=g).to(bf16)
        mask = torch.ones(1, L, dtype=torch.int64, device=dev)
        o, lse = ops.attention_tc_fwd(q, k, v, mask, 1, L, Hq, Hkv, D, True)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)

        def run(w):
            def f():
                ops.attention_tc_fwd(q, k, v, mask, 1, L, Hq, Hkv, D, True, out=o, window=w)
                ops.attention_tc_bwd(q, k, v, mask, o, lse, do, 1, L, Hq, Hkv, D, True, dq=dq, dk=dk, dv=dv, window=w)
            return f

        reps = max(5, 40 * 4096 // L)
        t_win, t_full = time_pair(run(window), run(0), reps=reps, rounds=5)
        tw, tf = kv_tiles(L, window), kv_tiles(L, 0)
        out.append({"L": L, "window": window, "fwd_bwd_us_window": t_win, "fwd_bwd_us_causal": t_full,
                    "time_ratio": t_win / t_full, "kv_tiles_window": tw, "kv_tiles_causal": tf, "tile_ratio": tw / tf})
        del q, k, v, do, o, lse, dq, dk, dv
    torch.cuda.empty_cache()
    return out


def hf_model(cfg, sd, dev):
    from transformers import MistralConfig, MistralForCausalLM
    from transformers.initialization import no_init_weights
    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
    with no_init_weights(), torch.device(dev):
        m = MistralForCausalLM(MistralConfig(**keep)).to(bf16)
    m.load_state_dict(sd, strict=True)
    m.generation_config.eos_token_id = None
    return m.eval()


def long_decode(dec, cfg, dev, B=8, L0=4096, new=1024):
    """prompt 4096 + 1024 new tokens with the checkpoint's window and with none (same weights, same kernels)"""
    res, own = {}, list(dec.windows)
    for tag, win in (("window", own), ("no_window", [0] * dec.nl)):
        dec.windows = win
        res[tag] = decode_rates(dec, None, cfg, dev, B, L0=L0, new=new)
        res[tag].pop("hf_tokens_per_s", None)
    dec.windows = own
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    ap.add_argument("--skip-step", action="store_true", help="leave out the training step")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mistral: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.init()
    torch.cuda.set_device(dev)
    cfg = synthetic.mistral_config("Mistral-7B-v0.1")
    res = {"what": "Mistral-7B-v0.1 shape, random weights", **card(), "torch": torch.__version__}
    res["attention_fwd_bwd"] = attention_sweep(dev)
    if not args.skip_step:
        res["cfg3_lora_step"] = lora_step(dev, cfg, args.steps, args.warmup)
        res["cfg3_lora_step"]["workload"] = "bge-large + Mistral-7B-v0.1, LoRA on both, bs 18, Lq 50 / Lp 128 / Lg 256, vocab 32000"
    sd = params.random_state_dict("mistral", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev)
    dec = LlamaDecoder(cfg, sd, device=dev)
    hf = None if args.skip_hf else hf_model(cfg, sd, dev)
    del sd
    torch.cuda.empty_cache()
    res["greedy_decode"] = [decode_rates(dec, hf, cfg, dev, B) for B in (8, 64)]
    del hf
    torch.cuda.empty_cache()
    res["greedy_decode_long"] = long_decode(dec, cfg, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
