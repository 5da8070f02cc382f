"""Llama-3.1-8B-shaped measurements on one GPU, on random weights, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * the cfg-3-shaped LoRA training step with Llama-3.1-8B as the generator: bge-large + Llama-3.1-8B, LoRA on both, bs 18,
    query / passage / generator lengths 50 / 128 / 256, vocab 128256, uniform random token ids with all-ones masks, the step
    replayed as one CUDA graph with Adam and the LoRA repack after it (as bench.py runs cfg-3): samples/s and peak memory;
  * greedy decode tokens/s (prompt 256, 256 new tokens, no EOS) at B = 8 (decode_gemm path) and B = 64 (wgmma path), next to
    transformers' `generate` on the same random bf16 weights on the same GPU.
    python tools/bench_llama3.py [--steps K] [--warmup W] [--skip-hf]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_qwen2 import card, decode_rates  # noqa: E402
from dalm_b200 import synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.llama import LlamaDecoder  # noqa: E402

bf16 = torch.bfloat16
BS, LQ, LP, LG = 18, 50, 128, 256


def random_batches(n, V, seed=0):
    g = torch.Generator().manual_seed(seed)
    rnd = lambda L, v: torch.randint(5, v, (BS, L), generator=g)
    ones = lambda L: torch.ones(BS, L, dtype=torch.int64)
    return [{"retriever_query_input_ids": rnd(LQ, 30522), "retriever_query_attention_mask": ones(LQ),
             "retriever_passage_input_ids": rnd(LP, 30522), "retriever_passage_attention_mask": ones(LP),
             "generator_input_input_ids": rnd(LG, V), "generator_input_attention_mask": ones(LG),
             "query_passage_input_len": torch.full((BS,), LG // 2)} for _ in range(n)]


def lora_step(dev, gcfg, steps, warmup):
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_rag_step
    torch.zeros(1, device=dev)                               # the caching allocator exists before its statistics are reset
    torch.cuda.reset_peak_memory_stats()
    bcfg = dict(synthetic.bert_config("bge-large-en"), _device_rng=True)
    enc = BertEncoder(bcfg, params.random_state_dict("bert", bcfg, seed=0, dtype=bf16, device=dev), device=dev, lora=True)
    lcfg = dict(gcfg, _device_rng=True)
    dec = LlamaDecoder(lcfg, params.random_state_dict("llama", lcfg, seed=0, dtype=bf16, device=dev), device=dev, lora=True)
    torch.cuda.empty_cache()
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH, _retriever=enc, _generator=dec, _load_tokenizers=False)
    opt = FusedAdam(model.parameters(), lr=1e-4)
    model.train()
    batches = [{k: v.to(dev) for k, v in b.items()} for b in random_batches(4, gcfg["vocab_size"])]
    graphed = GraphedStep(fused_rag_step, model, batches[0], 100.0, zero_grads=opt.zero_grad)

    def step(i):
        out = graphed(batches[i % len(batches)])
        opt.step()
        model.repack()
        opt.zero_grad()
        return out["loss"]

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = step(i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"workload": "bge-large + Llama-3.1-8B, LoRA on both, bs 18, Lq 50 / Lp 128 / Lg 256, vocab 128256",
           "steps": steps, "warmup": warmup, "ms_per_step": ms, "samples_per_s": BS * 1e3 / ms,
           "peak_memory_GiB": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "loss_finite": bool(torch.isfinite(loss).item())}
    del graphed, model, enc, dec, opt, batches
    torch.cuda.empty_cache()
    return res


def hf_model(cfg, sd, dev):
    from transformers import LlamaConfig, LlamaForCausalLM
    from transformers.initialization import no_init_weights
    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
    with no_init_weights(), torch.device(dev):
        m = LlamaForCausalLM(LlamaConfig(**keep)).to(bf16)
    m.load_state_dict(sd, strict=False)
    m.generation_config.eos_token_id = None
    assert m.config.rope_parameters["rope_type"] == "llama3"
    return m.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_llama3: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.init()
    torch.cuda.set_device(dev)
    cfg = synthetic.llama3_config("llama-3.1-8b")
    res = {"what": "Llama-3.1-8B shape, random weights", **card(), "torch": torch.__version__}
    res["cfg3_lora_step"] = lora_step(dev, cfg, args.steps, args.warmup)
    sd = params.random_state_dict("llama", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev)
    dec = LlamaDecoder(cfg, sd, device=dev)
    hf = None if args.skip_hf else hf_model(cfg, sd, dev)
    del sd
    torch.cuda.empty_cache()
    res["greedy_decode"] = [decode_rates(dec, hf, cfg, dev, B) for B in (8, 64)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
