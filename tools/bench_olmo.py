"""OLMo-2-1124-7B / OLMoE-1B-7B-shaped measurements on one GPU, on random weights, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * the new row kernels at the cfg-3 token count (bs 18 x 256 = 4 608 rows) and the OLMo-2-7B widths (q 4096, k 4096,
    hidden 4096): qk_fullnorm_rope forward (saving pre-norm columns and rstd) and backward, the deterministic norm weight
    gradient, postnorm forward and backward; us and the bytes each must move over that time. The post-norm backward is timed
    next to the alternative of an fp32 o_proj / down output fed to the existing rmsnorm_bwd (with the cast of the residual
    gradient to bf16 that it needs), with the saved activation bytes of each;
  * the cfg-3-shaped LoRA training step with OLMo-2-1124-7B as the generator (bge-large + OLMo-2-7B, LoRA on both, bs 18,
    lengths 50 / 128 / 256): samples/s and peak memory, eager and replayed as one CUDA graph;
  * one OLMoE-1B-7B layer (attention + routed MLP) forward and forward + backward at 4 608 tokens;
  * greedy decode tokens/s (prompt 256, 256 new tokens, no EOS) at B = 8 and 64 of OLMo-2-7B, next to transformers'
    `generate` on the same bf16 weights.
    python tools/bench_olmo.py [--steps K] [--warmup W] [--skip-hf] [--skip-step] [--skip-decode]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_llama3 import BS, random_batches  # noqa: E402
from bench_qwen2 import card, decode_rates  # noqa: E402
from bench_qwen3_moe import time_us  # noqa: E402
from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.llama import LlamaDecoder  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32
M = BS * 256


def kernels(dev, cfg):
    H, nh, nkv = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"]
    hd = H // nh
    Nq, Nk = nh * hd, nkv * hd
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(M, Nq + 2 * Nk, device=dev, generator=g).to(bf16)
    wq, wk = 1 + 0.1 * torch.randn(Nq, device=dev, generator=g), 1 + 0.1 * torch.randn(Nk, device=dev, generator=g)
    inv = params.rope_inv_freq(cfg, hd)
    fr = torch.outer(torch.arange(256, dtype=f32), inv)
    cos_t, sin_t = fr.cos().to(dev).contiguous(), fr.sin().to(dev).contiguous()
    pre, rstd = torch.empty(M, Nq + Nk, dtype=bf16, device=dev), torch.empty(M, 2, device=dev)
    work = qkv.clone()
    W = Nq + Nk
    res = {"rows": M, "q_cols": Nq, "k_cols": Nk}
    fwd = lambda: ops.qk_fullnorm_rope_(work, nh, nkv, hd, wq, wk, 1e-6, cos_t, sin_t, L=256, pre=pre, rstd=rstd)
    t = time_us(fwd)
    b = M * W * 2 * 3 + M * 8                                   # read q|k, write q|k, write pre; rstd
    res["qk_fullnorm_rope_fwd"] = {"us": t, "bytes": b, "GB_per_s": b / t / 1e3}
    d = qkv.clone()
    bwd = lambda: ops.qk_fullnorm_rope_bwd_(d, nh, nkv, hd, wq, wk, cos_t, sin_t, 256, pre, rstd)
    t = time_us(bwd)
    b = M * W * 2 * 3 + M * 8                                   # read d(q|k), pre; write d(q|k)
    res["qk_fullnorm_rope_bwd"] = {"us": t, "bytes": b, "GB_per_s": b / t / 1e3}
    dwq, dwk = torch.zeros(Nq, device=dev), torch.zeros(Nk, device=dev)
    wg = lambda: ops.norm_wgrad_(d[:, :W], pre, rstd, dwq, dwk, hd=hd, cos_t=cos_t, sin_t=sin_t, L=256)
    t = time_us(wg)
    b = M * W * 2 * 2
    res["qk_norm_wgrad"] = {"us": t, "bytes": b, "GB_per_s": b / t / 1e3}
    y = torch.randn(M, H, device=dev, generator=g).to(bf16)
    w = 1 + 0.1 * torch.randn(H, device=dev, generator=g)
    resid = torch.randn(M, H, device=dev, generator=g)
    h16 = torch.empty(M, H, dtype=bf16, device=dev)
    t = time_us(lambda: ops.postnorm_fwd(y, w, resid, 1e-6, out16=h16))
    b = M * H * (2 + 4 + 4 + 2)
    res["postnorm_fwd"] = {"us": t, "bytes": b, "GB_per_s": b / t / 1e3}
    _, r = ops.postnorm_fwd(y, w, resid, 1e-6)
    dres, dh = torch.randn(M, H, device=dev, generator=g), torch.randn(M, H, device=dev, generator=g).to(bf16)
    t = time_us(lambda: ops.postnorm_bwd(y, w, r, dres, dh=dh))
    b = M * H * (2 + 4 + 2 + 4 + 2)
    res["postnorm_bwd"] = {"us": t, "bytes": b, "GB_per_s": b / t / 1e3, "saved_y_bytes_per_sublayer": M * H * 2}
    # the alternative: an fp32 y saved by the GEMM, the residual gradient (+ the branch gradient) cast to bf16 for rmsnorm_bwd
    y32 = y.float()

    def alt():
        dsum = ops.masked_add(a=dres, b=dh)
        ops.rmsnorm_bwd(y32, w, r, ops.cast_f32_bf16(dsum))
    t = time_us(alt)
    res["alt_fp32_y_rmsnorm_bwd"] = {"us": t, "saved_y_bytes_per_sublayer": M * H * 4,
                                     "what": "masked_add + cast_f32_bf16 + rmsnorm_bwd on an fp32 y"}
    return res


def _olmo_decoder(dev, cfg, kind, lora):
    c = dict(cfg, _device_rng=True)
    return LlamaDecoder(c, params.random_state_dict(kind, c, seed=0, dtype=bf16, device=dev, router_std=0.5), device=dev, lora=lora)


def lora_step(dev, gcfg, steps, warmup):
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_rag_step
    torch.zeros(1, device=dev)
    torch.cuda.reset_peak_memory_stats()
    bcfg = dict(synthetic.bert_config("bge-large-en"), _device_rng=True)
    enc = BertEncoder(bcfg, params.random_state_dict("bert", bcfg, seed=0, dtype=bf16, device=dev), device=dev, lora=True)
    dec = _olmo_decoder(dev, gcfg, "olmo2", True)
    torch.cuda.empty_cache()
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH, _retriever=enc, _generator=dec, _load_tokenizers=False)
    opt = FusedAdam(model.parameters(), lr=1e-4)
    model.train()
    batches = [{k: v.to(dev) for k, v in b.items()} for b in random_batches(4, gcfg["vocab_size"])]
    res = {"workload": "bge-large + OLMo-2-1124-7B, LoRA on both, bs 18, Lq 50 / Lp 128 / Lg 256, vocab 100352"}
    for mode in ("eager", "graph"):
        torch.cuda.reset_peak_memory_stats()
        run = GraphedStep(fused_rag_step, model, batches[0], 100.0, zero_grads=opt.zero_grad) if mode == "graph" else \
            (lambda b: fused_rag_step(model, b, 100.0))

        def step(i):
            out = run(batches[i % len(batches)])
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
        res[mode] = {"steps": steps, "warmup": warmup, "ms_per_step": ms, "samples_per_s": BS * 1e3 / ms,
                     "peak_memory_GiB": torch.cuda.max_memory_allocated(dev) / 2 ** 30,
                     "loss_finite": bool(torch.isfinite(loss).item())}
        del run
    del model, enc, dec, opt, batches
    torch.cuda.empty_cache()
    return res


def olmoe_layer(dev, cfg):
    """one OLMoE-1B-7B decoder layer (a one-layer model's body: embedding gather, attention, routed MLP, final norm)"""
    c = dict(cfg, num_hidden_layers=1)
    dec = _olmo_decoder(dev, c, "olmoe", True)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(3, c["vocab_size"], (BS, 256), generator=g).to(dev)
    mask = torch.ones_like(ids)
    dhf = torch.randn(M, c["hidden_size"], device=dev).to(bf16)
    fwd = lambda: dec.forward_final(ids, mask, save=False)

    def both():
        ctx = dec.forward_final(ids, mask)
        dec.backward_final(ctx, dhf)
    res = {"tokens": M, "forward_us": time_us(fwd, reps=10), "forward_backward_us": time_us(both, reps=10)}
    del dec
    torch.cuda.empty_cache()
    return res


def hf_model(cfg, sd, dev):
    from transformers import Olmo2Config, Olmo2ForCausalLM
    from transformers.initialization import no_init_weights
    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
    with no_init_weights(), torch.device(dev):
        m = Olmo2ForCausalLM(Olmo2Config(**keep)).to(bf16)
    m.load_state_dict(sd, strict=True)
    m.generation_config.eos_token_id = None
    return m.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    ap.add_argument("--skip-step", action="store_true", help="leave out the training step")
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_olmo: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = synthetic.olmo_config("olmo-2-1124-7b")
    res = {"what": "OLMo-2-1124-7B / OLMoE-1B-7B shapes, random weights", **card(), "torch": torch.__version__}
    res["kernels"] = kernels(dev, cfg)
    if not args.skip_step:
        res["cfg3_lora_step"] = lora_step(dev, cfg, args.steps, args.warmup)
    res["olmoe_layer"] = olmoe_layer(dev, synthetic.olmo_config("olmoe-1b-7b"))
    if not args.skip_decode:
        sd = params.random_state_dict("olmo2", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev)
        dec = LlamaDecoder(cfg, sd, device=dev)
        hf = None if args.skip_hf else hf_model(cfg, sd, dev)
        del sd
        torch.cuda.empty_cache()
        res["greedy_decode"] = [decode_rates(dec, hf, cfg, dev, B) for B in (8, 64)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
