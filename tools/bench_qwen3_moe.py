"""Qwen3-30B-A3B-shaped measurements of the routed MLP on one GPU, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * the grouped wgmma GEMM at the 30B-A3B expert shapes (4 608 tokens, top-8 of 128 experts, random router logits): gate|up
    with the SwiGLU epilogue (N 1536, K 2048), down (N 2048, K 768) and both dgrads read from the same weights; us and TFLOP/s
    of the pairs' useful work (2 M k N K), next to a per-expert `ops.gemm` loop over the same padded segments (counts read
    back to the host first, as that loop needs) and to `torch._grouped_mm` on the unpadded rows where this torch build runs
    it, outputs compared;
  * the MoE layer's forward + backward (router GEMM, routing, experts, combine; backward to the layer input);
  * greedy decode tokens/s (prompt 256, 256 new tokens, no EOS) at B = 8 and 64 of the 30B-A3B shape cut to --layers
    layers (the full 48-layer model's random weights do not fit next to their packed copy), next to transformers' `generate`
    on the same weights for --hf-new tokens.
    python tools/bench_qwen3_moe.py [--layers 8] [--skip-hf] [--hf-new 32]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import moe, params  # noqa: E402
from tools.bench_qwen2 import card  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


def time_us(f, reps=50, rounds=5):
    """median over rounds of the per-call time (us), CUDA events"""
    for _ in range(5):
        f()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            f()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    return sorted(ts)[len(ts) // 2]


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def grouped_gemms(dev, cfg, M=4608):
    H, E, k, I = cfg["hidden_size"], cfg["num_experts"], cfg["num_experts_per_tok"], cfg["moe_intermediate_size"]
    g = torch.Generator(device=dev).manual_seed(0)
    ids, _ = ops.moe_router(torch.randn(M, E, device=dev, generator=g), k, True)
    r = ops.moe_permute(ids, E)
    x = (torch.randn(r.rows, H, device=dev, generator=g)).to(bf16)
    w_gu = (torch.randn(E, 2 * I, H, device=dev, generator=g) * H ** -0.5).to(bf16)
    w_d = (torch.randn(E, H, I, device=dev, generator=g) * I ** -0.5).to(bf16)
    act = (torch.randn(r.rows, I, device=dev, generator=g)).to(bf16)
    dy = (torch.randn(r.rows, H, device=dev, generator=g)).to(bf16)
    dgu = (torch.randn(r.rows, 2 * I, device=dev, generator=g)).to(bf16)
    counts, off = r.counts.cpu().tolist(), r.seg_off.cpu().tolist()
    P = M * k
    # (name, grouped call, per-expert call, useful flops, torch._grouped_mm call or None)
    gu_out, act_out = torch.empty(r.rows, 2 * I, dtype=bf16, device=dev), torch.empty(r.rows, I, dtype=bf16, device=dev)
    cases = [
        ("gate_up_swiglu", 2 * I, H,
         lambda: ops.gemm_grouped(x, w_gu, r.tile_expert, r.live, out=gu_out, swiglu=True, act=act_out),
         lambda e, s: ops.gemm_swiglu(x[s], w_gu[e], gu=gu_out[s], act=act_out[s]), gu_out, (x, w_gu, True)),
        ("down", H, I, lambda: ops.gemm_grouped(act, w_d, r.tile_expert, r.live, out=dy),
         lambda e, s: ops.gemm(act[s], w_d[e], out=dy[s]), dy, (act, w_d, True)),
        ("down_dgrad", I, H, lambda: ops.gemm_grouped(dy, w_d, r.tile_expert, r.live, layout=1, out=act),
         lambda e, s: ops.gemm(dy[s], w_d[e], out=act[s], layout=1), act, (dy, w_d, False)),
        ("gate_up_dgrad", H, 2 * I, lambda: ops.gemm_grouped(dgu, w_gu, r.tile_expert, r.live, layout=1, out=x),
         lambda e, s: ops.gemm(dgu[s], w_gu[e], out=x[s], layout=1), x, (dgu, w_gu, False)),
    ]
    live_rows = [slice(off[e], off[e] + counts[e]) for e in range(E)]
    pad_rows = [slice(off[e], off[e + 1]) for e in range(E)]
    res = {"tokens": M, "top_k": k, "experts": E, "hidden": H, "moe_intermediate": I, "padded_rows": off[-1], "pairs": P}
    for name, N, K, grouped, per_expert, out, (a, w, tn) in cases:
        flops = 2.0 * P * N * K
        t = time_us(grouped)
        grouped()
        want = out.clone()
        loop = lambda: [per_expert(e, pad_rows[e]) for e in range(E) if counts[e]]
        t_loop = time_us(loop, reps=10)
        loop()
        row = {"N": N, "K": K, "grouped_us": t, "grouped_tflops": flops / t / 1e6, "per_expert_loop_us": t_loop,
               "per_expert_loop_tflops": flops / t_loop / 1e6,
               "loop_vs_grouped_rel": max(rel(out[s], want[s]) for s in live_rows if s.stop > s.start)}
        if name != "gate_up_swiglu" and hasattr(torch, "_grouped_mm"):
            # unpadded rows: the live rows of each segment, packed; offs = cumulative segment ends
            sel = torch.cat([torch.arange(s.start, s.stop, device=dev) for s in live_rows])
            offs = torch.tensor(counts, device=dev).cumsum(0).to(torch.int32)
            b = w.transpose(1, 2) if tn else w                                       # [E, K, N]
            try:
                a_packed = a[sel].contiguous()
                f = lambda: torch._grouped_mm(a_packed, b, offs=offs)
                t_g = time_us(f)
                row.update(torch_grouped_mm_us=t_g, torch_grouped_mm_tflops=flops / t_g / 1e6,
                           torch_grouped_mm_vs_grouped_rel=rel(f(), want[sel]))
            except Exception as exc:                                                 # noqa: BLE001 - report, do not guess
                row["torch_grouped_mm"] = f"not run: {type(exc).__name__}: {str(exc)[:160]}"
        res[name] = row
    return res


def layer_fwd_bwd(dev, cfg, M=4608):
    H, E, k, I = cfg["hidden_size"], cfg["num_experts"], cfg["num_experts_per_tok"], cfg["moe_intermediate_size"]
    g = torch.Generator(device=dev).manual_seed(1)
    mw = moe.MoeWeights((torch.randn(E, H, device=dev, generator=g) * 0.02).to(bf16),
                        (torch.randn(E, 2 * I, H, device=dev, generator=g) * 0.02).to(bf16),
                        (torch.randn(E, H, I, device=dev, generator=g) * 0.02).to(bf16), k, True)
    x = torch.randn(M, H, device=dev, generator=g).to(bf16)
    resid = torch.randn(M, H, device=dev, generator=g)
    dy = torch.randn(M, H, device=dev, generator=g)
    fwd = lambda: moe.forward(x, mw, resid=resid)
    saved = {}

    def both():
        out, s = moe.forward(x, mw, resid=resid)
        saved["dx"] = moe.backward(dy, s, mw)
    return {"tokens": M, "forward_us": time_us(fwd, reps=20), "forward_backward_us": time_us(both, reps=20)}


def decode(dev, cfg, layers, skip_hf, hf_new):
    cfg = dict(cfg, num_hidden_layers=layers)
    sd = params.random_state_dict("qwen3_moe", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev, router_std=0.5)
    from dalm_b200.engine.llama import LlamaDecoder
    dec = LlamaDecoder(cfg, sd, device=dev)
    hf = None
    if not skip_hf:
        from transformers import Qwen3MoeConfig, Qwen3MoeForCausalLM
        from transformers.initialization import no_init_weights
        keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
        with no_init_weights(), torch.device(dev):
            hf = Qwen3MoeForCausalLM(Qwen3MoeConfig(**keep)).to(bf16)
        E = cfg["num_experts"]
        for l in range(layers):
            p = f"model.layers.{l}.mlp.experts."
            ex = lambda e, n: sd.pop(p + f"{e}.{n}_proj.weight")
            gu = torch.stack([torch.cat([ex(e, "gate"), ex(e, "up")]) for e in range(E)])
            dn = torch.stack([ex(e, "down") for e in range(E)])
            sd[p + "gate_up_proj"], sd[p + "down_proj"] = gu, dn
        missing, unexpected = hf.load_state_dict(sd, strict=False)
        assert not unexpected and not missing, (missing, unexpected)
        hf.eval()
    del sd
    torch.cuda.empty_cache()
    rows = []
    for B in (8, 64):
        gen = torch.Generator().manual_seed(B)
        ids = torch.randint(3, cfg["vocab_size"], (B, 256), generator=gen).to(dev)
        mask = torch.ones_like(ids)

        def run(f, new):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = f(new)
            e1.record()
            torch.cuda.synchronize()
            assert out.shape == (B, 256 + new), out.shape
            return e0.elapsed_time(e1) / 1e3

        ours = lambda new: dec.generate(input_ids=ids, attention_mask=mask, max_new_tokens=new, eos_token_id=[], pad_token_id=0)
        ours(8)
        s = run(ours, 256)
        row = {"B": B, "prompt": 256, "new_tokens": 256, "dalm_s": s, "dalm_tokens_per_s": B * 256 / s}
        if hf is not None:
            with torch.no_grad():
                theirs = lambda new: hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=new, min_new_tokens=new,
                                                 do_sample=False, pad_token_id=0, eos_token_id=None)
                theirs(2)
                h = run(theirs, hf_new)
            row.update(hf_new_tokens=hf_new, hf_s=h, hf_tokens_per_s=B * hf_new / h)
        else:
            row["hf_tokens_per_s"] = "not measured"
        rows.append(row)
    return {"layers": layers, "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8, help="decoder layers of the 30B-A3B shape built for the decode rates")
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--hf-new", type=int, default=32, help="new tokens of transformers' generate (its expert loop is slow)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qwen3_moe: needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = synthetic.qwen3_moe_config("qwen3-30b-a3b")
    res = {"what": "Qwen3-30B-A3B shape, random weights", **card(), "torch": torch.__version__}
    res["grouped_gemm"] = grouped_gemms(dev, cfg)
    res["moe_layer"] = layer_fwd_bwd(dev, cfg)
    if not args.skip_decode:
        res["greedy_decode"] = decode(dev, cfg, args.layers, args.skip_hf, args.hf_new)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
