"""ModernBERT-shaped measurements on one GPU, on random weights, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * the cfg-2-shaped retriever-only full fine-tuning step with Adam at the ModernBERT-base shape (gte-modernbert-base,
    modernbert-embed-base): bs 150, Lq 50 / Lp 128, a third of the rows padded, replayed as one CUDA graph: ms/step,
    samples/s and peak allocated memory; next to transformers' ModernBertModel (sdpa, bf16 autocast) with torch Adam on the
    same shapes; and the same step at bs 8 with Lp 2048 and 8192;
  * wgmma attention forward + backward at B 2, L 8192, 12 heads x 64: bidirectional window 65 (local_attention 128) against
    window 0, alternated, with the 64 x 64 KV tiles each visits, and the windowed output against fp32 on the visible keys;
  * geglu_fwd / geglu_bwd_ at the cfg-2 token count (150 x (50 + 128)) with F = 1152: us and bytes moved / us.
    python tools/bench_modernbert.py [--steps K] [--warmup W] [--skip-hf]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_qwen2 import card, time_pair  # noqa: E402
from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402

bf16, i64 = torch.bfloat16, torch.int64
BQ = BKV = 64


def kv_tiles(L, window):
    """KV tiles the forward visits per (sample, head): for each 64-query tile, from the tile holding q0 - window + 1 to the
    tile holding q0 + 63 + window - 1 (every tile without a window)"""
    n = 0
    for q0 in range(0, L, BQ):
        if window:
            first, last = max(0, q0 - window + 1) // BKV, (min(L, q0 + BQ - 1 + window) - 1) // BKV
        else:
            first, last = 0, (L - 1) // BKV
        n += last - first + 1
    return n


def batch(B, Lq, Lp, V, seed, dev):
    """[CLS] .. [SEP] rows, a third of them padded to ~60 % of their length"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for pre, L in (("query", Lq), ("passage", Lp)):
        ids = torch.randint(5, 50000, (B, L), generator=g)
        mask = torch.ones(B, L, dtype=i64)
        for b in range(0, B, 3):
            n = max(2, int(L * 0.6))
            mask[b, n:] = 0
            ids[b, n:] = 50283
        out[f"{pre}_input_ids"], out[f"{pre}_attention_mask"] = ids.to(dev), mask.to(dev)
    return out


def ours_step(dev, cfg, B, Lq, Lp, steps, warmup):
    from dalm_b200.engine.modernbert import ModernBertEncoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_retriever_step
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    sd = params.random_state_dict("modernbert", dict(cfg, _device_rng=True), seed=1, dtype=torch.float32, device=dev)
    enc = ModernBertEncoder(cfg, sd, device=dev, full=True)
    del sd
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    opt = FusedAdam(se.parameters(), lr=1e-5)
    b = batch(B, Lq, Lp, cfg["vocab_size"], 3, dev)
    step = GraphedStep(fused_retriever_step, se, b, 100.0, zero_grads=enc.zero_grad_buffers)

    def one():
        opt.zero_grad()
        out = step(b)
        opt.step()
        return out
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = one()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"ms_per_step": round(ms, 3), "samples_per_s": round(B / ms * 1e3, 1),
           "peak_alloc_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), "loss": float(out["loss"].item())}
    del step, opt, se, enc
    return res


def hf_step(dev, cfg, B, Lq, Lp, steps, warmup):
    from transformers import ModernBertConfig, ModernBertModel
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    c = ModernBertConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")},
                         _attn_implementation="sdpa")
    m = ModernBertModel(c).to(dev).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-5)
    b = batch(B, Lq, Lp, cfg["vocab_size"], 3, dev)

    def emb(ids, mask):
        h = m(ids, mask)[0]
        mf = mask[..., None].float()
        return torch.nn.functional.normalize((h * mf).sum(1) / mf.sum(1).clamp(min=1e-9), dim=-1)

    def one():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=bf16):
            q, p = emb(b["query_input_ids"], b["query_attention_mask"]), emb(b["passage_input_ids"], b["passage_attention_mask"])
        s = 100.0 * q.float() @ p.float().t()
        lab = torch.arange(B, device=dev)
        loss = (torch.nn.functional.cross_entropy(s, lab) + torch.nn.functional.cross_entropy(s.t(), lab)) / 2
        loss.backward()
        opt.step()
        return loss
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        one()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"ms_per_step": round(ms, 3), "samples_per_s": round(B / ms * 1e3, 1),
           "peak_alloc_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    del m, opt
    return res


def attention(dev, B=2, L=8192, H=12, D=64, window=65):
    g = torch.Generator(device=dev).manual_seed(L)
    q, k, v, do = (torch.randn(B * L, H * D, device=dev, generator=g).to(bf16) for _ in range(4))
    mask = torch.ones(B, L, dtype=i64, device=dev)
    mask[1, L * 3 // 4:] = 0
    o, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, False)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)

    def run(w):
        def f():
            ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, False, out=o, window=w, bidirectional=True)
            ops.attention_tc_bwd(q, k, v, mask, o, lse, do, B, L, H, H, D, False, dq=dq, dk=dk, dv=dv, window=w,
                                 bidirectional=True)
        return f
    t_win, t_full = time_pair(run(window), run(0), reps=20, rounds=5)
    ow, _ = ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, False, window=window, bidirectional=True)
    rows = slice(0, 1024)                                        # sample 0, queries 0..1023, every head, against fp32
    qs, ks, vs = (t[:L].float().view(L, H, D).transpose(0, 1) for t in (q, k, v))
    i = torch.arange(L, device=dev)
    vis = (i[rows, None] - i[None, :]).abs() < window
    s = (qs[:, rows] @ ks.transpose(-1, -2) / D ** 0.5).masked_fill(~vis, float("-inf"))
    ref = (torch.softmax(s, -1) @ vs).transpose(0, 1).reshape(-1, H * D)
    got = ow[rows].float()
    return {"B": B, "L": L, "heads": H, "head_dim": D, "window": window, "fwd_bwd_us_window": round(t_win, 1),
            "fwd_bwd_us_full": round(t_full, 1), "speedup": round(t_full / t_win, 2),
            "kv_tiles_window": kv_tiles(L, window), "kv_tiles_full": kv_tiles(L, 0),
            "max_abs_err_vs_fp32": float((got - ref).abs().max()), "rel_err_vs_fp32": float((got - ref).norm() / ref.norm())}


def geglu(dev, M=150 * (50 + 128), F=1152):
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(M, 2 * F, device=dev, generator=g).to(bf16)
    x0 = x.clone()
    d = torch.randn(M, F, device=dev, generator=g).to(bf16)
    act = torch.empty(M, F, dtype=bf16, device=dev)
    t_f, t_b = time_pair(lambda: ops.geglu_fwd(x0, F, act=act), lambda: ops.geglu_bwd_(x, d, F), reps=200, rounds=5)
    bf, bb = M * (2 * F + F) * 2, M * (2 * F + F + 2 * F) * 2
    return {"M": M, "F": F, "fwd_us": round(t_f, 2), "bwd_us": round(t_b, 2),
            "fwd_GBps": round(bf / t_f / 1e3, 1), "bwd_GBps": round(bb / t_b / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-hf", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_modernbert needs a GPU")
    dev = torch.device("cuda", 0)
    cfg = synthetic.modernbert_config("ModernBERT-base")
    res = {"card": card(), "attention": attention(dev), "geglu": geglu(dev), "step": {}}
    for B, Lq, Lp in ((150, 50, 128), (8, 50, 2048), (8, 50, 8192)):
        key = f"bs{B}_Lq{Lq}_Lp{Lp}"
        r = {"dalm_b200": ours_step(dev, cfg, B, Lq, Lp, a.steps, a.warmup)}
        if not a.skip_hf:
            try:
                r["transformers_sdpa_torch_adam"] = hf_step(dev, cfg, B, Lq, Lp, max(3, a.steps // 2), 2)
            except torch.cuda.OutOfMemoryError:
                torch.cuda.empty_cache()
                r["transformers_sdpa_torch_adam"] = "out of memory"
        res["step"][key] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
