"""XLM-RoBERTa (bge-m3-shaped) retriever measurements on one GPU, on random weights, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * the cfg-2-shaped retriever-only LoRA step (bs 150, Lq 50, Lp 128, uniform random ids, about a third of each row padded
    with <pad> = 1) with the bge-m3 shape against the bge-large-en shape, both replayed as one CUDA graph with Adam and the
    LoRA repack after it, alternated in rounds in this one process. The GEMM shapes are identical (24 x 1024, FFN 4096), so
    the gap is the embedding kernel and the 250 002-row word table;
  * roberta_embed + the padding-aware scatter against bert_embed + embed_scatter_add at that step's M = 150 x (50 + 128),
    CUDA events over many launches;
  * peak allocated memory of a fully fine-tuned bge-m3 retriever-only step (bs 150, Lq 50 / Lp 128, eager, one Adam step);
  * the bge-m3 LoRA retriever-only step at bs 8 with Lq 50 and Lp 2048 / 8192 (the longest bge-m3 serves).
    python tools/bench_roberta.py [--steps K] [--warmup W] [--rounds R]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from bench_qwen2 import card  # noqa: E402
from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.bert import BertEncoder  # noqa: E402

bf16 = torch.bfloat16
BS, LQ, LP = 150, 50, 128


def batches(n, B, Lq, Lp, V, pad, seed=0):
    """random ids; row b keeps its first L - (b % 3) * L // 6 tokens and pads the rest (pad id, mask 0)"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        b = {}
        for key, L in (("query", Lq), ("passage", Lp)):
            ids = torch.randint(5, V, (B, L), generator=g)
            mask = torch.ones(B, L, dtype=torch.int64)
            for r in range(B):
                n_keep = L - (r % 3) * L // 6
                ids[r, n_keep:], mask[r, n_keep:] = pad, 0
            b[key + "_input_ids"], b[key + "_attention_mask"] = ids, mask
        out.append(b)
    return out


def encoder(kind, name, dev, **kw):
    cfg = synthetic.roberta_config(name) if kind == "roberta" else synthetic.bert_config(name)
    cfg = dict(cfg, _device_rng=True)
    return cfg, BertEncoder(cfg, params.random_state_dict(kind, cfg, seed=0, dtype=bf16, device=dev), device=dev, **kw)


class LoraStep:
    """one encoder's retriever-only LoRA step, graphed, with Adam and the repack after it"""

    def __init__(self, kind, name, dev, B, Lq, Lp):
        from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
        from dalm_b200.optim import FusedAdam
        from dalm_b200.training.utils.train_utils import GraphedStep, fused_retriever_step
        cfg, self.enc = encoder(kind, name, dev, lora=True)
        self.se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, _model=self.enc, _load_tokenizer=False)
        self.se.train()
        self.opt = FusedAdam(self.se.parameters(), lr=1e-4)
        self.batches = [{k: v.to(dev) for k, v in b.items()}
                        for b in batches(4, B, Lq, Lp, cfg["vocab_size"], cfg.get("pad_token_id", 0))]
        self.graphed = GraphedStep(fused_retriever_step, self.se, self.batches[0], 100.0, zero_grads=self.opt.zero_grad)
        self.i = 0

    def step(self):
        out = self.graphed(self.batches[self.i % len(self.batches)])
        self.opt.step()
        self.enc.repack_lora()
        self.opt.zero_grad()
        self.i += 1
        return out["loss"]

    def time(self, steps, warmup):
        for _ in range(warmup):
            self.step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = self.step()
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(loss).item()
        return e0.elapsed_time(e1) / steps


def alternated(dev, steps, warmup, rounds):
    runs = {"bge-m3": LoraStep("roberta", "bge-m3", dev, BS, LQ, LP), "bge-large-en": LoraStep("bert", "bge-large-en", dev, BS, LQ, LP)}
    ms = {k: [] for k in runs}
    for _ in range(rounds):
        for k, r in runs.items():
            ms[k].append(r.time(steps, warmup))
    del runs
    torch.cuda.empty_cache()
    res = {"workload": f"retriever-only LoRA step, bs {BS}, Lq {LQ} / Lp {LP}, graphed, Adam + repack", "steps": steps,
           "warmup": warmup, "rounds": rounds}
    for k, v in ms.items():
        res[k] = {"ms_per_step_each_round": [round(x, 3) for x in v], "samples_per_s_best": BS * 1e3 / min(v)}
    return res


def embed_kernels(dev, iters=200):
    """forward embedding + backward scatter (word and position tables) at the cfg-2 step's M, for both families"""
    H, M = 1024, BS * (LQ + LP)
    g = torch.Generator(device=dev).manual_seed(0)
    out = {"M": M, "H": H, "iters": iters}
    for kind, V, P, pad in (("roberta", 250002, 514, 1), ("bert", 30522, 512, 0)):
        word = torch.randn(V, H, generator=g, device=dev).to(bf16)
        pos = torch.randn(P, H, generator=g, device=dev).to(bf16)
        typ = torch.randn(H, generator=g, device=dev).to(bf16)
        b = batches(1, BS, LQ, LP, V, pad)[0]
        segs, r0 = [], 0                                   # the query and the passage segment, as the engine launches them
        for key in ("query", "passage"):
            ids = b[key + "_input_ids"].to(dev)
            n = ids.numel()
            segs.append((ids, ids.view(-1), slice(r0, r0 + n), ids.shape[1]))
            r0 += n
        z = torch.empty(M, H, device=dev)
        pid = torch.empty(M, dtype=torch.int64, device=dev)
        dw, dp = torch.zeros(V, H, device=dev), torch.zeros(P, H, device=dev)

        def run():
            for ids, flat, rows, L in segs:
                if kind == "roberta":
                    ops.roberta_embed(ids, word, pos, typ, pad, out=z[rows], pos_ids=pid[rows])
                    ops.embed_scatter_add_(z[rows], flat, dw, dp, L, pos_ids=pid[rows], pad_id=pad)
                else:
                    ops.bert_embed(ids, word, pos, typ, out=z[rows])
                    ops.embed_scatter_add_(z[rows], flat, dw, dp, L)
        for _ in range(10):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            run()
        e1.record()
        torch.cuda.synchronize()
        out[("roberta_embed + scatter(pos_ids, pad_id)" if kind == "roberta" else "bert_embed + embed_scatter_add") + " us"] = \
            e0.elapsed_time(e1) * 1e3 / iters
        del word, pos, dw, dp, z
        torch.cuda.empty_cache()
    return out


def full_ft_peak(dev):
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    cfg, enc = encoder("roberta", "bge-m3", dev, full=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    se.train()
    opt = FusedAdam(se.parameters(), lr=1e-5)
    b = {k: v.to(dev) for k, v in batches(1, BS, LQ, LP, cfg["vocab_size"], 1)[0].items()}
    opt.zero_grad()
    loss = fused_retriever_step(se, b, 100.0)["loss"]
    opt.step()
    torch.cuda.synchronize()
    res = {"workload": f"bge-m3 fully fine-tuned, retriever-only step + Adam, bs {BS}, Lq {LQ} / Lp {LP}",
           "peak_memory_GiB": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "loss_finite": bool(torch.isfinite(loss).item())}
    del se, enc, opt
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_roberta: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.init()
    torch.cuda.set_device(dev)
    res = {"what": "bge-m3 shape (XLM-RoBERTa) vs bge-large-en shape (BERT), random weights", **card(), "torch": torch.__version__}
    res["cfg2_lora_step"] = alternated(dev, args.steps, args.warmup, args.rounds)
    res["embedding_kernels"] = embed_kernels(dev)
    res["full_ft_peak"] = full_ft_peak(dev)
    res["long_passages"] = []
    for Lp in (2048, 8192):
        try:
            r = LoraStep("roberta", "bge-m3", dev, 8, LQ, Lp)
            ms = r.time(args.steps, args.warmup)
            res["long_passages"].append({"bs": 8, "Lq": LQ, "Lp": Lp, "ms_per_step": ms, "samples_per_s": 8e3 / ms})
            del r
        except torch.cuda.OutOfMemoryError as e:
            res["long_passages"].append({"bs": 8, "Lq": LQ, "Lp": Lp, "error": f"out of memory: {str(e)[:200]}"})
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
