"""Whole-model scaffolding shared by the GPU tests: bf16-rounded weights, LoRA factors shared with the transformers oracle,
the bge-tiny + decoder RAG pair, batches, and the checks that compare an engine with its oracle.

Every helper draws from the generator or seed it is given, so a test's inputs are fixed by its own arguments. The default
tolerances are the ones the model tests use (bf16 GEMM operands and activations through a few layers)."""
import csv as _csv
import json
import os
import shutil

import torch

bf16 = torch.bfloat16


def rel(a, b):
    """relative L2 error of a against b, in fp64 on b's device (large kernel outputs are not copied to the host)"""
    a, b = a.double().to(b.device), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def r16(sd):
    """every tensor rounded to bf16: the engine's bf16 weights and fp32 masters start equal to the oracle's fp32 weights"""
    return {k: v.to(bf16).float() for k, v in sd.items()}


def r16_2d(sd):
    """matrices rounded to bf16 (what the engine stores in bf16); vectors stay fp32"""
    return {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def pad_mask(B, L, pad):
    """right: row 0 ends in 5 pad tokens; left: rows 0 and 1 start with 5 and 2"""
    mask = torch.ones(B, L, dtype=torch.int64)
    if pad == "right":
        mask[0, L - 5:] = 0
    else:
        mask[0, :5] = 0; mask[1, :2] = 0
    return mask


def prompt(B, L0, V, seed, low=3):
    """generation prompts: ids in [low, V), row 1 left-padded by 3, row 2 right-padded by 3"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(low, V, (B, L0), generator=g)
    mask = torch.ones(B, L0, dtype=torch.int64)
    mask[1, :3] = 0
    mask[2, L0 - 3:] = 0
    return ids, mask


# ----------------------------------------------------------------------------------------------------------------
# LoRA
# ----------------------------------------------------------------------------------------------------------------
def draw_lora_B(engine, g):
    """non-zero B ~ N(0, 0.02) from g, so the LoRA path shows in the forward and dA is non-trivial"""
    for n, _, _ in engine.lora.specs:
        engine.lora.B[n].copy_((torch.randn(engine.lora.B[n].shape, generator=g) * 0.02).to(engine.dev))
    engine.repack_lora()


def lora_factors(engine, strip=""):
    """the engine's LoRA factors under the oracle's module names (`strip` drops the prefix a headless checkpoint lacks)"""
    return {n[len(strip):]: {"A": engine.lora.A[n].cpu(), "B": engine.lora.B[n].cpu()} for n, _, _ in engine.lora.specs}


def attach_lora(ref, engine, strip="", dropout=0.0):
    from oracle import models as om
    om.attach_lora(ref, lora_factors(engine, strip), dropout=dropout)


def hf_grads(module):
    """{parameter name: gradient} of an oracle module after its backward"""
    return {n: p.grad for n, p in module.named_parameters() if p.grad is not None}


def lora_grad_error(engine, grads, prefix="", strip=""):
    """worst relative error of the engine's LoRA gA / gB against `grads` ({prefix + module + '.lora_A': gradient})"""
    return max(max(rel(engine.lora.gA[n], grads[prefix + n[len(strip):] + ".lora_A"]),
                   rel(engine.lora.gB[n], grads[prefix + n[len(strip):] + ".lora_B"])) for n, _, _ in engine.lora.specs)


def check_rag_lora_grads(enc, dec, ref, tol=6e-2):
    """both engines' LoRA gradients against oracle.models.rag_step's"""
    worst = max(lora_grad_error(enc, ref["grads"], "retriever."), lora_grad_error(dec, ref["grads"], "generator."))
    assert worst < tol, worst


# ----------------------------------------------------------------------------------------------------------------
# full fine-tuning
# ----------------------------------------------------------------------------------------------------------------
def full_grads(engine):
    """{HF parameter name: gradient rows} sliced out of the engine's DenseBank"""
    got = {}
    for key, parts in engine._rows.items():
        gw, r = engine.full.g(key), 0
        for name, rows in parts:
            got[name] = gw[r:r + rows]
            r += rows
    return got


def compare_full_grads(engine, ref_grads, prefix, skip=(), tol=6e-2, abs_floor=1e-7):
    """every HF parameter of the fully fine-tuned engine model vs the oracle's autograd gradient"""
    worst, checked = ("", 0.0), 0
    for name, gt in full_grads(engine).items():
        if name in skip:
            continue
        rg = ref_grads[prefix + name]
        if rg.norm().item() < abs_floor:                    # a mathematically zero gradient (key bias: softmax is shift
            assert gt.float().norm().item() < 1e-4, name    # invariant): ours is bf16 rounding noise, compare absolutely
            continue
        e = rel(gt, rg)
        checked += 1
        if e > worst[1]:
            worst = (name, e)
    assert worst[1] < tol, worst
    return checked


# ----------------------------------------------------------------------------------------------------------------
# the RAG pair: a bge-tiny retriever and a Llama-family generator
# ----------------------------------------------------------------------------------------------------------------
def rag_models(dev, gcfg, gsd, lora_r=True, lora_g=True, round_bert=r16, attn_implementation=None):
    """engines and oracles of bge-tiny (vocab 600, seed 11) and the given generator. Each side is LoRA or fully fine-tuned;
    the LoRA B factors are drawn from one generator seeded 13, retriever first. -> model, enc, dec, bert, ref"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from oracle import models as om
    bcfg = synthetic.bert_config("bge-tiny", 600)
    bsd = round_bert(params.random_state_dict("bert", bcfg, seed=11))
    enc = BertEncoder(bcfg, bsd, device=dev, lora=lora_r, full=not lora_r)
    dec = LlamaDecoder(gcfg, gsd, device=dev, lora=lora_g, full=not lora_g)
    bert, ref = om.build_bert(bcfg, bsd), om.build_causal_lm(gcfg, gsd, attn_implementation=attn_implementation)
    g = torch.Generator().manual_seed(13)
    for engine, oracle, lora in ((enc, bert, lora_r), (dec, ref, lora_g)):
        if lora:
            draw_lora_B(engine, g)
            attach_lora(oracle, engine)
    mode = {(True, True): Mode.BOTH, (True, False): Mode.RETRIEVER, (False, True): Mode.GENERATOR, (False, False): None}
    model = AutoModelForRagE2E("", "", get_peft=mode[(lora_r, lora_g)], _retriever=enc, _generator=dec, _load_tokenizers=False)
    return model, enc, dec, bert, ref


def llama_rag_models(dev, vl, rnd, lora_r=True, lora_g=True):
    """rag_models with llama-tiny (seed 12) as the generator, both models' weights rounded by `rnd`"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    lcfg = synthetic.llama_config("llama-tiny", vl)
    return rag_models(dev, lcfg, rnd(params.random_state_dict("llama", lcfg, seed=12)), lora_r, lora_g, round_bert=rnd)


def rag_batch(B, Lq, Lp, Lg, vb, vl, seed, pad="left"):
    """a RAG training batch: query row 0 and passage row 1 right-padded; generator row 0 padded by 5 on the `pad` side"""
    g = torch.Generator().manual_seed(seed)
    mk = lambda L: torch.ones(B, L, dtype=torch.int64)
    b = {"retriever_query_input_ids": torch.randint(5, vb, (B, Lq), generator=g), "retriever_query_attention_mask": mk(Lq),
         "retriever_passage_input_ids": torch.randint(5, vb, (B, Lp), generator=g), "retriever_passage_attention_mask": mk(Lp),
         "generator_input_input_ids": torch.randint(3, vl, (B, Lg), generator=g), "generator_input_attention_mask": mk(Lg),
         "query_passage_input_len": torch.randint(1, Lg + 3, (B,), generator=g)}
    b["retriever_query_attention_mask"][0, Lq - 3:] = 0
    b["retriever_passage_attention_mask"][1, Lp // 2:] = 0
    if pad == "left":
        b["generator_input_attention_mask"][0, :5] = 0
    else:
        b["generator_input_attention_mask"][0, Lg - 5:] = 0
    return b


def retriever_batch(b):
    """the retriever half of a RAG batch, under the retriever-only names"""
    return {"query_input_ids": b["retriever_query_input_ids"], "query_attention_mask": b["retriever_query_attention_mask"],
            "passage_input_ids": b["retriever_passage_input_ids"], "passage_attention_mask": b["retriever_passage_attention_mask"]}


def rag_step_vs_oracle(model, enc, dec, bert, ref, batch):
    """the fused step from zeroed gradients against oracle.models.rag_step: total loss within 1e-3. -> (oracle, ours)"""
    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    want = om.rag_step(bert, ref, batch)
    enc.zero_grad_buffers(); dec.zero_grad_buffers()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["losses"][2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    return want, out


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
def check_decoder(dec, ref, g, V, B, L, pad, lora_tol=5e-2):
    """ids and the similarity matrix drawn from g: logits on valid rows within 1.5e-2, the marginalised loss within 1e-3,
    then the backward; with lora_tol the LoRA gradients within it. -> ids, mask, oracle logits"""
    from dalm_b200 import ops
    from oracle import losses
    dev = dec.dev
    ids = torch.randint(3, V, (B, L), generator=g)
    mask = pad_mask(B, L, pad)
    qlen = torch.tensor([3, L // 2, L + 2][:B])
    S = torch.randn(B, B, generator=g) * 3
    logits, ctx = dec.forward_logits(ids.to(dev), mask.to(dev))
    ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2
    ref_loss = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    ref_loss.backward()
    cvec, nsum = ops.marginal_counts(mask.to(dev), qlen.to(dev))
    tok_lp, dl = ops.ce_marginal(logits, ids.to(dev), mask.to(dev), nsum)
    mine = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(mine.item() - ref_loss.item()) / abs(ref_loss.item()) < 1e-3          # north_star tolerance
    dec.lora.zero_grad()
    dec.backward_logits(ctx, dl)
    if lora_tol is not None:
        worst = lora_grad_error(dec, hf_grads(ref))
        assert worst < lora_tol, worst
    return ids, mask, ref_logits


def check_autoregressive_retriever(enc, ref, g, V, Lq, Lp, strip=""):
    """`is_autoregressive=True` over a causal LM with LoRA (last hidden state, eos pooling): 4 left-padded queries and
    passages drawn from g, the contrastive loss within 2e-2 and the LoRA gradients within 8e-2. -> model, batch, oracle q"""
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import losses, models as om
    model = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, is_autoregressive=True, _model=enc, _load_tokenizer=False)
    B = 4
    mk = lambda L: torch.ones(B, L, dtype=torch.int64)
    rb = {"query_input_ids": torch.randint(3, V, (B, Lq), generator=g), "query_attention_mask": mk(Lq),
          "passage_input_ids": torch.randint(3, V, (B, Lp), generator=g), "passage_attention_mask": mk(Lp)}
    rb["query_attention_mask"][0, :3] = 0; rb["passage_attention_mask"][2, :6] = 0          # left padding (tokenizer default)
    q = om.retrieval_forward_autoregressive(ref, rb["query_input_ids"], rb["query_attention_mask"])
    p = om.retrieval_forward_autoregressive(ref, rb["passage_input_ids"], rb["passage_attention_mask"])
    loss = losses.contrastive_loss(losses.get_cosine_sim(q, p, 100.0))
    loss.backward()
    enc.lora.zero_grad()
    out = fused_retriever_step(model, rb, 100.0)
    assert abs(out["loss"].item() - loss.item()) / abs(loss.item()) < 2e-2
    worst = lora_grad_error(enc, hf_grads(ref), strip=strip)
    assert worst < 8e-2, worst
    return model, rb, q


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
def check_against_oracle(dec, ref, ids, mask, T, eos, pad, monkeypatch):
    """runs dec.generate with every step's logits recorded, then replays the emitted tokens through the oracle"""
    from dalm_b200 import ops
    from dalm_b200.engine import decoding
    from oracle import generate as og
    i64 = torch.int64
    rec = []
    real = ops.greedy_step_

    def recording(logits, V, *a, **k):
        rec.append(logits[:, :V].float().cpu())
        return real(logits, V, *a, **k)

    eos_list = [] if eos is None else list(eos)
    gen = lambda: dec.generate(input_ids=ids.to(dec.dev), attention_mask=mask.to(dec.dev), max_length=T, early_stopping=True,
                               eos_token_id=eos_list, pad_token_id=pad).cpu()       # [] = no EOS (None would mean the config's)
    # pass 1: eager launches with every step's logits recorded (the recorder reads them back, which a graph capture cannot)
    monkeypatch.setenv("DALM_B200_DECODE_GRAPH", "0")
    monkeypatch.setattr(ops, "greedy_step_", recording)
    out = gen()
    monkeypatch.setattr(ops, "greedy_step_", real)
    assert decoding.LAST_RUN["graph_replays"] == 0
    # pass 2: the default launch mode — the decode step captured once as a CUDA graph and replayed; same kernels, same
    # arguments, so the tokens must be IDENTICAL to the eager pass
    monkeypatch.setenv("DALM_B200_DECODE_GRAPH", "1")
    replayed = gen()
    assert decoding.LAST_RUN["graph_replays"] >= min(4, out.shape[1] - ids.shape[1] - 2), decoding.LAST_RUN
    assert torch.equal(replayed, out)
    B, L0 = ids.shape
    assert out.dtype == i64 and out.shape[0] == B and L0 < out.shape[1] <= T
    assert torch.equal(out[:, :L0], ids)                                    # prompt passes through untouched
    n_new = out.shape[1] - L0
    assert len(rec) >= n_new
    # oracle logits for every generated column, teacher-forced on OUR tokens (full re-run of the prefix, no cache)
    am = torch.cat([mask, torch.ones(B, n_new, dtype=i64)], 1)
    pos = (am.cumsum(-1) - 1).masked_fill(am == 0, 1)
    with torch.no_grad():
        want = ref(input_ids=out, attention_mask=am, position_ids=pos).logits.float()
    finished = torch.zeros(B, dtype=torch.bool)
    worst_rel, worst_margin = 0.0, 0.0
    for j in range(n_new):
        col = L0 + j
        live = ~finished
        w, g = want[:, col - 1], rec[j]
        if live.any():
            worst_rel = max(worst_rel, rel(g[live], w[live]))
            margin = w.max(-1).values - w.gather(1, out[:, col:col + 1]).squeeze(1)
            worst_margin = max(worst_margin, float(margin[live].max()))
        assert (out[finished, col] == pad).all()                             # finished rows emit the pad id
        for e in eos_list:
            finished |= live & (out[:, col] == e)
    assert worst_rel < 3e-2, worst_rel
    assert worst_margin < 0.05, worst_margin
    if eos_list and out.shape[1] < T:
        assert finished.all()                                                # stopped early only because every row hit EOS
        # ... and not a step later than HF would: before the last column someone was still generating
        f2 = torch.zeros(B, dtype=torch.bool)
        for col in range(L0, out.shape[1] - 1):
            for e in eos_list:
                f2 |= out[:, col] == e
        assert not f2.all()
    # the oracle generating from the same prompt: identical wherever its own top-1 / top-2 gap exceeds the bf16 noise
    mine = og.greedy_generate(ref, ids, mask, T, eos_token_ids=eos_list, pad_token_id=pad)
    return out, mine


def hf_generate_agreement(ref, ids, mask, out, T):
    """HF `generate` (greedy, no EOS) from the same prompt; where its tokens first differ from `out`, HF's own choice must be
    a near tie (top-1 / top-2 gap below 0.05, which bf16 may resolve either way). -> HF's tokens, per row the column up to
    which they equal `out`"""
    B, L0 = ids.shape
    ref.generation_config.eos_token_id = None                                 # no EOS: both run to max_length
    with torch.no_grad():
        hf = ref.generate(input_ids=ids, attention_mask=mask, max_length=T, do_sample=False, pad_token_id=0)
        am = torch.ones(B, T, dtype=torch.int64)
        am[:, :L0] = mask
        pos = (am.cumsum(-1) - 1).masked_fill(am == 0, 1)
        want = ref(input_ids=out, attention_mask=am, position_ids=pos).logits.float()
    agree = []
    for r in range(B):
        diff = (out[r] != hf[r]).nonzero()
        if diff.numel():
            c = int(diff[0])                                                  # same prefix up to c: HF's logits there are ours
            top2 = want[r, c - 1].topk(2).values
            assert float(top2[0] - top2[1]) < 0.05, (r, c)
        agree.append(int(diff[0]) if diff.numel() else T)
    return hf, agree


# ----------------------------------------------------------------------------------------------------------------
# trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def toy_rag_inputs(tmp_path):
    """a 12-row Abstract / Question / Answer CSV whose prompts fit well inside max_length, and a bge-tiny directory"""
    from dalm_b200 import synthetic
    words = synthetic.word_list()
    csv = str(tmp_path / "short.csv")
    with open(csv, "w", newline="") as f:
        w = _csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for i in range(12):
            w.writerow({"Abstract": " ".join(words[20 + 6 * i:26 + 6 * i]), "Question": " ".join(words[200 + 4 * i:204 + 4 * i]),
                        "Answer": " ".join(words[400 + i:402 + i])})
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    return csv, rdir


def train_rag_lora(csv, rdir, gdir, tmp_path, generator_max_len=64):
    """train_e2e with LoRA on both models; both adapters are written and the generator's B moved. -> output directory"""
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32,
              generator_max_len=generator_max_len, num_train_epochs=1, output_dir=out, use_peft=Mode.BOTH, num_warmup_steps=1,
              with_tracking=False)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out, sub, "adapter_model.bin"))
    sd = torch.load(os.path.join(out, "generator", "adapter_model.bin"), weights_only=True)
    assert any(v.abs().max() > 0 for k, v in sd.items() if "lora_B" in k)
    return out


def eval_rag_generator(csv, rdir, gdir, out, capsys):
    """evaluate_rag with the trained adapters and generation on: all 12 rows evaluated and the generator report printed"""
    from dalm_b200.eval.eval_rag import evaluate_rag
    capsys.readouterr()
    res = evaluate_rag(csv, rdir, gdir, os.path.join(out, "retriever"), os.path.join(out, "generator"), "Abstract", "Question",
                       "Answer", embed_dim=64, max_length=160, test_batch_size=4, query_batch_size=4, top_k=3,
                       evaluate_generator=True)
    text = capsys.readouterr().out
    assert res.total_examples == 12 and "Generator evaluation:" in text and "Exact match:" in text


def instruct_copy(gdir, idir, generation_config):
    """a copy of the generator directory that differs only in generation_config.json"""
    shutil.copytree(gdir, idir)
    with open(os.path.join(idir, "generation_config.json"), "w") as f:
        json.dump(generation_config, f)
    return idir
