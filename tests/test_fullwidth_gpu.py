"""-m gpu: parity at the REAL widths of every BASELINE.json config (VERDICT r1, "what's weak" 1).

One- or two-layer models with the public layer shapes — bge-large-en (1024, 16 x 64, FFN 4096, V 30522), Llama-2-7b-hf
(4096, 32 x 128, FFN 11008, V 32000), Falcon-7B (4544, 71 q / 1 kv x 64, FFN 18176, V 65024, tied head) — at the
configs' batch and sequence sizes, against the CPU fp32 oracle (HF modeling code + the reference's loss code,
oracle/models.py, oracle/losses.py) on identical seeded weights and inputs. Depth is truncated (the oracle has to finish in
seconds on host cores); width, head geometry, vocabulary, sequence lengths and batch sizes are the real ones, so every
kernel runs the tile shapes, TMA boxes and K-augmentation strides of the full models.

Tolerances: north_star's <= 1e-3 relative on the fp32 loss under bf16 forward (asserted wherever a loss exists);
hidden states / logits / gradients in relative L2 with the bf16 budgets written at each check.
"""
import math

import pytest
import torch

from model_helpers import rel

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


def _r16(sd):
    """the engine stores matmul weights in bf16: the oracle gets the same rounded values (isolates arithmetic)"""
    return {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def _nonzero_B(bank, dev, seed):
    g = torch.Generator().manual_seed(seed)
    for n, _, _ in bank.specs:
        bank.B[n].copy_((torch.randn(bank.B[n].shape, generator=g) * 0.02).to(dev))


def _factors(bank):
    return {n: {"A": bank.A[n].cpu(), "B": bank.B[n].cpu()} for n, _, _ in bank.specs}


def _worst_lora(bank, grads, prefix):
    return max(max(rel(bank.gA[n], grads[prefix + n + ".lora_A"]), rel(bank.gB[n], grads[prefix + n + ".lora_B"]))
               for n, _, _ in bank.specs)


def _rag_batch(B, Lq, Lp, Lg, vb, vl, seed):
    g = torch.Generator().manual_seed(seed)
    ones = lambda L: torch.ones(B, L, dtype=torch.int64)
    b = {"retriever_query_input_ids": torch.randint(5, vb, (B, Lq), generator=g), "retriever_query_attention_mask": ones(Lq),
         "retriever_passage_input_ids": torch.randint(5, vb, (B, Lp), generator=g), "retriever_passage_attention_mask": ones(Lp),
         "generator_input_input_ids": torch.randint(3, vl, (B, Lg), generator=g), "generator_input_attention_mask": ones(Lg),
         "query_passage_input_len": torch.randint(1, Lg + 3, (B,), generator=g)}
    b["retriever_query_attention_mask"][0, Lq - 7:] = 0                 # right padding (BERT tokenizer)
    b["retriever_passage_attention_mask"][1, Lp // 2:] = 0
    b["generator_input_attention_mask"][0, :9] = 0                       # left padding (generator tokenizer, pad = eos)
    b["generator_input_attention_mask"][2, :100] = 0
    return b


# ----------------------------------------------------------------------------------------------------------------
# cfg-3 / cfg-4: bge-large-en + Llama-2-7b-hf + PEFT(both), B 18, Lq 50 / Lp 128 / Lg 256 — the whole fused step
# ----------------------------------------------------------------------------------------------------------------
def test_cfg3_step_at_full_width(cuda_dev):
    """2 encoder layers + 1 decoder layer at the real widths through `fused_rag_step` (wgmma GEMMs incl. the K-augmented
    QKV projection and the 32000-wide lm_head, wgmma attention at (18, 256, 32 x 128), the 32000-wide CE, the fused
    in-batch loss) vs the oracle's loop body (reference train_rage2e.py:431-471)."""
    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    dev = cuda_dev
    bcfg = dict(synthetic.bert_config("bge-large-en"), num_hidden_layers=2)
    lcfg = dict(synthetic.llama_config("Llama-2-7b-hf"), num_hidden_layers=1)
    bsd, lsd = _r16(params.random_state_dict("bert", bcfg, seed=101)), _r16(params.random_state_dict("llama", lcfg, seed=102))
    enc, dec = BertEncoder(bcfg, bsd, device=dev, lora=True), LlamaDecoder(lcfg, lsd, device=dev, lora=True)
    _nonzero_B(enc.lora, dev, 103); _nonzero_B(dec.lora, dev, 104)
    enc.repack_lora(); dec.repack_lora()
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH, _retriever=enc, _generator=dec, _load_tokenizers=False)
    batch = _rag_batch(18, 50, 128, 256, bcfg["vocab_size"], lcfg["vocab_size"], seed=105)
    bert, llama = om.build_bert(bcfg, bsd), om.build_llama(lcfg, lsd)
    om.attach_lora(bert, _factors(enc.lora)); om.attach_lora(llama, _factors(dec.lora))
    torch.set_num_threads(min(torch.get_num_threads(), 32))
    ref = om.rag_step(bert, llama, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    got = out["losses"].cpu()
    relerr = lambda a, b: abs(a - b) / abs(b)
    assert relerr(got[2].item(), ref["loss"].item()) < 1e-3, (got, ref["loss"])                     # north_star tolerance
    assert relerr(got[1].item(), ref["Lm"].item()) < 1e-3
    # Lc: cross-entropy is 1-Lipschitz in the sup norm of its logits (each direction), so |dLc| <= 2 max|dS| whatever the
    # kernel does; S = 100 * cos-sim of bf16-forward embeddings, so max|dS| is the number that carries the bf16 budget
    dS = (out["S"].cpu() - ref["S"]).abs().max().item()
    assert dS < 0.15, dS                                              # 100 x 1.5e-3: bf16 GEMM operands through 2 layers
    assert abs(got[0].item() - ref["Lc"].item()) <= 2.0 * dS + 1e-5
    # ... and with the ORACLE's fp32 embeddings as input the fused loss kernel reproduces Lc / S to fp32 rounding: the
    # looser bound above is the encoder's bf16 forward, not the loss kernel (VERDICT r1 weak 1: "justify 2e-2")
    cvec, nsum = ops.marginal_counts(batch["generator_input_attention_mask"].to(dev), batch["query_passage_input_len"].to(dev))
    r = ops.inbatch_loss(ref["q"].to(dev), ref["p"].to(dev), 100.0, cvec, nsum, need_grad=False)
    assert relerr(r["losses"][0].item(), ref["Lc"].item()) < 1e-5
    assert (r["S"].cpu() - ref["S"]).abs().max().item() < 1e-3
    # gradients of every LoRA factor (bf16 activations and gradients: 6e-2 relative L2 per factor, as at toy widths)
    assert _worst_lora(enc.lora, ref["grads"], "retriever.") < 6e-2
    assert _worst_lora(dec.lora, ref["grads"], "generator.") < 6e-2
    # logits of the real-width decoder on the valid positions
    logits, _ = dec.forward_logits(batch["generator_input_input_ids"].to(dev), batch["generator_input_attention_mask"].to(dev), save=False)
    valid = batch["generator_input_attention_mask"].bool()
    assert rel(logits.float().cpu()[valid], ref["logits"][valid]) < 1.5e-2


# ----------------------------------------------------------------------------------------------------------------
# cfg-2: bge-large-en retriever-only, per-device batch 150
# ----------------------------------------------------------------------------------------------------------------
def test_cfg2_retriever_step_at_full_width(cuda_dev):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import models as om
    dev = cuda_dev
    cfg = dict(synthetic.bert_config("bge-large-en"), num_hidden_layers=1)
    sd = _r16(params.random_state_dict("bert", cfg, seed=111))
    enc = BertEncoder(cfg, sd, device=dev, lora=True)
    _nonzero_B(enc.lora, dev, 112)
    enc.repack_lora()
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, _model=enc, _load_tokenizer=False)
    B, Lq, Lp = 150, 50, 128
    g = torch.Generator().manual_seed(113)
    batch = {"query_input_ids": torch.randint(5, cfg["vocab_size"], (B, Lq), generator=g),
             "query_attention_mask": torch.ones(B, Lq, dtype=torch.int64),
             "passage_input_ids": torch.randint(5, cfg["vocab_size"], (B, Lp), generator=g),
             "passage_attention_mask": torch.ones(B, Lp, dtype=torch.int64)}
    for b in range(0, B, 7):                                           # ragged real lengths, right padded
        batch["query_attention_mask"][b, 12 + b % 30:] = 0
        batch["passage_attention_mask"][b, 40 + b % 80:] = 0
    bert = om.build_bert(cfg, sd)
    om.attach_lora(bert, _factors(enc.lora))
    ref = om.retriever_step(bert, batch)
    enc.lora.zero_grad()
    out = fused_retriever_step(se, batch, 100.0)
    dS = (out["S"].cpu() - ref["S"]).abs().max().item()
    assert dS < 0.15, dS
    assert abs(out["loss"].item() - ref["loss"].item()) <= 2.0 * dS + 1e-5        # CE is 1-Lipschitz per direction
    assert abs(out["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-2
    assert _worst_lora(enc.lora, ref["grads"], "retriever.") < 6e-2


# ----------------------------------------------------------------------------------------------------------------
# cfg-5: Falcon-7B layer shapes (4544, 71 q heads / 1 kv head x 64, FFN 18176, V 65024 tied), L 2048
# ----------------------------------------------------------------------------------------------------------------
def _falcon(dev, full):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.falcon import FalconDecoder
    from oracle import models as om
    cfg = dict(synthetic.falcon_config("falcon-7b"), num_hidden_layers=1)
    sd = _r16(params.random_state_dict("falcon", cfg, seed=121))
    return cfg, sd, FalconDecoder(cfg, sd, device=dev, full=full), om.build_falcon(cfg, sd)


def test_cfg5_falcon_forward_at_full_width(cuda_dev):
    """frozen generator: logits + the marginalised loss at B 2, L 2048 (the config's sequence length)"""
    from oracle import losses
    cfg, sd, dec, ref = _falcon(cuda_dev, full=False)
    B, L = 2, 2048
    g = torch.Generator().manual_seed(122)
    ids = torch.randint(3, cfg["vocab_size"], (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    mask[0, :37] = 0                                                   # left padding
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    with torch.no_grad():
        ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2
    S = torch.randn(B, B, generator=g) * 3
    qlen = torch.tensor([700, 2050])
    want = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    got = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(got.item() - want.item()) / abs(want.item()) < 1e-3


def test_cfg5_falcon_full_finetune_grads_at_full_width(cuda_dev):
    """`--use-peft retriever` on Falcon = the generator is FULLY fine-tuned (reference quirk 10): gradient of every HF
    parameter of one real-width layer (+ tied embedding / head, final LayerNorm) vs the oracle's autograd, B 1, L 1024"""
    from dalm_b200 import ops
    from oracle import losses
    cfg, sd, dec, ref = _falcon(cuda_dev, full=True)
    for p in ref.parameters():
        p.requires_grad_(True)
    B, L = 1, 1024
    g = torch.Generator().manual_seed(123)
    ids = torch.randint(3, cfg["vocab_size"], (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    mask[0, L - 50:] = 0
    S = torch.zeros(B, B)
    qlen = torch.tensor([300])
    ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    ref_loss = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    ref_loss.backward()
    dev = cuda_dev
    dec.full.zero_grad()
    logits, ctx = dec.forward_logits(ids.to(dev), mask.to(dev), save=True)
    cvec, nsum = ops.marginal_counts(mask.to(dev), qlen.to(dev))
    tok_lp, dl = ops.ce_marginal(logits, ids.to(dev), mask.to(dev), nsum)
    mine = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(mine.item() - ref_loss.item()) / abs(ref_loss.item()) < 1e-3
    dec.backward_logits(ctx, dl)
    got = {name: dec.full.g(key) for key, _, name in dec._names}
    worst, worst_name = 0.0, None
    for name, p_ in ref.named_parameters():
        if name == "lm_head.weight" or p_.grad is None:                 # tied: accumulated into the embedding gradient
            continue
        e = rel(got[name], p_.grad)
        if e > worst:
            worst, worst_name = e, name
    assert worst < 6e-2, (worst, worst_name)


# ----------------------------------------------------------------------------------------------------------------
# wgmma attention at the cfg-3 decoder shape against fp64 (not against the repo's own mma.sync kernel)
# ----------------------------------------------------------------------------------------------------------------
def _attn_ref64(q, k, v, mask, causal, B, L, Hq, Hkv, D, d_out=None):
    """fp64 attention, one sequence at a time (memory: Hq x L x L doubles per chunk); with d_out also (dq, dk, dv)"""
    outs, dqs, dks, dvs = [], [], [], []
    for b in range(B):
        rows = slice(b * L, (b + 1) * L)
        qd, kd, vd = (t[rows].detach().double().requires_grad_(d_out is not None) for t in (q, k, v))
        qh = qd.view(L, Hq, D).transpose(0, 1)
        kh = kd.view(L, Hkv, D).transpose(0, 1).repeat_interleave(Hq // Hkv, dim=0)
        vh = vd.view(L, Hkv, D).transpose(0, 1).repeat_interleave(Hq // Hkv, dim=0)
        s = qh @ kh.transpose(-1, -2) / math.sqrt(D)
        if mask is not None:
            s = s.masked_fill(mask[b].view(1, 1, L) == 0, float("-inf"))
        if causal:
            s = s.masked_fill(torch.triu(torch.ones(L, L, device=q.device, dtype=torch.bool), 1), float("-inf"))
        p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
        o = (p @ vh).transpose(0, 1).reshape(L, Hq * D)
        outs.append(o.detach())
        if d_out is not None:
            o.backward(d_out[rows].double())
            dqs.append(qd.grad); dks.append(kd.grad); dvs.append(vd.grad)
    if d_out is None:
        return torch.cat(outs)
    return torch.cat(outs), torch.cat(dqs), torch.cat(dks), torch.cat(dvs)


@pytest.mark.parametrize("pad", ["none", "left"])
def test_attention_tc_cfg3_shape_vs_fp64(cuda_dev, pad):
    from dalm_b200 import ops
    B, L, H, D = 18, 256, 32, 128
    dev = cuda_dev
    torch.manual_seed(1825632)
    qkv = torch.randn(B * L, 3 * H * D, device=dev).to(bf16)
    q, k, v = qkv[:, :H * D], qkv[:, H * D:2 * H * D], qkv[:, 2 * H * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    if pad == "left":
        for b in range(B):
            mask[b, :(11 * b) % 200] = 0
    rows = mask.bool().view(-1)
    d_out = torch.randn(B * L, H * D, device=dev).to(bf16)
    d_out[~rows] = 0
    out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, True)
    dq, dk, dv = ops.attention_tc_bwd(q, k, v, mask, out, lse, d_out, B, L, H, H, D, True)
    ref, rq, rk, rv = _attn_ref64(q, k, v, mask, True, B, L, H, H, D, d_out)
    assert rel(out.float()[rows], ref[rows]) < 1e-2
    assert out.float()[~rows].abs().max().item() == 0.0 if (~rows).any() else True
    assert rel(dq.float()[rows], rq[rows]) < 2e-2
    assert rel(dk.float(), rk) < 2e-2
    assert rel(dv.float(), rv) < 2e-2
