"""-m gpu: Llama 3.x generators and retrievers (Llama with GQA and llama3 RoPE frequency scaling).

No kernel is new: every RoPE consumer (the QKV GEMM's RoPE epilogue at head_dim 128, the rope row kernel at head_dim 64, the
position-indexed kernel of prefill and decode) reads the cos / sin tables the decoder builds from `params.rope_inv_freq`. So
the checks are whole models against transformers' LlamaForCausalLM (fp32, same bf16-rounded weights) with the scaling on:
llama3-tiny (head_dim 128, the fused epilogue, untied) and llama3.2-tiny (head_dim 64, the row kernel, tied head), at sequence
lengths past original_max_position_embeddings (64). The q / k projections are drawn 2.5x wider than initializer_range so that
attention depends strongly on position: the same decoder with default (unscaled) tables then misses the logits by 10x the
tolerance (the control), which shows that these tests tell the two apart. Tolerances are those of test_qwen3_gpu.py.
"""
import pytest
import torch

from model_helpers import (attach_lora, check_against_oracle, check_autoregressive_retriever, check_decoder, check_rag_lora_grads,
                           compare_full_grads, draw_lora_B, eval_rag_generator, hf_generate_agreement, instruct_copy, prompt, r16,
                           r16_2d, rag_batch, rag_models, rag_step_vs_oracle, rel, toy_rag_inputs, train_rag_lora)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
QK_SCALE = 2.5


def _hf(cfg, sd):
    """transformers' LlamaForCausalLM with llama3 frequency scaling"""
    from oracle import models as om
    m = om.build_causal_lm(cfg, sd)
    assert m.config.rope_parameters["rope_type"] == "llama3"
    return m


def _llama3(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.llama3_config(name, vocab_size=V)
    sd = params.random_state_dict("llama", cfg, seed=seed)
    sd = {k: (v * QK_SCALE if k.endswith(("q_proj.weight", "k_proj.weight")) else v) for k, v in sd.items()}
    return cfg, r16_2d(sd)


def _default_tables(dec):
    """turn `dec` into the control: the same weights with the unscaled frequencies"""
    dec.inv_freq = 1.0 / (dec.cfg["rope_theta"] ** (torch.arange(0, dec.hd, 2, dtype=f32) / dec.hd))
    dec._rope_cache.clear()


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,L,pad", [("llama3-tiny", 3, 72, "right"), ("llama3-tiny", 2, 130, "left"),
                                           ("llama3.2-tiny", 3, 72, "left"), ("llama3.2-tiny", 2, 130, "right")])
def test_llama3_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF LlamaForCausalLM with llama3 scaling; then the control: the
    same decoder on default tables fails the logits tolerance"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _llama3(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    fused = ((dec.nh + dec.nkv) * dec.hd) % 256 == 0 and dec.fuse_rope
    assert fused == (name == "llama3-tiny") and dec.nkv < dec.nh
    ref = _hf(cfg, sd)
    assert torch.equal(ref.model.rotary_emb.inv_freq, dec.inv_freq)
    draw_lora_B(dec, torch.Generator().manual_seed(9))
    attach_lora(ref, dec)
    ids, mask, ref_logits = check_decoder(dec, ref, torch.Generator().manual_seed(9), V, B, L, pad)
    valid = mask.bool()
    _default_tables(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert rel(control.float().cpu()[valid], ref_logits[valid]) > 10 * 1.5e-2


@pytest.mark.parametrize("name,pad", [("llama3-tiny", "left"), ("llama3.2-tiny", "right")])
def test_fused_rag_step_llama3_lora(cuda_dev, name, pad):
    """bge + Llama 3 generator, LoRA on both, generator length 80 (past original_max_position_embeddings): the fused training
    step against the reference loop body"""
    cfg, sd = _llama3(name, 504, seed=12)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd)
    assert ref.config.rope_parameters["rope_type"] == "llama3"
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 80, 600, 504, seed=21, pad=pad))
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["llama3-tiny", "llama3.2-tiny"])
def test_full_finetune_llama3_gradients(cuda_dev, name):
    """full fine-tuning: every parameter's gradient against autograd through HF; on llama3.2-tiny the head is tied, so the
    embedding table's gradient holds the head's and the gather's parts"""
    cfg, sd = _llama3(name, 504, seed=14)
    sd = r16(sd)                                                          # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, lora_r=False, lora_g=False)
    assert ref.config.rope_parameters["rope_type"] == "llama3"
    assert dec.tied == (name == "llama3.2-tiny")
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 80, 600, 504, seed=21))
    checked = compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 7 * cfg["num_hidden_layers"] + 2
    emb = dec.full.g("embed")
    assert rel(emb, want["grads"]["generator.model.embed_tokens.weight"]) < 6e-2
    if dec.tied:
        assert "lm_head.weight" not in dec.hf_state_dict()


def test_autoregressive_llama3_retriever(cuda_dev):
    """`is_autoregressive=True` with a Llama 3 model: last hidden state, eos pooling, LoRA on q_proj / v_proj, lengths past
    original_max_position_embeddings"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _llama3("llama3-tiny", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    ref = _hf(cfg, sd)
    draw_lora_B(enc, torch.Generator().manual_seed(32))
    attach_lora(ref, enc)
    check_autoregressive_retriever(enc, ref, torch.Generator().manual_seed(32), V, 24, 90)


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,lora", [("llama3-tiny", 4, False), ("llama3.2-tiny", 4, True), ("llama3-tiny", 20, False)])
def test_llama3_generate_greedy(cuda_dev, monkeypatch, name, B, lora):
    """greedy decoding to position 99 (past original_max_position_embeddings = 64): per-step logits and choices vs HF
    teacher-forced on our tokens, graph replay == eager, and the tokens equal HF `generate`'s wherever HF's own choice is not
    a near tie (top-1 / top-2 gap above bf16 noise); B <= 16 decodes through decode_gemm, B = 20 through wgmma"""
    from dalm_b200.engine.llama import LlamaDecoder
    V, L0, T = 504, 12, 100
    cfg, sd = _llama3(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = _hf(cfg, sd)
    if lora:
        draw_lora_B(dec, torch.Generator().manual_seed(9))
        attach_lora(ref, dec)
    ids, mask = prompt(B, L0, V, seed=1, low=4)
    out, _ = check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert out.shape == (B, T)
    hf, agree = hf_generate_agreement(ref, ids, mask, out, T)
    assert hf.shape == (B, T)
    assert max(agree) == T and L0 + 64 < T                                    # some row agrees to the end, past position 64


def test_llama3_instruct_sampling_distribution(cuda_dev, monkeypatch):
    """the Instruct generation config (sampling, temperature 0.6, top-p 0.9, top-k left at 50, three EOS ids): 4096 copies of a
    70-token prompt (its last positions past original_max_position_embeddings), one new token each, fit the oracle distribution
    of the engine's own prefill logits; those logits match HF's; under the same seed graph replay gives the eager tokens"""
    import numpy as np
    from scipy.stats import chisquare

    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import decoding
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import sampling as osmp
    V = 504
    cfg, sd = _llama3("llama3-tiny", V, seed=5)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    ref = _hf(cfg, sd)
    dec.generation_config = dict(synthetic.LLAMA3_GENERATION["instruct"])
    assert decoding.decoding_mode(dec) == "sampling (temperature 0.6, top-k 50, top-p 0.9)"
    ids = torch.randint(4, V, (1, 70), generator=torch.Generator().manual_seed(5))
    mask = torch.ones_like(ids)
    N, T, k, p = 4096, 0.6, 50, 0.9
    rec = []
    real = ops.sample_step_

    def recording(logits, V_, *a, **kw):
        rec.append(logits[:, :V_].float().cpu())
        return real(logits, V_, *a, **kw)

    monkeypatch.setattr(ops, "sample_step_", recording)
    torch.manual_seed(0)
    out = dec.generate(input_ids=ids.expand(N, -1).to(cuda_dev), attention_mask=mask.expand(N, -1).to(cuda_dev),
                       max_new_tokens=1).cpu()
    monkeypatch.setattr(ops, "sample_step_", real)
    assert out.shape == (N, 71) and len(rec) == 1
    with torch.no_grad():
        hf_last = ref(input_ids=ids, attention_mask=mask).logits[0, -1].float()
    assert rel(rec[0][0], hf_last) < 3e-2
    first = out[:, 70].numpy()
    uniq, inv = torch.unique(rec[0], dim=0, return_inverse=True)
    prob = np.zeros(V)
    for i in range(uniq.shape[0]):
        prob += osmp.probs(osmp.warp(uniq[i].to(bf16).float(), T, k, p)) * int((inv == i).sum())
    counts = np.bincount(first, minlength=V)
    assert counts[prob == 0].sum() == 0
    kept = prob > 0
    big = prob[kept] >= 5
    f_obs = np.append(counts[kept][big], counts[kept][~big].sum())
    f_exp = np.append(prob[kept][big], prob[kept][~big].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    assert chisquare(f_obs, f_exp).pvalue > 1e-6

    def gen(seed, graph):
        monkeypatch.setenv("DALM_B200_DECODE_GRAPH", graph)
        torch.manual_seed(seed)
        return dec.generate(input_ids=ids.expand(4, -1).to(cuda_dev), attention_mask=mask.expand(4, -1).to(cuda_dev),
                            max_length=100, eos_token_id=[], pad_token_id=0).cpu()

    eager = gen(7, "0")
    assert eager.shape == (4, 100) and torch.equal(gen(7, "0"), eager)
    assert torch.equal(gen(7, "1"), eager) and decoding.LAST_RUN["graph_replays"] >= 4


# ----------------------------------------------------------------------------------------------------------------
# trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_llama3_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Llama 3 directory (Llama 3 tokenizer, llama3 RoPE) writes
    PEFT adapters; eval_rag loads them and samples under the base and the Instruct generation config"""
    from dalm_b200 import synthetic
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama3.2-tiny"), "llama", "llama3.2-tiny", vocab_size=1200,
                                     generation_config=synthetic.LLAMA3_GENERATION["base"])
    out = train_rag_lora(csv, rdir, gdir, tmp_path, generator_max_len=80)
    idir = instruct_copy(gdir, str(tmp_path / "llama3.2-tiny-instruct"), synthetic.LLAMA3_GENERATION["instruct"])
    for d in (gdir, idir):
        torch.manual_seed(0)
        eval_rag_generator(csv, rdir, d, out, capsys)
