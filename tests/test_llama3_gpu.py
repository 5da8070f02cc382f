"""-m gpu: Llama 3.x generators and retrievers (Llama with GQA and llama3 RoPE frequency scaling).

No kernel is new: every RoPE consumer (the QKV GEMM's RoPE epilogue at head_dim 128, the rope row kernel at head_dim 64, the
position-indexed kernel of prefill and decode) reads the cos / sin tables the decoder builds from `params.rope_inv_freq`. So
the checks are whole models against transformers' LlamaForCausalLM (fp32, same bf16-rounded weights) with the scaling on:
llama3-tiny (head_dim 128, the fused epilogue, untied) and llama3.2-tiny (head_dim 64, the row kernel, tied head), at sequence
lengths past original_max_position_embeddings (64). The q / k projections are drawn 2.5x wider than initializer_range so that
attention depends strongly on position: the same decoder with default (unscaled) tables then misses the logits by 10x the
tolerance (the control), which shows that these tests tell the two apart. Tolerances are those of test_qwen3_gpu.py.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64
QK_SCALE = 2.5


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def build_llama3(cfg, sd):
    """transformers' LlamaForCausalLM, fp32, on the given HF-named weights (tied configs store no lm_head)"""
    from transformers import LlamaConfig, LlamaForCausalLM
    m = LlamaForCausalLM(LlamaConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}))
    assert m.config.rope_parameters["rope_type"] == "llama3"
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected and set(missing) <= ({"lm_head.weight"} if cfg.get("tie_word_embeddings") else set()), (missing, unexpected)
    return m.float().eval()


def _llama3(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.llama3_config(name, vocab_size=V)
    sd = params.random_state_dict("llama", cfg, seed=seed)
    sd = {k: (v * QK_SCALE if k.endswith(("q_proj.weight", "k_proj.weight")) else v) for k, v in sd.items()}
    return cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def _default_tables(dec):
    """turn `dec` into the control: the same weights with the unscaled frequencies"""
    dec.inv_freq = 1.0 / (dec.cfg["rope_theta"] ** (torch.arange(0, dec.hd, 2, dtype=f32) / dec.hd))
    dec._rope_cache.clear()


def _mask(B, L, pad):
    mask = torch.ones(B, L, dtype=i64)
    if pad == "right":
        mask[0, L - 5:] = 0
    else:
        mask[0, :5] = 0; mask[1, :2] = 0
    return mask


def _lora_init(dec, ref, seed):
    from oracle import models as om
    g = torch.Generator().manual_seed(seed)
    for n, _, _ in dec.lora.specs:
        dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(dec.dev))
    dec.repack_lora()
    om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,L,pad", [("llama3-tiny", 3, 72, "right"), ("llama3-tiny", 2, 130, "left"),
                                           ("llama3.2-tiny", 3, 72, "left"), ("llama3.2-tiny", 2, 130, "right")])
def test_llama3_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF LlamaForCausalLM with llama3 scaling; then the control: the
    same decoder on default tables fails the logits tolerance"""
    from dalm_b200 import ops
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import losses, models as om
    V = 504
    cfg, sd = _llama3(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    fused = ((dec.nh + dec.nkv) * dec.hd) % 256 == 0 and dec.fuse_rope
    assert fused == (name == "llama3-tiny") and dec.nkv < dec.nh
    ref = build_llama3(cfg, sd)
    assert torch.equal(ref.model.rotary_emb.inv_freq, dec.inv_freq)
    _lora_init(dec, ref, 9)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(3, V, (B, L), generator=g)
    mask = _mask(B, L, pad)
    qlen = torch.tensor([3, L // 2, L + 2][:B])
    S = torch.randn(B, B, generator=g) * 3
    logits, ctx = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev))
    ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert _rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2
    ref_loss = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    ref_loss.backward()
    cvec, nsum = ops.marginal_counts(mask.to(cuda_dev), qlen.to(cuda_dev))
    tok_lp, dl = ops.ce_marginal(logits, ids.to(cuda_dev), mask.to(cuda_dev), nsum)
    mine = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(mine.item() - ref_loss.item()) / abs(ref_loss.item()) < 1e-3
    dec.lora.zero_grad()
    dec.backward_logits(ctx, dl)
    worst = 0.0
    for n, _, _ in dec.lora.specs:
        mod = om._get_module(ref, n)
        worst = max(worst, _rel(dec.lora.gA[n], mod.lora_A.grad), _rel(dec.lora.gB[n], mod.lora_B.grad))
    assert worst < 5e-2, worst
    _default_tables(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert _rel(control.float().cpu()[valid], ref_logits[valid]) > 10 * 1.5e-2


def _rag_models(dev, gcfg, gsd, lora):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from oracle import models as om
    bcfg = synthetic.bert_config("bge-tiny", 600)
    r16 = lambda sd: {k: v.to(bf16).float() for k, v in sd.items()}
    bsd = r16(params.random_state_dict("bert", bcfg, seed=11))
    enc = BertEncoder(bcfg, bsd, device=dev, lora=lora, full=not lora)
    dec = LlamaDecoder(gcfg, gsd, device=dev, lora=lora, full=not lora)
    bert, ref = om.build_bert(bcfg, bsd), build_llama3(gcfg, gsd)
    if lora:
        g = torch.Generator().manual_seed(13)
        for bank in (enc.lora, dec.lora):
            for n, _, _ in bank.specs:
                bank.B[n].copy_((torch.randn(bank.B[n].shape, generator=g) * 0.02).to(dev))
        enc.repack_lora(); dec.repack_lora()
        om.attach_lora(bert, {n: {"A": enc.lora.A[n].cpu(), "B": enc.lora.B[n].cpu()} for n, _, _ in enc.lora.specs})
        om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH if lora else None, _retriever=enc, _generator=dec, _load_tokenizers=False)
    return model, enc, dec, bert, ref


@pytest.mark.parametrize("name,pad", [("llama3-tiny", "left"), ("llama3.2-tiny", "right")])
def test_fused_rag_step_llama3_lora(cuda_dev, name, pad):
    """bge + Llama 3 generator, LoRA on both, generator length 80 (past original_max_position_embeddings): the fused training
    step against the reference loop body"""
    from test_step_gpu import _batch, _check_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _llama3(name, 504, seed=12)
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=True)
    batch = _batch(5, 12, 24, 80, 600, 504, seed=21, pad=pad)
    want = om.rag_step(bert, ref, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    got = out["losses"].cpu()
    assert abs(got[2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    _check_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["llama3-tiny", "llama3.2-tiny"])
def test_full_finetune_llama3_gradients(cuda_dev, name):
    """full fine-tuning: every parameter's gradient against autograd through HF; on llama3.2-tiny the head is tied, so the
    embedding table's gradient holds the head's and the gather's parts"""
    from test_full_ft_gpu import _batch, _compare_full_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _llama3(name, 504, seed=14)
    sd = {k: v.to(bf16).float() for k, v in sd.items()}                 # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=False)
    assert dec.tied == (name == "llama3.2-tiny")
    batch = _batch(5, 12, 24, 80, 600, 504, seed=21)
    want = om.rag_step(bert, ref, batch)
    enc.full.zero_grad(); dec.full.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["losses"][2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    checked = _compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 7 * cfg["num_hidden_layers"] + 2
    emb = dec.full.g("embed")
    assert _rel(emb, want["grads"]["generator.model.embed_tokens.weight"]) < 6e-2
    if dec.tied:
        assert "lm_head.weight" not in dec.hf_state_dict()


def test_autoregressive_llama3_retriever(cuda_dev):
    """`is_autoregressive=True` with a Llama 3 model: last hidden state, eos pooling, LoRA on q_proj / v_proj, lengths past
    original_max_position_embeddings"""
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import losses, models as om
    V = 504
    cfg, sd = _llama3("llama3-tiny", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    ref = build_llama3(cfg, sd)
    _lora_init(enc, ref, 32)
    g = torch.Generator().manual_seed(32)
    model = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, is_autoregressive=True, _model=enc, _load_tokenizer=False)
    B, Lq, Lp = 4, 24, 90
    mk = lambda L: torch.ones(B, L, dtype=i64)
    rb = {"query_input_ids": torch.randint(3, V, (B, Lq), generator=g), "query_attention_mask": mk(Lq),
          "passage_input_ids": torch.randint(3, V, (B, Lp), generator=g), "passage_attention_mask": mk(Lp)}
    rb["query_attention_mask"][0, :3] = 0; rb["passage_attention_mask"][2, :6] = 0
    q = om.retrieval_forward_autoregressive(ref, rb["query_input_ids"], rb["query_attention_mask"])
    p = om.retrieval_forward_autoregressive(ref, rb["passage_input_ids"], rb["passage_attention_mask"])
    loss = losses.contrastive_loss(losses.get_cosine_sim(q, p, 100.0))
    loss.backward()
    enc.lora.zero_grad()
    out = fused_retriever_step(model, rb, 100.0)
    assert abs(out["loss"].item() - loss.item()) / abs(loss.item()) < 2e-2
    worst = 0.0
    for n, _, _ in enc.lora.specs:
        mod = om._get_module(ref, n)
        worst = max(worst, _rel(enc.lora.gA[n], mod.lora_A.grad), _rel(enc.lora.gB[n], mod.lora_B.grad))
    assert worst < 8e-2, worst


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,lora", [("llama3-tiny", 4, False), ("llama3.2-tiny", 4, True), ("llama3-tiny", 20, False)])
def test_llama3_generate_greedy(cuda_dev, monkeypatch, name, B, lora):
    """greedy decoding to position 99 (past original_max_position_embeddings = 64): per-step logits and choices vs HF
    teacher-forced on our tokens, graph replay == eager, and the tokens equal HF `generate`'s wherever HF's own choice is not
    a near tie (top-1 / top-2 gap above bf16 noise); B <= 16 decodes through decode_gemm, B = 20 through wgmma"""
    from test_generate_gpu import _check_against_oracle

    from dalm_b200.engine.llama import LlamaDecoder
    V, L0, T = 504, 12, 100
    cfg, sd = _llama3(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = build_llama3(cfg, sd)
    if lora:
        _lora_init(dec, ref, 9)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(4, V, (B, L0), generator=g)
    mask = torch.ones(B, L0, dtype=i64)
    mask[1, :3] = 0
    mask[2, 9:] = 0
    out, _ = _check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert out.shape == (B, T)
    ref.generation_config.eos_token_id = None                                 # no EOS: both run to max_length
    with torch.no_grad():
        hf = ref.generate(input_ids=ids, attention_mask=mask, max_length=T, do_sample=False, pad_token_id=0)
        am = torch.ones(B, T, dtype=i64)
        am[:, :L0] = mask
        pos = (am.cumsum(-1) - 1).masked_fill(am == 0, 1)
        want = ref(input_ids=out, attention_mask=am, position_ids=pos).logits.float()
    assert hf.shape == (B, T)
    agree = []                                                                # columns up to which each row equals HF's
    for r in range(B):
        diff = (out[r] != hf[r]).nonzero()
        if diff.numel():
            c = int(diff[0])                                                  # same prefix up to c: HF's logits there are ours
            top2 = want[r, c - 1].topk(2).values
            assert float(top2[0] - top2[1]) < 0.05, (r, c)                    # a near tie that bf16 may resolve either way
        agree.append(int(diff[0]) if diff.numel() else T)
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
    ref = build_llama3(cfg, sd)
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
    assert _rel(rec[0][0], hf_last) < 3e-2
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
    import csv as _csv
    import json
    import shutil

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    words = synthetic.word_list()
    csv = str(tmp_path / "short.csv")
    with open(csv, "w", newline="") as f:
        w = _csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for i in range(12):
            w.writerow({"Abstract": " ".join(words[20 + 6 * i:26 + 6 * i]), "Question": " ".join(words[200 + 4 * i:204 + 4 * i]),
                        "Answer": " ".join(words[400 + i:402 + i])})
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama3.2-tiny"), "llama", "llama3.2-tiny", vocab_size=1200,
                                     generation_config=synthetic.LLAMA3_GENERATION["base"])
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=80,
              num_train_epochs=1, output_dir=out, use_peft=Mode.BOTH, num_warmup_steps=1, with_tracking=False)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out, sub, "adapter_model.bin"))
    sd = torch.load(os.path.join(out, "generator", "adapter_model.bin"), weights_only=True)
    assert any(v.abs().max() > 0 for k, v in sd.items() if "lora_B" in k)
    idir = str(tmp_path / "llama3.2-tiny-instruct")                            # differs only in generation_config.json
    shutil.copytree(gdir, idir)
    with open(os.path.join(idir, "generation_config.json"), "w") as f:
        json.dump(synthetic.LLAMA3_GENERATION["instruct"], f)
    for d in (gdir, idir):
        capsys.readouterr()
        torch.manual_seed(0)
        res = evaluate_rag(csv, rdir, d, os.path.join(out, "retriever"), os.path.join(out, "generator"), "Abstract", "Question",
                           "Answer", embed_dim=64, max_length=160, test_batch_size=4, query_batch_size=4, top_k=3,
                           evaluate_generator=True)
        text = capsys.readouterr().out
        assert res.total_examples == 12 and "Generator evaluation:" in text and "Exact match:" in text
