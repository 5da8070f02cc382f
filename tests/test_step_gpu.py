"""-m gpu: the whole loop body (reference train_rage2e.py:431-474 / train_retriever_only.py:365-379) — fused launch
sequence AND the reference-style autograd loop over the drop-in API — against the CPU fp32 oracle; then the trainers
end to end on a toy CSV with tiny random-init models (BASELINE config 1 on the GPU side)."""
import json
import os

import pytest
import torch

from model_helpers import (attach_lora, check_autoregressive_retriever, check_rag_lora_grads, draw_lora_B, lora_grad_error,
                           llama_rag_models, r16_2d, rag_batch, rag_step_vs_oracle, rel, retriever_batch)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("pad", ["left", "right"])
def test_fused_rag_step_matches_oracle(cuda_dev, pad):
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 500, r16_2d)
    batch = rag_batch(5, 12, 24, 40, 600, 500, seed=21, pad=pad)
    ref, out = rag_step_vs_oracle(model, enc, dec, bert, llama, batch)                        # total loss: north_star 1e-3
    got = out["losses"].cpu()
    assert abs(got[0].item() - ref["Lc"].item()) / abs(ref["Lc"].item()) < 2e-2               # bf16 embeddings x logit_scale 100
    assert abs(got[1].item() - ref["Lm"].item()) / abs(ref["Lm"].item()) < 1e-3
    check_rag_lora_grads(enc, dec, ref)


def test_reference_style_loop_body_over_the_dropin_api(cuda_dev):
    """the reference's loop body, verbatim structure (train_rage2e.py:431-474), driving dalm_b200 through autograd"""
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import (compute_marginalized_loss_from_logits, fused_rag_step,
                                                      get_cosine_sim, get_nt_xent_loss)
    from oracle import models as om
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 500, r16_2d)
    batch = rag_batch(4, 10, 20, 32, 600, 500, seed=31)
    ref = om.rag_step(bert, llama, batch)
    dbatch = {k: v.to(cuda_dev) for k, v in batch.items()}
    optimizer = FusedAdam(model.parameters(), lr=1e-3)
    optimizer.zero_grad()
    q = model("retrieval", dbatch["retriever_query_input_ids"], dbatch["retriever_query_attention_mask"])
    p = model("retrieval", dbatch["retriever_passage_input_ids"], dbatch["retriever_passage_attention_mask"])
    logits = get_cosine_sim(q, p, 100)
    loss_c = (get_nt_xent_loss(logits) + get_nt_xent_loss(logits.t())) / 2.0
    gen_logits = model("generation", dbatch["generator_input_input_ids"], dbatch["generator_input_attention_mask"])
    loss_m = compute_marginalized_loss_from_logits(gen_logits, dbatch["generator_input_input_ids"],
                                                   dbatch["generator_input_attention_mask"], logits,
                                                   dbatch["query_passage_input_len"])
    loss = loss_c + loss_m
    loss.backward()
    assert abs(loss.item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    check_rag_lora_grads(enc, dec, ref)
    # same gradients as the fused launch sequence
    g_auto = [enc.lora.grad.clone(), dec.lora.grad.clone()]
    optimizer.zero_grad()
    fused_rag_step(model, batch, 100.0)
    assert rel(enc.lora.grad, g_auto[0]) < 1e-2 and rel(dec.lora.grad, g_auto[1]) < 1e-2
    before = dec.lora.flat.clone()
    optimizer.step(); model.repack()
    assert (dec.lora.flat - before).abs().max().item() > 0


def test_retriever_only_step_and_stepwise_training(cuda_dev):
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import models as om
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 500, r16_2d)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, _model=enc, _load_tokenizer=False)
    rb = retriever_batch(rag_batch(6, 12, 24, 8, 600, 500, seed=41))
    ref = om.retriever_step(bert, rb)
    enc.lora.zero_grad()
    out = fused_retriever_step(se, rb, 100.0)
    assert abs(out["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 2e-2
    # a few optimizer steps reduce the contrastive loss on a fixed batch
    opt = FusedAdam(se.parameters(), lr=2e-3)
    first = None
    for i in range(8):
        opt.zero_grad()
        l = fused_retriever_step(se, rb, 100.0)["loss"].item()
        first = l if first is None else first
        opt.step(); enc.repack_lora()
    assert l < first


def test_trainers_end_to_end_on_toy_csv(cuda_dev, tmp_path):
    """BASELINE config 1 shape of run (toy CSV, tiny random-init models, bs 2) through train_e2e / train_retriever,
    including checkpointing, final adapter artefacts and resume."""
    from dalm_b200 import synthetic
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    from dalm_b200.training.retriever_only.train_retriever_only import train_retriever
    from dalm_b200.models.rag_e2e_base_model import Mode
    csv = synthetic.write_csv(str(tmp_path / "toy.csv"), 12, seed=5)
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=900)
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64,
              num_train_epochs=1, output_dir=out, checkpointing_steps="3", use_peft=Mode.BOTH, num_warmup_steps=1,
              with_tracking=True)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out, sub, "adapter_config.json"))
        assert os.path.exists(os.path.join(out, sub, "adapter_model.bin"))
        assert json.load(open(os.path.join(out, sub, "adapter_config.json")))["r"] == 8
    assert os.path.isdir(os.path.join(out, "step_3")) and os.path.exists(os.path.join(out, "metrics.jsonl"))
    sd = torch.load(os.path.join(out, "generator", "adapter_model.bin"), weights_only=True)
    assert any(v.abs().max() > 0 for k, v in sd.items() if "lora_B" in k)          # B moved away from its zero init
    # resume from the step checkpoint
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64,
              num_train_epochs=1, output_dir=out, resume_from_checkpoint=os.path.join(out, "step_3"), use_peft=Mode.BOTH,
              with_tracking=False)
    out2 = str(tmp_path / "out_ret")
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out2, use_peft=True, use_bnb=False, with_tracking=False)
    assert os.path.exists(os.path.join(out2, "retriever", "adapter_model.bin"))


def test_fused_step_with_frozen_falcon_generator(cuda_dev):
    """BASELINE config 5 family at toy size: bge encoder with LoRA (use_peft='retriever') + frozen Falcon generator. The LM
    loss reaches the retriever only through the doc log-prob term; generator backward is never launched."""
    from dalm_b200 import synthetic, _lib
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.falcon import FalconDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    bcfg, fcfg = synthetic.bert_config("bge-tiny", 600), synthetic.falcon_config("falcon-tiny", 504)
    bsd, fsd = r16_2d(params.random_state_dict("bert", bcfg, seed=21)), r16_2d(params.random_state_dict("falcon", fcfg, seed=22))
    enc, dec = BertEncoder(bcfg, bsd, device=cuda_dev, lora=True), FalconDecoder(fcfg, fsd, device=cuda_dev)
    draw_lora_B(enc, torch.Generator().manual_seed(23))
    model = AutoModelForRagE2E("", "", get_peft=Mode.RETRIEVER, _retriever=enc, _generator=dec, _load_tokenizers=False)
    batch = rag_batch(4, 10, 20, 48, 600, 504, seed=24)
    bert, falcon = om.build_bert(bcfg, bsd), om.build_falcon(fcfg, fsd)
    attach_lora(bert, enc)
    for p_ in falcon.parameters():
        p_.requires_grad_(False)
    ref = om.rag_step(bert, falcon, batch)
    enc.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    worst = lora_grad_error(enc, ref["grads"], "retriever.")
    assert worst < 6e-2, worst


def test_autoregressive_retriever(cuda_dev):
    """`is_autoregressive=True`: a causal LM as the retriever (last hidden state, eos pooling, LoRA on q_proj / v_proj) —
    reference retriever_only_base_model.py:48-58 / rag_e2e_base_model.py:84-90"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.training.utils.train_utils import get_cosine_sim, get_nt_xent_loss
    from oracle import models as om
    cfg = synthetic.llama_config("llama-tiny", 400)
    sd = r16_2d(params.random_state_dict("llama", cfg, seed=31))
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    g = torch.Generator().manual_seed(32)
    draw_lora_B(enc, g)
    ref = om.build_llama(cfg, sd)
    attach_lora(ref, enc)
    model, rb, q = check_autoregressive_retriever(enc, ref, g, 400, 12, 20)
    # the wrapper's own forward (autograd bridge) gives the same embeddings and gradients
    g_fused = enc.lora.grad.clone()
    enc.lora.zero_grad()
    dq = {k: v.to(cuda_dev) for k, v in rb.items()}
    qe = model(dq["query_input_ids"], dq["query_attention_mask"]); pe = model(dq["passage_input_ids"], dq["passage_attention_mask"])
    assert rel(qe, q.detach()) < 2e-2
    S = get_cosine_sim(qe, pe, 100)
    ((get_nt_xent_loss(S) + get_nt_xent_loss(S.t())) / 2.0).backward()
    assert rel(enc.lora.grad, g_fused) < 2e-2


def test_packed_loader_trains_like_the_reference_pipeline(cuda_dev, tmp_path, monkeypatch):
    """DALM_B200_PACKED_LOADER=1 (memory-mapped int32 matrix, one gather per batch) through `train_e2e`: same batches in the same
    order, so the logged epoch loss equals the default DataLoader + collate run (up to the LoRA wgrad's atomic summation order)"""
    from dalm_b200 import synthetic
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    from dalm_b200.models.rag_e2e_base_model import Mode
    csv = synthetic.write_csv(str(tmp_path / "toy.csv"), 14, seed=6)
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=900)
    losses = []
    for packed in ("0", "1"):
        monkeypatch.setenv("DALM_B200_PACKED_LOADER", packed)
        out = str(tmp_path / f"out{packed}")
        train_e2e(csv, rdir, gdir, per_device_train_batch_size=4, query_max_len=16, passage_max_len=32, generator_max_len=64,
                  num_train_epochs=1, output_dir=out, use_peft=Mode.BOTH, num_warmup_steps=1, with_tracking=True, seed=7)
        rec = [json.loads(l) for l in open(os.path.join(out, "metrics.jsonl")) if "train/epoch_loss" in l]
        losses.append(rec[-1]["train/epoch_loss"])
        if packed == "1":
            assert any(f.startswith("packed_") and f.endswith(".npy") for f in os.listdir(os.path.join(out, ".packed_cache")))
    assert abs(losses[0] - losses[1]) < 2e-2 * abs(losses[0]), losses      # one epoch over the same rows; batch identity itself is pinned on CPU
