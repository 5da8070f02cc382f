"""-m gpu: FULL fine-tuning (the reference's default `use_peft=None` / `--no-use-peft`: Adam over every parameter,
train_rage2e.py:336, train_retriever_only.py:262) — the MN-major GEMM layouts behind dgrad / wgrad, the parameter-gradient
kernels, the shadowed Adam, and the whole step's gradients for EVERY parameter against the CPU fp32 oracle's autograd."""
import os

import pytest
import torch

from model_helpers import (attach_lora, compare_full_grads, draw_lora_B, llama_rag_models, lora_grad_error, r16, rag_batch,
                           rag_step_vs_oracle, rel, retriever_batch)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32

# ---------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,bn,max_ctas", [(300, 200, 136, 0, 0), (128, 256, 64, 256, 0), (520, 1096, 328, 128, 3),
                                               (257, 72, 1000, 64, 2), (1024, 512, 512, 256, 0)])
def test_gemm_nn_layout_is_dgrad_against_untransposed_weight(cuda_dev, M, N, K, bn, max_ctas):
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(cuda_dev, bf16)
    w = (torch.randn(K, N, generator=g) * 0.1).to(cuda_dev, bf16)          # W[out=K, in=N]: dx = dy W
    out = ops.gemm(a, w, layout=1, block_n=bn, max_ctas=max_ctas)
    ref = a.float() @ w.float()
    assert rel(out.float(), ref) < 5e-3
    out32 = ops.gemm(a, w, layout=1, out_dtype=f32, block_n=bn, max_ctas=max_ctas)
    assert rel(out32, ref) < 1e-4


@pytest.mark.parametrize("T,M,N,bn,max_ctas", [(1000, 192, 320, 0, 0), (64, 128, 256, 256, 0), (3204, 264, 1096, 128, 4),
                                               (777, 72, 136, 64, 2), (130, 1024, 512, 256, 0)])
def test_gemm_wgrad_layout_contracts_over_token_rows(cuda_dev, T, M, N, bn, max_ctas):
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(T + M + N)
    dy = torch.randn(T, M, generator=g).to(cuda_dev, bf16)
    x = torch.randn(T, N, generator=g).to(cuda_dev, bf16)
    ref = dy.float().t() @ x.float()
    gw = torch.full((M, N), 7.0, dtype=f32, device=cuda_dev)
    ops.gemm(dy, x, out=gw, layout=2, block_n=bn, max_ctas=max_ctas)       # fresh gradient: written, not accumulated
    assert rel(gw, ref) < 1e-4
    ops.wgrad_(dy, x, gw, accumulate=True)                                # second contribution: +=
    assert rel(gw, 2 * ref) < 1e-4
    # strided views (column blocks of a fused activation buffer), as the engine passes them
    buf = torch.randn(T, M + 64, generator=g).to(cuda_dev, bf16)
    gw2 = torch.empty(M, N, dtype=f32, device=cuda_dev)
    ops.wgrad_(buf[:, :M], x, gw2, accumulate=False)
    assert rel(gw2, buf[:, :M].float().t() @ x.float()) < 1e-4


def test_col_reduce_bias_and_norm_gradients(cuda_dev):
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    for M, H in ((1000, 384), (77, 1024), (5000, 132)):
        dya = torch.randn(M, H, generator=g).to(cuda_dev)
        dyb = torch.randn(M, H + 8, generator=g).to(cuda_dev, bf16)[:, :H]
        z = torch.randn(M, H, generator=g).to(cuda_dev) * 2 + 0.3
        mean, var = z.mean(1), z.var(1, unbiased=False)
        rstd = (var + 1e-5).rsqrt()
        dy = dya + dyb.float()
        zh = (z - mean[:, None]) * rstd[:, None]
        s, p = torch.zeros(H, device=cuda_dev), torch.ones(H, device=cuda_dev)
        ops.col_reduce_(dy_f32=dya, dy_bf16=dyb, z=z, mean=mean, rstd=rstd, out_sum=s, out_prod=p)
        assert rel(s, dy.sum(0)) < 1e-5 and rel(p - 1, (dy * zh).sum(0)) < 1e-4
        # bias gradient: bf16 only; RMSNorm gain: no mean
        s2 = torch.zeros(H, device=cuda_dev)
        ops.col_reduce_(dy_bf16=dyb, out_sum=s2)
        assert rel(s2, dyb.float().sum(0)) < 1e-5
        p2 = torch.zeros(H, device=cuda_dev)
        ops.col_reduce_(dy_bf16=dyb, z=z, rstd=rstd, out_prod=p2)
        assert rel(p2, (dyb.float() * z * rstd[:, None]).sum(0)) < 1e-4


def test_embed_scatter_add_and_masked_add(cuda_dev):
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(6)
    B, L, H, V = 7, 12, 64, 50
    d = torch.randn(B * L, H, generator=g).to(cuda_dev)
    ids = torch.randint(0, V, (B, L), generator=g).to(cuda_dev)
    dw, dp = torch.zeros(V, H, device=cuda_dev), torch.zeros(32, H, device=cuda_dev)
    ops.embed_scatter_add_(d, ids, dw, dp, L)
    rw = torch.zeros(V, H, device=cuda_dev).index_add_(0, ids.view(-1), d)
    rp = torch.zeros(32, H, device=cuda_dev)
    rp[:L] = d.view(B, L, H).sum(0)
    assert rel(dw, rw) < 1e-6 and rel(dp, rp) < 1e-6
    a = torch.randn(B * L, H, generator=g).to(cuda_dev)
    b = torch.randn(B * L, H, generator=g).to(cuda_dev, bf16)
    drop = ops.Drop(0.1, 1234, 99, None)
    mask = ops.dropout_scale(B * L * H, drop, cuda_dev).view(B * L, H)
    out = ops.masked_add(a, b, drop=drop)
    assert torch.equal(out, (a + b.float()) * mask)
    assert 0.05 < (mask == 0).float().mean().item() < 0.15
    assert torch.equal(ops.masked_add(a, b, drop=None), a + b.float())


def test_adam_shadow_matches_torch_adam(cuda_dev):
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(7)
    n = 4096 + 64
    p0 = torch.randn(n, generator=g)
    p = p0.clone().to(cuda_dev); m = torch.zeros_like(p); v = torch.zeros_like(p)
    shadow = torch.zeros(n, dtype=bf16, device=cuda_dev)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-2)
    for step in range(1, 4):
        grad = torch.randn(n, generator=g)
        ref.grad = grad.clone()
        opt.step()
        ops.adam_step_shadow_(p, grad.to(cuda_dev), m, v, shadow, 1e-2, 0.9, 0.999, 1e-8, step)
    assert (p.cpu() - ref.detach()).abs().max().item() < 1e-5
    assert torch.equal(shadow, p.to(bf16))


# ---------------------------------------------------------------------------------------------------------------
# whole-step parity: every parameter's gradient
# ---------------------------------------------------------------------------------------------------------------
def test_full_finetune_rag_step_gradients_match_oracle(cuda_dev):
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import fused_rag_step
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 504, r16, lora_r=False, lora_g=False)
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=21)
    opt = FusedAdam(model.parameters(), lr=1e-3)
    ref, out = rag_step_vs_oracle(model, enc, dec, bert, llama, batch)
    n_r = compare_full_grads(enc, ref["grads"], "retriever.")
    n_g = compare_full_grads(dec, ref["grads"], "generator.")
    assert n_r > 30 and n_g > 15
    # a second backward without zero_grad accumulates (un-fused API path / gradient accumulation)
    g1r, g1g = enc.full.g32.clone(), dec.full.g32.clone()
    fused_rag_step(model, batch, 100.0)
    assert rel(enc.full.g32, 2 * g1r) < 1e-3 and rel(dec.full.g32, 2 * g1g) < 1e-3
    # zero_grad + step again gives the single-step gradient back (fresh wgrads overwrite, atomics start from zero)
    opt.zero_grad()
    fused_rag_step(model, batch, 100.0)
    assert rel(enc.full.g32, g1r) < 1e-3 and rel(dec.full.g32, g1g) < 1e-3
    # Adam: master weights move like torch.optim.Adam on the oracle's gradients; the bf16 shadow follows the master
    w_before = dec.full.w32("L0.Wqkv").clone()
    opt.step()
    delta = dec.full.w32("L0.Wqkv") - w_before
    gq = ref["grads"]["generator.model.layers.0.self_attn.q_proj.weight"].to(cuda_dev)
    rows = gq.shape[0]
    big = gq.abs() > gq.abs().max() * 0.05
    assert (torch.sign(delta[:rows][big]) == -torch.sign(gq[big])).float().mean().item() > 0.99     # first Adam step = -lr*sign(g)
    assert abs(delta.abs().max().item() - 1e-3) < 1e-5
    assert torch.equal(dec.full.p16, dec.full.p32.to(bf16)) and torch.equal(enc.full.p16, enc.full.p32.to(bf16))
    l0 = out["loss"].item()
    for _ in range(5):
        opt.zero_grad()
        l = fused_rag_step(model, batch, 100.0)["loss"].item()
        opt.step()
    assert l < l0


def test_full_finetune_through_the_reference_style_autograd_loop(cuda_dev):
    """the reference's loop body over the drop-in API with use_peft=None: query and passage batches are two encoder calls,
    so the second backward must accumulate into the first one's weight gradients"""
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import compute_marginalized_loss_from_logits, get_cosine_sim, get_nt_xent_loss
    from oracle import models as om
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 500, r16, lora_r=False, lora_g=False)   # vocab not a multiple of 8:
    batch = rag_batch(4, 10, 20, 32, 600, 500, seed=31)                                                 # padded lm_head rows
    ref = om.rag_step(bert, llama, batch)
    d = {k: v.to(cuda_dev) for k, v in batch.items()}
    opt = FusedAdam(model.parameters(), lr=1e-3)
    opt.zero_grad()
    q = model("retrieval", d["retriever_query_input_ids"], d["retriever_query_attention_mask"])
    p = model("retrieval", d["retriever_passage_input_ids"], d["retriever_passage_attention_mask"])
    S = get_cosine_sim(q, p, 100)
    loss_c = (get_nt_xent_loss(S) + get_nt_xent_loss(S.t())) / 2.0
    lg = model("generation", d["generator_input_input_ids"], d["generator_input_attention_mask"])
    loss = loss_c + compute_marginalized_loss_from_logits(lg, d["generator_input_input_ids"], d["generator_input_attention_mask"],
                                                          S, d["query_passage_input_len"])
    loss.backward()
    assert abs(loss.item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    compare_full_grads(enc, ref["grads"], "retriever.")
    compare_full_grads(dec, ref["grads"], "generator.")


def test_mixed_peft_retriever_lora_generator_full(cuda_dev):
    """`--use-peft retriever`: adapters on the retriever, the generator fully fine-tuned (reference rag_e2e_base_model.py:61-80:
    only the named sub-model goes through get_peft_model)"""
    model, enc, dec, bert, llama = llama_rag_models(cuda_dev, 504, r16, lora_r=True, lora_g=False)
    batch = rag_batch(4, 10, 20, 32, 600, 504, seed=41)
    ref, out = rag_step_vs_oracle(model, enc, dec, bert, llama, batch)
    compare_full_grads(dec, ref["grads"], "generator.")
    worst = lora_grad_error(enc, ref["grads"], "retriever.")
    assert worst < 6e-2, worst
    assert len(model.trainable_banks()) == 2


def test_full_finetune_retriever_only_with_dropout_and_graph(cuda_dev):
    """train() mode (hidden / attention dropout on, incl. the embedding dropout whose gradient is masked) under a CUDA graph:
    loss decreases and the graph's gradients equal the eager ones for the same dropout stream"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_retriever_step
    bcfg = synthetic.bert_config("bge-tiny", 600)
    enc = BertEncoder(bcfg, params.random_state_dict("bert", bcfg, seed=3), device=cuda_dev, full=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    rb = retriever_batch(rag_batch(6, 12, 24, 8, 600, 504, seed=51))
    se.train()
    opt = FusedAdam(se.parameters(), lr=2e-4)
    graphed = GraphedStep(fused_retriever_step, se, rb, 100.0, zero_grads=opt.zero_grad)
    losses = []
    for i in range(12):
        opt.zero_grad()
        losses.append(graphed(rb)["loss"].item())
        opt.step()
    assert losses[-1] < losses[0], losses
    assert all(torch.isfinite(torch.tensor(losses)))
    assert torch.isfinite(enc.full.g32).all()


def test_full_finetune_trainer_end_to_end_and_resume(cuda_dev, tmp_path):
    """`dalm train-retriever-only --no-use-peft` and `dalm train-rag-e2e` without --use-peft on a toy CSV: save_pretrained
    artefacts (config.json + model.safetensors under HF names) that reload into HF classes with moved weights"""
    from safetensors.torch import load_file
    from dalm_b200 import synthetic
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    from dalm_b200.training.retriever_only.train_retriever_only import train_retriever
    from oracle import models as om
    csv = synthetic.write_csv(str(tmp_path / "toy.csv"), 12, seed=5)
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=904)
    out = str(tmp_path / "out_ret")
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out, use_peft=False, use_bnb=False, with_tracking=False, checkpointing_steps="3")
    sd = load_file(os.path.join(out, "retriever", "model.safetensors"))
    sd0 = load_file(os.path.join(rdir, "model.safetensors"))
    moved = [k for k in sd0 if k in sd and not k.startswith("pooler") and (sd[k].float() - sd0[k].float()).abs().max() > 0]
    assert len(moved) > 30                                                    # weights, biases, LayerNorms, embeddings all moved
    import json
    om.build_bert(json.load(open(os.path.join(out, "retriever", "config.json"))), sd)          # loads into HF BertModel
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out, use_peft=False, use_bnb=False, with_tracking=False,
                    resume_from_checkpoint=os.path.join(out, "step_3"))
    out2 = str(tmp_path / "out_e2e")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64,
              num_train_epochs=1, output_dir=out2, use_peft=None, num_warmup_steps=1, with_tracking=False)
    gsd = load_file(os.path.join(out2, "generator", "model.safetensors"))
    g0 = load_file(os.path.join(gdir, "model.safetensors"))
    assert sum((gsd[k].float() - g0[k].float()).abs().max() > 0 for k in g0) == len(g0)
    om.build_llama(json.load(open(os.path.join(out2, "generator", "config.json"))), gsd)


def test_falcon_full_finetune_with_recompute_matches_oracle(cuda_dev):
    """BASELINE config 5 family at toy size with the reference's semantics for `--use-peft retriever`: LoRA retriever, Falcon
    generator FULLY fine-tuned (MQA attention backward, parallel attn+MLP block, tied head). The backward recomputes every
    layer from its saved input; every Falcon parameter's gradient is checked against HF FalconForCausalLM autograd."""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.falcon import FalconDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_rag_step
    from oracle import models as om
    bcfg, fcfg = synthetic.bert_config("bge-tiny", 600), synthetic.falcon_config("falcon-tiny", 504)
    bsd, fsd = r16(params.random_state_dict("bert", bcfg, seed=21)), r16(params.random_state_dict("falcon", fcfg, seed=22))
    enc, dec = BertEncoder(bcfg, bsd, device=cuda_dev, lora=True), FalconDecoder(fcfg, fsd, device=cuda_dev, full=True)
    draw_lora_B(enc, torch.Generator().manual_seed(23))
    model = AutoModelForRagE2E("", "", get_peft=Mode.RETRIEVER, _retriever=enc, _generator=dec, _load_tokenizers=False)
    batch = rag_batch(4, 10, 20, 48, 600, 504, seed=24)
    bert, falcon = om.build_bert(bcfg, bsd), om.build_falcon(fcfg, fsd)
    attach_lora(bert, enc)
    ref = om.rag_step(bert, falcon, batch)
    opt = FusedAdam(model.parameters(), lr=1e-3)
    opt.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    worst, checked = ("", 0.0), 0
    for key, _, name in dec._names:
        rg = ref["grads"]["generator." + name]
        extra = ref["grads"].get("generator.lm_head.weight")
        if name == "transformer.word_embeddings.weight" and extra is not None and extra.data_ptr() != rg.data_ptr():
            rg = rg + extra                                                        # untied in the oracle build: sum of both uses
        e = rel(dec.full.g(key), rg)
        checked += 1
        if e > worst[1]:
            worst = (name, e)
    assert worst[1] < 6e-2 and checked == 3 + 6 * fcfg["num_hidden_layers"], (worst, checked)
    w = lora_grad_error(enc, ref["grads"], "retriever.")
    assert w < 6e-2, w
    # training under a CUDA graph (recomputation inside the captured backward) decreases the loss
    graphed = GraphedStep(fused_rag_step, model, batch, 100.0, zero_grads=opt.zero_grad)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        losses.append(graphed(batch)["loss"].item())
        opt.step(); enc.repack_lora()
    assert losses[-1] < losses[0], losses
    sd = dec.hf_state_dict()
    assert torch.equal(sd["lm_head.weight"], sd["transformer.word_embeddings.weight"]) and len(sd) == 4 + 6 * fcfg["num_hidden_layers"]
