"""-m gpu: encoder / decoder forward+backward of the engine against the CPU fp32 oracle (HF modeling code + LoRA
restatement, oracle/models.py) on identical seeded weights and inputs.

Tolerance (north_star): <= 1e-3 relative on the fp32 loss under bf16 forward. Hidden states / logits are compared in
relative L2 norm with bf16-forward budgets written at each check; LoRA gradients likewise."""
import pytest
import torch

from model_helpers import attach_lora, check_decoder, draw_lora_B, hf_grads, lora_grad_error, r16_2d, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,B,L", [("bge-tiny", 3, 20), ("bge-small-en", 2, 50)])
def test_bert_encoder_fwd_bwd(cuda_dev, name, B, L):
    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from oracle import models as om, pooling
    cfg = synthetic.bert_config(name, vocab_size=1000)
    sd = params.random_state_dict("bert", cfg, seed=1)
    # the engine stores matmul weights in bf16: give the oracle the same (bf16-rounded) values so the comparison
    # isolates arithmetic, not weight quantisation
    sd = r16_2d(sd)
    enc = BertEncoder(cfg, sd, device=cuda_dev, lora=True)
    g = torch.Generator().manual_seed(5)
    draw_lora_B(enc, g)
    ref = om.build_bert(cfg, sd)
    attach_lora(ref, enc)
    ids = torch.randint(5, 1000, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    mask[0, L - 6:] = 0
    hid, ctx = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev))
    ref_hid = ref(ids, mask)[0]
    valid = mask.bool()
    # bf16 GEMM operands through N layers: budget 1e-2 relative on the hidden states of valid tokens
    assert rel(hid.cpu()[valid], ref_hid[valid]) < 1e-2
    emb, norm = ops.pool_norm_fwd(hid, mask.to(cuda_dev), True)
    ref_emb = pooling.normalize(pooling.mean_pooling(ref_hid, mask))
    assert rel(emb, ref_emb) < 5e-3
    # backward from a random embedding gradient
    d_emb = torch.randn(B, cfg["hidden_size"], generator=g)
    ref_emb.backward(d_emb)
    d_hid = ops.pool_norm_bwd(emb, norm, d_emb.to(cuda_dev), mask.to(cuda_dev), L, True)
    enc.lora.zero_grad()
    enc.backward_hidden(ctx, d_hid)
    worst = lora_grad_error(enc, hf_grads(ref))
    # gradients flow through bf16 activations/gradients: budget 5e-2 relative per factor
    assert worst < 5e-2, worst


@pytest.mark.parametrize("name,B,L,pad", [("llama-tiny", 3, 24, "right"), ("llama-tiny", 2, 40, "left"), ("llama-mini", 2, 64, "right"),
                                           ("llama-hd128", 2, 150, "right"), ("llama-hd128", 2, 72, "left")])
def test_llama_decoder_fwd_bwd(cuda_dev, name, B, L, pad):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    cfg = synthetic.llama_config(name, vocab_size=512)
    sd = r16_2d(params.random_state_dict("llama", cfg, seed=2))
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    g = torch.Generator().manual_seed(9)
    draw_lora_B(dec, g)
    ref = om.build_llama(cfg, sd)
    attach_lora(ref, dec)
    check_decoder(dec, ref, g, 512, B, L, pad)                            # the ids continue the LoRA draws' generator


@pytest.mark.parametrize("name,B,L,pad", [("falcon-tiny", 3, 40, "right"), ("falcon-mini", 2, 130, "left")])
def test_falcon_decoder_forward(cuda_dev, name, B, L, pad):
    """BASELINE config 5's generator family (parallel attention + MLP, MQA, LayerNorm, GELU, tied lm_head): logits and
    the marginalised loss vs HF FalconForCausalLM; adapters are refused like peft would refuse them"""
    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.falcon import FalconDecoder
    from oracle import models as om, losses
    cfg = synthetic.falcon_config(name, vocab_size=504)
    sd = r16_2d(params.random_state_dict("falcon", cfg, seed=4))
    dec = FalconDecoder(cfg, sd, device=cuda_dev)
    with pytest.raises(ValueError):
        FalconDecoder(cfg, sd, device=cuda_dev, lora=True)
    ref = om.build_falcon(cfg, sd)
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(3, 504, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    if pad == "right": mask[0, L - 7:] = 0
    else: mask[0, :6] = 0
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev))
    with torch.no_grad():
        ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2
    S = torch.randn(B, B, generator=g) * 3
    qlen = torch.tensor([3, L // 2, L + 2][:B])
    want = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    got = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(got.item() - want.item()) / abs(want.item()) < 1e-3
