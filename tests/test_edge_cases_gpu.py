"""-m gpu: edge cases — single-sample batches, length-1 sequences, ragged tiles, fully masked rows, rejected empty inputs."""
import pytest
import torch

from model_helpers import rel

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


def test_single_sample_batch_losses(cuda_dev):
    """B = 1: the in-batch softmax has one entry, so both contrastive terms and the doc log-prob are exactly 0"""
    from dalm_b200 import ops
    from oracle import losses
    g = torch.Generator().manual_seed(0)
    q = torch.nn.functional.normalize(torch.randn(1, 64, generator=g), dim=1)
    p = torch.nn.functional.normalize(torch.randn(1, 64, generator=g), dim=1)
    L, V = 7, 40
    logits = torch.randn(1, L, V, generator=g); ids = torch.randint(0, V, (1, L), generator=g)
    mask = torch.ones(1, L, dtype=torch.int64); qlen = torch.tensor([3])
    ref = losses.rag_loss_and_grads(q, p, 100.0, logits, ids, mask, qlen)
    dev = cuda_dev
    cvec, nsum = ops.marginal_counts(mask.to(dev), qlen.to(dev))
    r = ops.inbatch_loss(q.to(dev), p.to(dev), 100.0, cvec, nsum)
    assert r["losses"][0].item() == 0.0 and r["dlp"][0].item() == 0.0
    assert r["dQ"].abs().max().item() == 0.0 and r["dP"].abs().max().item() == 0.0
    tok_lp, dl = ops.ce_marginal(logits.to(dev), ids.to(dev), mask.to(dev), nsum)
    out = ops.finalize_loss(tok_lp, mask.to(dev), nsum, r["losses"])
    assert abs(out[2].item() - ref["loss"].item()) < 1e-5 * abs(ref["loss"].item())
    assert rel(dl, ref["dlogits"]) < 1e-5


def test_fully_masked_and_single_position(cuda_dev):
    from dalm_b200 import ops
    from oracle import losses
    dev = cuda_dev
    g = torch.Generator().manual_seed(1)
    B, L, V = 3, 5, 33                      # V odd: scalar (unvectorised) CE path
    logits = torch.randn(B, L, V, generator=g); ids = torch.randint(0, V, (B, L), generator=g)
    mask = torch.zeros(B, L, dtype=torch.int64); mask[1, 2] = 1          # exactly one scored position in the batch
    qlen = torch.tensor([1, 9, 2])
    S = torch.randn(B, B, generator=g)
    want = losses.marginalized_loss_loopform(logits, ids, mask, S, qlen)
    cvec, nsum = ops.marginal_counts(mask.to(dev), qlen.to(dev))
    assert nsum.item() == 1.0
    tok_lp, dl = ops.ce_marginal(logits.to(dev), ids.to(dev), mask.to(dev), nsum)
    lm = -(tok_lp[1, 1]).item()                                            # t = 1 predicts position 2
    dlp = torch.log_softmax(S, 1).diag()
    assert abs(lm - (cvec.cpu() * dlp).sum().item() - want.item()) < 1e-4
    assert dl[0].abs().max().item() == 0 and dl[2].abs().max().item() == 0 and dl[1, [0, 2, 3, 4]].abs().max().item() == 0


def test_length_one_sequences_and_single_row_gemm(cuda_dev):
    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from oracle import models as om
    cfg = synthetic.bert_config("bge-tiny", vocab_size=300)
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in params.random_state_dict("bert", cfg, seed=3).items()}
    enc = BertEncoder(cfg, sd, device=cuda_dev, lora=False)
    ref = om.build_bert(cfg, sd)
    ids = torch.tensor([[7]]); mask = torch.ones(1, 1, dtype=torch.int64)              # B = 1, L = 1
    hid, _ = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert rel(hid, ref(ids, mask)[0]) < 1e-2
    a = torch.randn(1, 64, device=cuda_dev).to(bf16); b = torch.randn(8, 64, device=cuda_dev).to(bf16)
    assert rel(ops.gemm(a, b, out_dtype=f32), a.float() @ b.float().t()) < 1e-5


@pytest.mark.parametrize("L", [1, 5, 127, 129, 257])
def test_tc_attention_ragged_lengths(cuda_dev, L):
    from dalm_b200 import ops
    B, H, D = 2, 2, 128
    torch.manual_seed(L)
    qkv = torch.randn(B * L, 3 * H * D, device=cuda_dev).to(bf16)
    q, k, v = qkv[:, :H * D], qkv[:, H * D:2 * H * D], qkv[:, 2 * H * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=cuda_dev)
    o1, l1 = ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, True)
    o2, l2 = ops.attention_fwd(q, k, v, mask, B, L, H, H, D, True)
    assert rel(o1.float(), o2.float()) < 1.5e-2 and (l1 - l2).abs().max().item() < 2e-2
    do = torch.randn_like(o1)
    g1 = ops.attention_tc_bwd(q, k, v, mask, o1, l1, do, B, L, H, H, D, True)
    g2 = ops.attention_bwd(q, k, v, mask, o1, l1, do, B, L, H, H, D, True)
    for a, b in zip(g1, g2):
        if b.float().norm().item() < 1e-3:                    # L = 1: dq = dk = 0 analytically (softmax of one entry); compare absolutely
            assert (a.float() - b.float()).abs().max().item() < 1e-5
        else:
            assert rel(a.float(), b.float()) < 3e-2


def test_empty_inputs_are_rejected(cuda_dev):
    from dalm_b200 import ops, _lib
    z = torch.zeros(0, 16, device=cuda_dev)
    with pytest.raises(_lib.DalmB200Error):
        ops.inbatch_loss(z, z, 100.0)
    with pytest.raises(_lib.DalmB200Error):
        ops.gemm(torch.zeros(0, 16, device=cuda_dev, dtype=bf16), torch.zeros(8, 16, device=cuda_dev, dtype=bf16))
    with pytest.raises(_lib.DalmB200Error):
        ops.inbatch_loss(torch.zeros(3, 16, device=cuda_dev), torch.zeros(2, 16, device=cuda_dev), 100.0)   # ragged: |Q| != |P|
    from dalm_b200.training.utils.train_utils import compute_marginalized_loss_from_logits
    with pytest.raises(ValueError):                                                      # zip(strict=True) in the reference
        compute_marginalized_loss_from_logits(torch.zeros(2, 4, 8, device=cuda_dev), torch.zeros(2, 4, dtype=torch.int64, device=cuda_dev),
                                              torch.ones(2, 4, dtype=torch.int64, device=cuda_dev), torch.zeros(3, 3, device=cuda_dev),
                                              torch.ones(2, dtype=torch.int64, device=cuda_dev))
