"""-m gpu: dropout (the reference trains under model.train(): BERT hidden / attention-prob dropout 0.1, LoRA input dropout
0.05). Masks are counter-based (Philox) and never stored, so they can be extracted with `ops.dropout_scale` and applied
identically in a torch reference: every dropout site is checked EXACTLY (same mask), plus the statistics of the generator,
plus the whole encoder in train() mode against HF modeling code with torch.nn.functional.dropout patched to replay our masks."""
import math

import pytest
import torch

from model_helpers import rel

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


def test_generator_statistics_and_counters(cuda_dev):
    from dalm_b200 import ops
    n = 1 << 20
    off = torch.zeros(1, dtype=torch.int64, device=cuda_dev)
    d = ops.Drop(0.1, 1234, 77, off)
    m1 = ops.dropout_scale(n, d, cuda_dev)
    vals = torch.unique(m1)
    assert vals.numel() == 2 and vals[0].item() == 0.0 and abs(vals[1].item() - 1 / 0.9) < 1e-4   # p quantised to 1/65536
    keep = (m1 > 0).float().mean().item()
    assert abs(keep - 0.9) < 3e-3                                  # ~10 sigma of a Bernoulli(0.9) over 2^20 draws
    assert abs(m1.mean().item() - 1.0) < 5e-3                      # unbiased: E[scale] = 1
    assert torch.equal(m1, ops.dropout_scale(n, d, cuda_dev))      # deterministic
    m2 = ops.dropout_scale(n, ops.Drop(0.1, 1234, 78, off), cuda_dev)
    assert 0.75 < ((m1 > 0) == (m2 > 0)).float().mean().item() < 0.9          # independent streams agree ~ 0.82
    ops.bump_counter_(off)
    assert off.item() == 1
    m3 = ops.dropout_scale(n, d, cuda_dev)
    assert not torch.equal(m1, m3)                                 # a bumped step counter draws a fresh mask
    assert torch.equal(ops.dropout_scale(n, ops.Drop(0.0, 1, 1, None), cuda_dev), torch.ones(n, device=cuda_dev))


def test_gemm_and_layernorm_sites_exact(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(0)
    dev = cuda_dev
    M, N, K = 300, 264, 192
    a = (torch.randn(M, K, device=dev) * 0.3).to(bf16); b = (torch.randn(N, K, device=dev) * 0.3).to(bf16)
    bias = torch.randn(N, device=dev); res = torch.randn(M, N, device=dev)
    d = ops.Drop(0.1, 99, 5 << 8 | 1, None)
    out = ops.gemm(a, b, out_dtype=f32, bias=bias, resid=res, drop=d)
    mask = ops.dropout_scale(M * N, d, dev).view(M, N)
    ref = (a.float() @ b.float().t() + bias) * mask + res          # dropout(dense) + residual (BertSelfOutput)
    assert rel(out, ref) < 1e-5
    for bn in (64, 128, 2128):
        assert rel(ops.gemm(a, b, out_dtype=f32, bias=bias, resid=res, drop=d, block_n=bn), ref) < 1e-5
    # layernorm: forward output dropout, backward bf16-branch mask
    for H in (256, 1024, 384):                                     # warp-per-row kernels (256, 1024) and the CTA-per-row ones (384)
        z = torch.randn(M, H, device=dev); g = torch.randn(H, device=dev); be = torch.randn(H, device=dev)
        d0 = ops.Drop(0.1, 99, 7, None)
        y32, y16, mean, rstd = ops.layernorm_fwd(z, g, be, 1e-12, drop=d0)
        m0 = ops.dropout_scale(M * H, d0, dev).view(M, H)
        assert rel(y32, torch.nn.functional.layer_norm(z, (H,), g, be, 1e-12) * m0) < 1e-5
        dy = torch.randn(M, H, device=dev)
        dz32, dz16 = ops.layernorm_bwd(z, g, mean, rstd, dy_f32=dy, drop16=d0)
        dz32b, dz16b = ops.layernorm_bwd(z, g, mean, rstd, dy_f32=dy)
        assert torch.equal(dz32, dz32b)                                # residual branch unmasked
        assert rel(dz16.float(), dz32 * m0) < 4e-3                    # dense branch = mask * dz / (1-p)


@pytest.mark.parametrize("B,L,H,D", [(2, 50, 4, 64), (3, 37, 2, 32)])
def test_attention_probability_dropout_exact(cuda_dev, B, L, H, D):
    from dalm_b200 import ops
    torch.manual_seed(1)
    dev = cuda_dev
    qkv = torch.randn(B * L, 3 * H * D, device=dev).to(bf16)
    q, k, v = qkv[:, :H * D], qkv[:, H * D:2 * H * D], qkv[:, 2 * H * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev); mask[0, L - 4:] = 0
    d = ops.Drop(0.1, 5, 3 << 8 | 8, None)
    out, lse = ops.attention_fwd(q, k, v, mask, B, L, H, H, D, False, drop=d)
    Lp = (L + 7) // 8 * 8                                           # mask rows are pitched to a Philox group of 8
    dm = ops.dropout_scale(B * H * L * Lp, d, dev).view(B, H, L, Lp)[..., :L].double()
    qd, kd, vd = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    qh = qd.view(B, L, H, D).transpose(1, 2); kh = kd.view(B, L, H, D).transpose(1, 2); vh = vd.view(B, L, H, D).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2) / math.sqrt(D)).masked_fill(mask.view(B, 1, 1, L) == 0, float("-inf"))
    ref = ((torch.softmax(s, -1) * dm) @ vh).transpose(1, 2).reshape(B * L, H * D)
    assert rel(out.float(), ref) < 1.5e-2
    do = torch.randn(B * L, H * D, device=dev).to(bf16)
    ref.backward(do.double())
    dq, dk, dv = ops.attention_bwd(q, k, v, mask, out, lse, do, B, L, H, H, D, False, drop=d)
    assert rel(dq.float(), qd.grad) < 3e-2 and rel(dk.float(), kd.grad) < 3e-2 and rel(dv.float(), vd.grad) < 3e-2


def test_lora_input_dropout_sites_exact(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(2)
    dev = cuda_dev
    M, K, R = 700, 512, 16
    buf = torch.zeros(M, K + 64, device=dev, dtype=bf16); buf[:, :K] = (torch.randn(M, K, device=dev) * 0.5).to(bf16)
    x = buf[:, :K]
    a_stack = (torch.randn(64, K, device=dev) * 0.3).to(bf16)
    d = ops.Drop(0.05, 11, 2 << 8 | 3, None)
    xm = x.float() * ops.dropout_scale(M * K, d, dev).view(M, K)
    ops.skinny_gemm(x, a_stack, buf[:, K:], K=K, R=R, dropx=d)
    assert rel(buf[:, K:K + R].float(), xm @ a_stack[:R].float().t()) < 5e-3
    g = (torch.randn(M, R, device=dev) * 0.2).to(bf16)
    o0 = torch.zeros(8, K, device=dev); o1 = torch.zeros(8, K, device=dev)
    ops.lora_wgrad_(x, g, o0, K, 1, K, R, 1.0, out1=o1, dropx=d)
    xm16 = xm.to(bf16).float()                                     # the kernel masks the bf16 tile before the MMA
    assert rel(o0, g[:, :8].float().t() @ xm16) < 1e-4 and rel(o1, g[:, 8:].float().t() @ xm16) < 1e-4
    dh = (torch.randn(M, K, device=dev) * 0.1).to(bf16)
    ref = dh.float() + ops.dropout_scale(M * K, d, dev).view(M, K) * (g.float() @ a_stack[:R].float())
    ops.lora_dx_(dh, g, a_stack, K=K, R=R, drop=d)
    assert rel(dh.float(), ref) < 4e-3


def test_bert_encoder_train_mode_matches_hf_with_replayed_masks(cuda_dev, monkeypatch):
    """the whole encoder forward + LoRA backward in train() mode vs HF BertModel (eager attention) whose
    torch.nn.functional.dropout is patched to replay OUR masks in call order"""
    from dalm_b200 import ops, synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from oracle import models as om, pooling
    cfg = dict(synthetic.bert_config("bge-tiny", vocab_size=800), _attn_implementation="eager")
    sd = params.random_state_dict("bert", cfg, seed=3)
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}
    enc = BertEncoder(cfg, sd, device=cuda_dev, lora=True)
    g = torch.Generator().manual_seed(4)
    for n, _, _ in enc.lora.specs:
        enc.lora.B[n].copy_((torch.randn(enc.lora.B[n].shape, generator=g) * 0.02).to(cuda_dev))
    enc.repack_lora()
    enc.train()
    B, L, H, nh = 3, 20, cfg["hidden_size"], cfg["num_attention_heads"]
    ids = torch.randint(5, 800, (B, L), generator=g); mask = torch.ones(B, L, dtype=torch.int64); mask[1, 14:] = 0
    hid, ctx = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev))
    call = ctx.call
    sc = lambda p, layer, site, shape: ops.dropout_scale(int(torch.tensor(shape).prod()), ops.Drop(p, enc.drop_seed, (call << 24) | (layer << 8) | site, enc.drop_offset), cuda_dev).view(shape).cpu()
    Lp = (L + 7) // 8 * 8
    # HF call order: embeddings.dropout; per layer: LoRA dropout for query, key, value (our mask is shared by the three
    # adapters of a layer - documented deviation from peft's independent masks), attention probs, self-output, output
    queue = [sc(enc.p_hidden, 255, 0, (B, L, H))]
    for l in range(enc.nl):
        lm = sc(enc.p_lora, l, 3, (B, L, H))
        queue += [lm, lm, lm, sc(enc.p_attn, l, 8, (B, nh, L, Lp))[..., :L], sc(enc.p_hidden, l, 1, (B, L, H)), sc(enc.p_hidden, l, 2, (B, L, H))]
    ref = om.build_bert(cfg, sd)
    om.attach_lora(ref, {n: {"A": enc.lora.A[n].cpu(), "B": enc.lora.B[n].cpu()} for n, _, _ in enc.lora.specs}, dropout=0.05)
    ref.train()
    used = []

    def replay(x, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return x
        m = queue[len(used)]
        assert tuple(m.shape) == tuple(x.shape), (len(used), m.shape, x.shape)
        used.append(p)
        return x * m.to(x.dtype)
    monkeypatch.setattr(torch.nn.functional, "dropout", replay)
    monkeypatch.setattr(torch, "dropout", lambda x, p, train: replay(x, p, train))
    ref_hid = ref(ids, mask)[0]
    assert len(used) == len(queue)
    valid = mask.bool()
    assert rel(hid.cpu()[valid], ref_hid[valid]) < 1.2e-2
    emb, norm = ops.pool_norm_fwd(hid, mask.to(cuda_dev), True)
    ref_emb = pooling.normalize(pooling.mean_pooling(ref_hid, mask))
    d_emb = torch.randn(B, H, generator=g)
    ref_emb.backward(d_emb)
    enc.lora.zero_grad()
    enc.backward_hidden(ctx, ops.pool_norm_bwd(emb, norm, d_emb.to(cuda_dev), mask.to(cuda_dev), L, True))
    worst = 0.0
    for n, _, _ in enc.lora.specs:
        mod = om._get_module(ref, n)
        worst = max(worst, rel(enc.lora.gA[n], mod.lora_A.grad), rel(enc.lora.gB[n], mod.lora_B.grad))
    assert worst < 6e-2, worst
    # eval() switches every site off again
    enc.eval()
    h2, _ = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    h3, _ = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert torch.equal(h2, h3)


@pytest.mark.parametrize("M,K,R,p", [(333, 200, 8, 0.05), (1000, 1024, 24, 0.05), (130, 4096, 16, 0.05), (64, 2304, 24, 0.0)])
def test_lora_dx_row_widths(cuda_dev, M, K, R, p):
    """dh += mask/(1-p) * (g A) for rows narrower, equal to and wider than one CTA (the launch width follows the row width);
    p = 0 is the un-dropped form the NF4-storage backward uses"""
    from dalm_b200 import ops
    dev = cuda_dev
    g0 = torch.Generator(device="cpu").manual_seed(M + K + R)
    a_stack = (torch.randn(64, K, generator=g0) * 0.3).to(bf16).to(dev)
    g = (torch.randn(M, R, generator=g0) * 0.2).to(bf16).to(dev)
    dh = (torch.randn(M, K, generator=g0) * 0.1).to(bf16).to(dev)
    d = ops.Drop(p, 11, 2 << 8 | 3, None) if p > 0 else None
    scale = ops.dropout_scale(M * K, d, dev).view(M, K) if d is not None else 1.0
    ref = dh.float() + scale * (g.float() @ a_stack[:R].float())
    ops.lora_dx_(dh, g, a_stack, K=K, R=R, drop=d)
    assert rel(dh.float(), ref) < 4e-3
