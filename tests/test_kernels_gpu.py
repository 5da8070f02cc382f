"""-m gpu: every C-ABI kernel against a plain torch fp32/fp64 reference of the same op (floating-point kernels), on
seeded inputs. Tolerances are written next to each check."""
import math

import pytest
import torch

from model_helpers import rel

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32


# ----------------------------------------------------------------------------------------------------------------
# GEMM (wgmma)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,bn", [
    (128, 64, 64, 64), (128, 128, 128, 128), (128, 256, 256, 256),       # single tile per config
    (256, 512, 1024, 0), (900, 1024, 1024, 0), (3204, 3072, 1048, 0),     # ragged M, K-augmented (1024+24)
    (4608, 4096, 4112, 256), (300, 24, 1024, 64), (77, 4096, 512, 128),   # LoRA-down shape N=24, tiny M
    (1000, 1000, 72, 0),                                                  # K tail inside one k-block
    (256, 256, 128, 2256), (256, 128, 64, 2128), (900, 1024, 1048, 2128), (3204, 3072, 1048, 2256),   # CTA-pair kernel
    (4608, 4096, 4112, 2256), (77, 512, 512, 2256), (385, 1032, 520, 2128), (4608, 12288, 4112, 0),
])
def test_gemm_plain(cuda_dev, M, N, K, bn):
    from dalm_b200 import ops
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=cuda_dev) * 0.5).to(bf16)
    b = (torch.randn(N, K, device=cuda_dev) * 0.5).to(bf16)
    out = ops.gemm(a, b, block_n=bn)
    ref = a.float() @ b.float().t()
    # bf16 output rounding: rel 2^-9 per element; accumulate order differs only in fp32
    assert rel(out.float(), ref) < 4e-3
    assert torch.isfinite(out.float()).all()


def test_gemm_multi_tile_per_cta(cuda_dev):
    """force few CTAs so each walks many tiles: exercises the smem ring wrap-around and the parked-accumulator hand-off between tiles"""
    from dalm_b200 import ops
    torch.manual_seed(0)
    M, N, K = 1024, 2048, 768
    a = (torch.randn(M, K, device=cuda_dev) * 0.5).to(bf16)
    b = (torch.randn(N, K, device=cuda_dev) * 0.5).to(bf16)
    ref = a.float() @ b.float().t()
    for bn in (64, 128, 256, 2128, 2256):
        for ctas in (2, 3, 7):
            out = ops.gemm(a, b, block_n=bn, max_ctas=ctas, out_dtype=f32)
            assert rel(out, ref) < 1e-5, (bn, ctas)


def test_gemm_epilogues(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(1)
    M, N, K = 515, 1032, 520
    a = (torch.randn(M, K, device=cuda_dev) * 0.3).to(bf16)
    b = (torch.randn(N, K, device=cuda_dev) * 0.3).to(bf16)
    bias = torch.randn(N, device=cuda_dev)
    r32 = torch.randn(M, N, device=cuda_dev)
    r16 = torch.randn(M, N, device=cuda_dev).to(bf16)
    acc = a.float() @ b.float().t()
    out = ops.gemm(a, b, out_dtype=f32, bias=bias, resid=r32, alpha=0.5)
    assert rel(out, 0.5 * acc + bias + r32) < 1e-5
    out = ops.gemm(a, b, out_dtype=f32, bias=bias, act=1)
    assert rel(out, torch.nn.functional.gelu(acc + bias)) < 1e-5
    out = ops.gemm(a, b, out_dtype=bf16, resid=r16)
    assert rel(out.float(), acc + r16.float()) < 4e-3
    for bn in (2128, 2256):                                   # same epilogue through the CTA-pair kernel
        out = ops.gemm(a, b, out_dtype=f32, bias=bias, resid=r32, alpha=0.5, block_n=bn)
        assert rel(out, 0.5 * acc + bias + r32) < 1e-5
        out = ops.gemm(a, b, out_dtype=f32, bias=bias, act=1, block_n=bn)
        assert rel(out, torch.nn.functional.gelu(acc + bias)) < 1e-5
    # strided views: A and output are column slices of wider buffers (the LoRA K-augmentation layout)
    wide_a = torch.zeros(M, K + 24, device=cuda_dev, dtype=bf16); wide_a[:, :K] = a
    wide_o = torch.zeros(M, N + 40, device=cuda_dev, dtype=bf16)
    ops.gemm(wide_a[:, :K], b, out=wide_o[:, 40:])
    assert rel(wide_o[:, 40:].float(), acc) < 4e-3
    assert wide_o[:, :40].abs().max().item() == 0


def test_gemm_rejects_bad_args(cuda_dev):
    from dalm_b200 import ops, _lib
    a = torch.zeros(16, 12, device=cuda_dev, dtype=bf16)
    b = torch.zeros(16, 12, device=cuda_dev, dtype=bf16)
    with pytest.raises(_lib.DalmB200Error):
        ops.gemm(a, b)                       # K=12 not a multiple of 8
    with pytest.raises(_lib.DalmB200Error):
        ops.gemm(a.cpu(), b.cpu())           # no CPU path


# ----------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------
def _attn_ref(q, k, v, mask, causal, B, L, Hq, Hkv, D):
    # q: [B*L, Hq*D] etc. fp64 reference with the same masking convention (-inf on dropped keys)
    qh = q.double().view(B, L, Hq, D).transpose(1, 2)
    kh = k.double().view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    vh = v.double().view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(D)
    if mask is not None:
        s = s.masked_fill(mask.view(B, 1, 1, L) == 0, float("-inf"))
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(L, L, device=q.device, dtype=torch.bool), 1), float("-inf"))
    p = torch.softmax(s, dim=-1)
    p = torch.nan_to_num(p, nan=0.0)          # fully masked rows -> zero output
    o = (p @ vh).transpose(1, 2).reshape(B * L, Hq * D)
    return o


@pytest.mark.parametrize("B,L,Hq,Hkv,D,causal,pad", [
    (2, 50, 4, 4, 64, False, "right"), (3, 128, 2, 2, 64, False, "right"), (2, 37, 3, 3, 32, False, "right"),
    (2, 256, 2, 2, 128, True, "none"), (2, 200, 4, 4, 128, True, "right"), (2, 96, 4, 4, 128, True, "left"),
    (1, 130, 4, 1, 64, True, "right"),
])
def test_attention_fwd_bwd(cuda_dev, B, L, Hq, Hkv, D, causal, pad):
    from dalm_b200 import ops
    torch.manual_seed(B * 1000 + L)
    dev = cuda_dev
    qkv = (torch.randn(B * L, (Hq + 2 * Hkv) * D, device=dev)).to(bf16)
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    if pad == "right":
        for b in range(B):
            mask[b, L - 3 - 5 * b:] = 0
    elif pad == "left":
        for b in range(B):
            mask[b, :4 + 3 * b] = 0
    out, lse = ops.attention_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal)
    qd, kd, vd = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _attn_ref(qd, kd, vd, mask, causal, B, L, Hq, Hkv, D)
    valid = torch.ones(B, L, dtype=torch.bool, device=dev)
    if causal and pad == "left":
        valid = mask.bool()                   # fully-masked (left pad) query rows: compared separately below
    vrows = valid.view(-1)
    # bf16 P and bf16 output: ~1e-2 relative on the tile
    assert rel(out.float()[vrows], ref[vrows]) < 1.5e-2
    if causal and pad == "left":
        assert out.float()[~vrows].abs().max().item() == 0.0      # fully masked rows produce zeros
    d_out = torch.randn(B * L, Hq * D, device=dev).to(bf16)
    d_out_eff = d_out.clone()
    d_out_eff[~vrows] = 0
    ref.backward(d_out_eff.double())
    dq, dk, dv = ops.attention_bwd(q, k, v, mask, out, lse, d_out_eff, B, L, Hq, Hkv, D, causal)
    assert rel(dq.float(), qd.grad) < 3e-2
    assert rel(dk.float(), kd.grad) < 3e-2
    assert rel(dv.float(), vd.grad) < 3e-2


# ----------------------------------------------------------------------------------------------------------------
# row-wise kernels
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,H", [(333, 1024), (26700, 1024), (77, 384), (130, 256), (9, 2048), (50, 4544), (257, 512), (131, 768)])
def test_layernorm_fwd_bwd(cuda_dev, M, H):
    """H in {256, 512, 1024, 2048} runs the warp-per-row kernels, other widths (bge-small 384, bge-base 768, Falcon 4544) the
    CTA-per-row ones"""
    from dalm_b200 import ops
    torch.manual_seed(2)
    z = torch.randn(M, H, device=cuda_dev) * 2 + 0.3
    g = torch.randn(H, device=cuda_dev); b = torch.randn(H, device=cuda_dev)
    y32, y16, mean, rstd = ops.layernorm_fwd(z, g, b, 1e-12)
    zd = z.double().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(zd, (H,), g.double(), b.double(), 1e-12)
    assert rel(y32, ref) < 1e-5
    assert rel(y16.float(), ref) < 4e-3
    dy_a = torch.randn(M, H, device=cuda_dev)
    dy_b = torch.randn(M, H, device=cuda_dev).to(bf16)
    ref.backward(dy_a.double() + dy_b.double())
    dz32, dz16 = ops.layernorm_bwd(z, g, mean, rstd, dy_f32=dy_a, dy_bf16=dy_b)
    assert rel(dz32, zd.grad) < 1e-4
    assert rel(dz16.float(), zd.grad) < 4e-3
    # pre-LN form (Falcon): the residual's gradient is added to both outputs, in place
    dres = torch.randn(M, H, device=cuda_dev)
    want = zd.grad + dres.double()
    dz32r, dz16r = ops.layernorm_bwd_res(z, g, mean, rstd, dy_b + dy_a.to(bf16) * 0, dres, dz32=dres)
    ref2 = torch.nn.functional.layer_norm(zd.detach().requires_grad_(True), (H,), g.double(), b.double(), 1e-12)
    # (dy_bf16-only variant: recompute the reference for that input)
    zd2 = z.double().requires_grad_(True)
    torch.nn.functional.layer_norm(zd2, (H,), g.double(), b.double(), 1e-12).backward(dy_b.double())
    assert rel(dz32r, zd2.grad + (want - zd.grad)) < 1e-4 and dz32r.data_ptr() == dres.data_ptr()
    assert rel(dz16r.float(), zd2.grad + (want - zd.grad)) < 4e-3


def test_rmsnorm_fwd_bwd(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(3)
    M, H = 257, 4096
    x = torch.randn(M, H, device=cuda_dev) * 1.7
    g = torch.rand(H, device=cuda_dev) + 0.5
    h, rstd = ops.rmsnorm_fwd(x, g, 1e-5)
    xd = x.double().requires_grad_(True)
    ref = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-5) * g.double()
    assert rel(h.float(), ref) < 4e-3
    dh = torch.randn(M, H, device=cuda_dev).to(bf16)
    dres = torch.randn(M, H, device=cuda_dev)
    ref.backward(dh.double())
    out32, out16 = ops.rmsnorm_bwd(x, g, rstd, dh, dres_in=dres)
    assert rel(out32, xd.grad + dres.double()) < 1e-5
    assert rel(out16.float(), xd.grad + dres.double()) < 4e-3


def test_embeddings_rope_swiglu_gelu(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(4)
    dev = cuda_dev
    B, L, H, V = 3, 17, 128, 500
    ids = torch.randint(0, V, (B, L), device=dev)
    word = torch.randn(V, H, device=dev).to(bf16); pos = torch.randn(64, H, device=dev).to(bf16)
    typ = torch.randn(H, device=dev).to(bf16)
    z = ops.bert_embed(ids, word, pos, typ)
    ref = word[ids.view(-1)].float() + pos[torch.arange(L, device=dev).repeat(B)].float() + typ.float()
    assert torch.equal(z, ref)
    x = ops.embed_gather(ids, word)
    assert torch.equal(x, word[ids.view(-1)].float())
    # rope (HF rotate_half convention)
    D, nh = 64, 3
    buf = torch.randn(B * L, nh * D + 8, device=dev).to(bf16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(L, dtype=torch.float32), inv)
    cos_t, sin_t = fr.cos().to(dev), fr.sin().to(dev)
    xh = buf[:, :nh * D].float().view(B, L, nh, D)
    c = torch.cat([cos_t, cos_t], -1)[None, :, None, :]; s = torch.cat([sin_t, sin_t], -1)[None, :, None, :]
    rot = torch.cat([-xh[..., D // 2:], xh[..., :D // 2]], -1)
    ref = (xh * c + rot * s).reshape(B * L, nh * D)
    tail = buf[:, nh * D:].clone()
    work = buf.clone()
    ops.rope_(work, 0, nh, D, cos_t, sin_t, L)
    assert rel(work[:, :nh * D].float(), ref) < 4e-3
    assert torch.equal(work[:, nh * D:], tail)
    ops.rope_(work, 0, nh, D, cos_t, sin_t, L, backward=True)          # inverse rotation restores the input
    assert rel(work[:, :nh * D].float(), buf[:, :nh * D].float()) < 8e-3
    # swiglu
    M, F = 50, 264
    gu = torch.randn(M, 2 * F, device=dev).to(bf16)
    act = ops.swiglu_fwd(gu, F)
    gd = gu.double().requires_grad_(True)
    ref = torch.nn.functional.silu(gd[:, :F]) * gd[:, F:]
    assert rel(act.float(), ref) < 4e-3
    dact = torch.randn(M, F, device=dev).to(bf16)
    ref.backward(dact.double())
    g2 = gu.clone()
    ops.swiglu_bwd_(g2, dact, F)
    assert rel(g2.float(), gd.grad) < 4e-3
    # gelu
    pre = torch.randn(M, F, device=dev).to(bf16)
    a = ops.gelu_fwd(pre)
    pd = pre.double().requires_grad_(True)
    ref = torch.nn.functional.gelu(pd)
    assert rel(a.float(), ref) < 4e-3
    d = torch.randn(M, F, device=dev).to(bf16)
    ref.backward(d.double())
    d2 = d.clone()
    ops.gelu_bwd_(pre, d2)
    assert rel(d2.float(), pd.grad) < 4e-3


@pytest.mark.parametrize("B,L,H", [(5, 23, 384), (18, 128, 1024), (150, 50, 1024), (3, 7, 72), (2, 300, 4096)])
def test_pool_norm(cuda_dev, B, L, H):
    """H % 128 == 0 takes the machine-wide two-launch forward (pool_sum + pool_finish), other widths the per-sample kernel;
    includes a sample with ONE valid token and the golden fixture's all-masked case (clamp 1e-9)"""
    from dalm_b200 import ops
    from oracle import pooling
    torch.manual_seed(5)
    hid = torch.randn(B, L, H, device=cuda_dev)
    mask = torch.ones(B, L, dtype=torch.int64, device=cuda_dev)
    mask[0, min(10, L - 1):] = 0; mask[min(3, B - 1), 1:] = 0
    emb, norm = ops.pool_norm_fwd(hid, mask, True)
    hd = hid.double().cpu().requires_grad_(True)
    ref = pooling.normalize(pooling.mean_pooling(hd, mask.cpu()).double())
    assert rel(emb.cpu(), ref) < 1e-5
    d = torch.randn(B, H, device=cuda_dev)
    ref.backward(d.double().cpu())
    dh = ops.pool_norm_bwd(emb, norm, d, mask, L, True)
    assert rel(dh.cpu(), hd.grad) < 1e-5
    emb2, _ = ops.pool_norm_fwd(hid, mask, False)
    assert rel(emb2.cpu(), pooling.mean_pooling(hid.cpu(), mask.cpu())) < 1e-5


def test_lora_wgrad_pack_adam(cuda_dev):
    from dalm_b200 import ops
    torch.manual_seed(6)
    dev = cuda_dev
    for (M, K) in ((1000, 520), (4608, 4096), (37, 64)):
        x = torch.randn(M, K + 24, device=dev).to(bf16)
        g = torch.randn(M, 40, device=dev).to(bf16)
        out = torch.zeros(8, K, device=dev)
        ops.lora_wgrad_(x[:, :K], g[:, 16:], out, K, 1, K, 8, 2.0)
        ref = 2.0 * g[:, 16:24].double().t() @ x[:, :K].double()
        assert rel(out, ref) < 1e-5, (M, K)
        outT = torch.zeros(K, 8, device=dev)
        ops.lora_wgrad_(x[:, :K], g[:, 16:], outT, 1, 8, K, 8, 2.0)
        ops.lora_wgrad_(x[:, :K], g[:, 16:], outT, 1, 8, K, 8, 2.0)          # accumulates
        assert rel(outT, 2 * ref.t()) < 1e-5
        # two adapters sharing X: rows 0-7 -> out0, rows 8-15 -> out1
        o0 = torch.zeros(8, K, device=dev); o1 = torch.zeros(8, K, device=dev)
        ops.lora_wgrad_(x[:, :K], g[:, 8:], o0, K, 1, K, 16, 1.0, out1=o1)
        assert rel(o0, g[:, 8:16].double().t() @ x[:, :K].double()) < 1e-5
        assert rel(o1, g[:, 16:24].double().t() @ x[:, :K].double()) < 1e-5
    # skinny GEMM: out[M,R] = X W^T written into the tail columns of a wider buffer
    for (M, K, R) in ((4608, 4096, 16), (900, 1024, 24), (33, 72, 8), (300, 512, 32)):
        buf = torch.zeros(M, K + 64, device=dev, dtype=bf16)
        buf[:, :K] = (torch.randn(M, K, device=dev) * 0.5).to(bf16)
        w = (torch.randn(64, K, device=dev) * 0.5).to(bf16)
        ops.skinny_gemm(buf[:, :K], w, buf[:, K:], K=K, R=R)
        ref = buf[:, :K].double() @ w[:R].double().t()
        assert rel(buf[:, K:K + R].float(), ref) < 4e-3, (M, K, R)
        assert buf[:, K + R:].abs().max().item() == 0
    K, R = 520, 8
    # pack
    src = torch.randn(K, R, device=dev)
    dst = torch.zeros(R + 2, K + 8, device=dev, dtype=bf16)
    ops.pack_scaled_bf16_(src, 1, R, dst[1:, 8:], R, K, 2.0)
    assert torch.equal(dst[1:R + 1, 8:], (src.t() * 2.0).to(bf16))
    assert dst[0].abs().max() == 0 and dst[:, :8].abs().max() == 0
    # adam vs torch.optim.Adam
    n = 10007
    p = torch.randn(n, device=dev); p_ref = p.clone().requires_grad_(True)
    m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
    opt = torch.optim.Adam([p_ref], lr=1e-3)
    for step in range(1, 4):
        grad = torch.randn(n, device=dev)
        p_ref.grad = grad.clone()
        opt.step()
        ops.adam_step_(p, grad, m, v, 1e-3, 0.9, 0.999, 1e-8, step)
    assert (p - p_ref.detach()).abs().max().item() < 1e-6


@pytest.mark.parametrize("M,N,K,kind", [(4608, 4096, 1024, "f32+resid"), (1300, 2304, 520, "bf16"), (3204, 1024, 256, "f32+resid"),
                                        (2000, 4096, 192, "f32")])
def test_gemm_rasterisation_orders_give_identical_results(cuda_dev, M, N, K, kind):
    """the tile walk (m-fastest / automatic ~square bands / explicit band heights, serpentine n order) only permutes which
    CTA computes which tile: every order must produce bit-identical outputs, including the register-prefetched fp32 residual"""
    from dalm_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    b = (torch.randn(N, K, generator=g) * 0.1).to(cuda_dev, torch.bfloat16)
    resid = torch.randn(M, N, generator=g).to(cuda_dev) if kind == "f32+resid" else None
    odt = torch.bfloat16 if kind == "bf16" else torch.float32
    lib = _lib.load()
    outs = []
    try:
        for gm in (-1, 0, 1, 5, 7, 64):
            lib.dalm_b200_gemm_set_raster(gm)
            for max_ctas in (0, 13):
                outs.append(ops.gemm(a, b, out_dtype=odt, resid=resid, max_ctas=max_ctas))
    finally:
        lib.dalm_b200_gemm_set_raster(0)
    ref = a.float() @ b.float().t() + (resid if resid is not None else 0)
    assert ((outs[0].float() - ref).norm() / ref.norm()).item() < (5e-3 if kind == "bf16" else 1e-4)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    if resid is not None:                                     # in-place accumulation (out aliases resid), as wgrad uses it
        acc = resid.clone()
        ops.gemm(a, b, out=acc, resid=acc)
        assert torch.equal(acc, outs[0])


@pytest.mark.parametrize("M,F,K", [(300, 256, 192), (4608, 1408, 512), (1000, 11008, 264), (130, 128, 72)])
def test_gemm_with_fused_swiglu_epilogue(cuda_dev, M, F, K):
    """gate|up projection + SiLU(gate)*up in one launch (interleaved 128-feature blocks) == separate GEMM + activation; the
    interleaved gate|up buffer it leaves behind feeds the (interleave-aware) SwiGLU backward"""
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + F + K)
    x = torch.randn(M, K + 8, generator=g).to(cuda_dev, torch.bfloat16)[:, :K]          # strided view, like an augmented buffer
    wg = (torch.randn(F, K, generator=g) * 0.2).to(cuda_dev, torch.bfloat16)
    wu = (torch.randn(F, K, generator=g) * 0.2).to(cuda_dev, torch.bfloat16)
    w_il = ops.interleave_gate_up(wg, wu, 128)
    gu, act = ops.gemm_swiglu(x, w_il)
    gate = x.float() @ wg.float().t()
    up = x.float() @ wu.float().t()
    want = torch.nn.functional.silu(gate) * up
    assert ((act.float() - want).norm() / want.norm()).item() < 5e-3
    # the gate|up output is the plain GEMM result in the interleaved layout
    gu_ref = ops.gemm(x, w_il)
    assert torch.equal(gu, gu_ref)
    blk = gu.float().view(M, F // 128, 2, 128)
    assert ((blk[:, :, 0].reshape(M, F) - gate).norm() / gate.norm()).item() < 5e-3
    assert ((blk[:, :, 1].reshape(M, F) - up).norm() / up.norm()).item() < 5e-3
    # activation kernels on the interleaved layout == on HF's [gate | up] layout
    gu_hf = torch.cat([blk[:, :, 0].reshape(M, F), blk[:, :, 1].reshape(M, F)], 1).to(torch.bfloat16).contiguous()
    assert torch.equal(ops.swiglu_fwd(gu, F, interleave=128), ops.swiglu_fwd(gu_hf, F))
    dact = torch.randn(M, F, generator=g).to(cuda_dev, torch.bfloat16)
    d_il = ops.swiglu_bwd_(gu.clone(), dact, F, interleave=128).float().view(M, F // 128, 2, 128)
    d_hf = ops.swiglu_bwd_(gu_hf.clone(), dact, F).float()
    assert torch.equal(d_il[:, :, 0].reshape(M, F), d_hf[:, :F]) and torch.equal(d_il[:, :, 1].reshape(M, F), d_hf[:, F:])


@pytest.mark.parametrize("B,L,nh,nkv,K", [(2, 24, 2, 2, 136), (18, 256, 4, 4, 264), (3, 150, 6, 2, 72)])
def test_gemm_with_fused_rope_epilogue(cuda_dev, B, L, nh, nkv, K):
    """q|k|v projection with RoPE (head_dim 128) in the GEMM epilogue == plain GEMM followed by the in-place rope kernel"""
    from dalm_b200 import ops
    D = 128
    g = torch.Generator(device="cpu").manual_seed(B * L + K)
    M, N = B * L, (nh + 2 * nkv) * D
    x = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.2).to(cuda_dev, torch.bfloat16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(L, dtype=torch.float32), inv)
    cos_t, sin_t = fr.cos().to(cuda_dev).contiguous(), fr.sin().to(cuda_dev).contiguous()
    rope_cols = (nh + nkv) * D
    if rope_cols % 256:
        with pytest.raises(Exception):
            ops.gemm_rope(x, w, cos_t, sin_t, L, rope_cols)
        return
    fused = ops.gemm_rope(x, w, cos_t, sin_t, L, rope_cols)
    # fp32 reference: rotate_half on the un-rounded projection
    y = (x.float() @ w.float().t()).view(B, L, nh + 2 * nkv, D)
    x1, x2 = y[..., :D // 2], y[..., D // 2:]
    c, s_ = cos_t.view(1, L, 1, D // 2), sin_t.view(1, L, 1, D // 2)
    rot = torch.cat([x1 * c - x2 * s_, x2 * c + x1 * s_], -1)
    want = torch.cat([rot[:, :, :nh + nkv], y[:, :, nh + nkv:]], 2).reshape(M, N)
    assert ((fused.float() - want).norm() / want.norm()).item() < 5e-3
    # and against the two-launch path (which rounds to bf16 before rotating)
    plain = ops.gemm(x, w)
    ops.rope_(plain, 0, nh + nkv, D, cos_t, sin_t, L)
    assert ((fused.float() - plain.float()).norm() / plain.float().norm()).item() < 6e-3
    assert torch.equal(fused[:, rope_cols:], ops.gemm(x, w)[:, rope_cols:])          # v columns untouched


@pytest.mark.parametrize("M,N,K,bias", [(300, 1024, 256, True), (3204, 4096, 1024, True), (260, 72, 136, False), (1000, 18176, 264, False),
                                        (26700, 4096, 1024, True)])
def test_gemm_with_fused_gelu_epilogues(cuda_dev, M, N, K, bias):
    """forward: pre-activation AND gelu(pre) from one launch == GEMM followed by gelu_fwd, bit for bit; backward: the dgrad GEMM
    with act=2 (x gelu'(pre) in the epilogue) == dgrad GEMM followed by gelu_bwd, bit for bit (TN and NN layouts); both against
    an fp32 torch reference (HF BertIntermediate: dense -> gelu(erf))"""
    from dalm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    x = torch.randn(M, K + 8, generator=g).to(cuda_dev, torch.bfloat16)[:, :K]          # strided view
    w = (torch.randn(N, K, generator=g) * 0.15).to(cuda_dev, torch.bfloat16)
    b = torch.randn(N, generator=g).to(cuda_dev) if bias else None
    pre, act = ops.gemm_gelu(x, w, bias=b)
    pre_ref = ops.gemm(x, w, bias=b)
    assert torch.equal(pre, pre_ref)
    assert torch.equal(act, ops.gelu_fwd(pre_ref))
    want = x.float() @ w.float().t() + (b if b is not None else 0)
    assert ((pre.float() - want).norm() / want.norm()).item() < 5e-3
    wa = torch.nn.functional.gelu(want)
    assert ((act.float() - wa).norm() / wa.norm()).item() < 5e-3
    # backward: dy [M,K2] through the output projection W2 [K2, N] (y = act W2^T): d act = dy W2, d pre = d act * gelu'(pre)
    K2 = 136 if M > 20000 else 264
    dy = torch.randn(M, K2, generator=g).to(cuda_dev, torch.bfloat16)
    w2 = (torch.randn(K2, N, generator=g) * 0.1).to(cuda_dev, torch.bfloat16)          # [out=K2, in=N]
    w2T = w2.t().contiguous()
    for kw, wt in ((dict(), w2T), (dict(layout=1), w2)):
        two = ops.gelu_bwd_(pre, ops.gemm(dy, wt, **kw))
        one = ops.gemm(dy, wt, act=2, resid=pre, **kw)
        assert torch.equal(one, two)
    xf = pre.float().requires_grad_(True)
    torch.nn.functional.gelu(xf).backward(dy.float() @ w2.float())
    assert ((one.float() - xf.grad).norm() / xf.grad.norm()).item() < 8e-3
    with pytest.raises(Exception):
        ops.gemm(dy, w2T, act=2)                                      # needs the pre-activation
    with pytest.raises(Exception):
        ops.gemm(dy, w2T, act=2, resid=pre.float())                   # ... in bf16


def test_gemm_l2_hints_and_raster_modes_do_not_change_results(cuda_dev):
    """TMA L2 eviction priorities and the raster rule (automatic / bands everywhere / m-fastest) are performance hints only"""
    from dalm_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(99)
    M, N, K = 2100, 2304, 328
    a = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    b = (torch.randn(N, K, generator=g) * 0.1).to(cuda_dev, torch.bfloat16)
    r = torch.randn(M, N, generator=g).to(cuda_dev)
    bi = torch.randn(N, generator=g).to(cuda_dev)
    wg = ops.interleave_gate_up(b[:1152], b[1152:], 128)
    bT = b.t().contiguous()                                           # [K, N]: the NN layout's B operand
    lib = _lib.load()
    base = None
    try:
        for raster in (0, -2, -1):
            for hints in (0, 1, 2, 4, 7):
                lib.dalm_b200_gemm_set_raster(raster); lib.dalm_b200_gemm_set_l2_hints(hints)
                got = (ops.gemm(a, b), ops.gemm(a, b, out_dtype=torch.float32, resid=r, max_ctas=11), *ops.gemm_swiglu(a, wg),
                       *ops.gemm_gelu(a, b, bias=bi), ops.gemm(a, bT, layout=1))
                if base is None:
                    base = got
                    ref = a.float() @ b.float().t()
                    assert ((got[0].float() - ref).norm() / ref.norm()).item() < 5e-3
                for x, y in zip(got, base):
                    assert torch.equal(x, y)
    finally:
        lib.dalm_b200_gemm_set_raster(0); lib.dalm_b200_gemm_set_l2_hints(-1)
