"""-m gpu: wgmma/TMA attention (head_dim 128 and 64) against the fp64 torch reference and the mma.sync kernels."""
import math

import pytest
import torch

from model_helpers import rel

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _ref(q, k, v, mask, causal, B, L, Hq, Hkv, D):
    qh = q.double().view(B, L, Hq, D).transpose(1, 2)
    kh = k.double().view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    vh = v.double().view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(D)
    if mask is not None:
        s = s.masked_fill(mask.view(B, 1, 1, L) == 0, float("-inf"))
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(L, L, device=q.device, dtype=torch.bool), 1), float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    return (p @ vh).transpose(1, 2).reshape(B * L, Hq * D)


@pytest.mark.parametrize("B,L,Hq,Hkv,causal,pad", [
    (2, 256, 2, 2, True, "none"), (2, 128, 2, 2, True, "none"), (3, 200, 4, 4, True, "right"), (2, 96, 4, 4, True, "left"),
    (1, 300, 4, 2, True, "right"), (2, 384, 2, 2, False, "right"), (18, 256, 32, 32, True, "none"),
])
def test_attention_tc_forward(cuda_dev, B, L, Hq, Hkv, causal, pad):
    from dalm_b200 import ops
    D = 128
    torch.manual_seed(B * 100 + L)
    dev = cuda_dev
    qkv = torch.randn(B * L, (Hq + 2 * Hkv) * D, device=dev).to(bf16)
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    if pad == "right":
        for b in range(B): mask[b, L - 3 - 5 * b:] = 0
    elif pad == "left":
        for b in range(B): mask[b, :4 + 3 * b] = 0
    out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal)
    out2, lse2 = ops.attention_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal)
    if B * L * Hq <= 20000:
        ref = _ref(q, k, v, mask, causal, B, L, Hq, Hkv, D)
        rows = mask.bool().view(-1) if (causal and pad == "left") else torch.ones(B * L, dtype=torch.bool, device=dev)
        assert rel(out.float()[rows], ref[rows]) < 1.5e-2
        if causal and pad == "left":
            assert out.float()[~rows].abs().max().item() == 0.0
    assert rel(out.float(), out2.float()) < 1.5e-2
    fin = torch.isfinite(lse2)
    assert torch.equal(torch.isfinite(lse), fin)
    assert (lse[fin] - lse2[fin]).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,L,Hq,Hkv,causal,pad", [
    (2, 256, 2, 2, True, "none"), (2, 128, 2, 2, True, "none"), (3, 200, 4, 4, True, "right"), (2, 96, 4, 4, True, "left"),
    (1, 300, 4, 2, True, "right"), (2, 384, 2, 2, False, "right"),
])
def test_attention_tc_backward(cuda_dev, B, L, Hq, Hkv, causal, pad):
    from dalm_b200 import ops
    D = 128
    torch.manual_seed(B * 77 + L)
    dev = cuda_dev
    qkv = torch.randn(B * L, (Hq + 2 * Hkv) * D, device=dev).to(bf16)
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    if pad == "right":
        for b in range(B): mask[b, L - 3 - 5 * b:] = 0
    elif pad == "left":
        for b in range(B): mask[b, :4 + 3 * b] = 0
    out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal)
    qd, kd, vd = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _ref(qd, kd, vd, mask, causal, B, L, Hq, Hkv, D)
    rows = mask.bool().view(-1) if (causal and pad == "left") else torch.ones(B * L, dtype=torch.bool, device=dev)
    d_out = torch.randn(B * L, Hq * D, device=dev).to(bf16)
    d_out[~rows] = 0
    ref.backward(d_out.double())
    dqkv = torch.zeros(B * L, (Hq + 2 * Hkv) * D + 64, device=dev, dtype=bf16)          # outputs are column slices of a wider buffer
    dq, dk, dv = ops.attention_tc_bwd(q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq=dqkv[:, :Hq * D],
                                      dk=dqkv[:, Hq * D:(Hq + Hkv) * D], dv=dqkv[:, (Hq + Hkv) * D:(Hq + 2 * Hkv) * D])
    assert rel(dq.float(), qd.grad) < 3e-2
    assert rel(dk.float(), kd.grad) < 3e-2
    assert rel(dv.float(), vd.grad) < 3e-2
    assert dqkv[:, (Hq + 2 * Hkv) * D:].abs().max().item() == 0
    # and against the mma.sync kernels
    dq2, dk2, dv2 = ops.attention_bwd(q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal)
    assert rel(dq.float(), dq2.float()) < 2e-2 and rel(dk.float(), dk2.float()) < 2e-2 and rel(dv.float(), dv2.float()) < 2e-2


def test_attention_tc_speed_report(cuda_dev, capsys):
    """not an assertion on speed, just a printed comparison at the cfg-3 decoder shape"""
    from dalm_b200 import ops
    B, L, H, D = 18, 256, 32, 128
    dev = cuda_dev
    qkv = torch.randn(B * L, 3 * H * D, device=dev).to(bf16)
    q, k, v = qkv[:, :H * D], qkv[:, H * D:2 * H * D], qkv[:, 2 * H * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)

    def t(fn, n=20):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n): fn()
        e.record(); torch.cuda.synchronize()
        return s.elapsed_time(e) / n * 1e3
    out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, True)
    do = torch.randn_like(out); dq = torch.empty_like(out); dk = torch.empty_like(out); dv = torch.empty_like(out)
    res = {"fwd_tc_us": t(lambda: ops.attention_tc_fwd(q, k, v, mask, B, L, H, H, D, True, out=out)),
           "fwd_mma_us": t(lambda: ops.attention_fwd(q, k, v, mask, B, L, H, H, D, True, out=out)),
           "bwd_tc_us": t(lambda: ops.attention_tc_bwd(q, k, v, mask, out, lse, do, B, L, H, H, D, True, dq=dq, dk=dk, dv=dv)),
           "bwd_mma_us": t(lambda: ops.attention_bwd(q, k, v, mask, out, lse, do, B, L, H, H, D, True, dq=dq, dk=dk, dv=dv))}
    with capsys.disabled():
        print("\nATTN_TC_TIMING", res)


# ----------------------------------------------------------------------------------------------------------------
# head_dim 64: bge-large encoder (bidirectional, key padding, attention-probability dropout) and Falcon (MQA, causal)
# ----------------------------------------------------------------------------------------------------------------
def _ref64(q, k, v, mask, causal, B, L, Hq, Hkv, D, dm=None):
    qh = q.view(B, L, Hq, D).transpose(1, 2)
    kh = k.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    vh = v.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(D)
    if mask is not None:
        s = s.masked_fill(mask.view(B, 1, 1, L) == 0, float("-inf"))
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(L, L, device=q.device, dtype=torch.bool), 1), float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    if dm is not None:
        p = p * dm
    return (p @ vh).transpose(1, 2).reshape(B * L, Hq * D)


@pytest.mark.parametrize("B,L,Hq,Hkv,causal,pad,p_drop", [
    (18, 50, 16, 16, False, "right", 0.0), (18, 128, 16, 16, False, "right", 0.0),        # bge-large query / passage segments
    (5, 50, 16, 16, False, "right", 0.1), (4, 128, 16, 16, False, "right", 0.1),          # ... in train() mode
    (3, 37, 4, 4, False, "none", 0.1), (2, 200, 2, 2, False, "right", 0.1),
    (2, 300, 7, 1, True, "left", 0.0), (1, 2048, 71, 1, True, "none", 0.0),               # Falcon: MQA, causal; 7B head geometry at L 2048
    (2, 384, 4, 2, True, "right", 0.0),
])
def test_attention_tc_head_dim_64(cuda_dev, B, L, Hq, Hkv, causal, pad, p_drop):
    from dalm_b200 import ops
    D = 64
    torch.manual_seed(B * 1000 + L + Hq)
    dev = cuda_dev
    wide = (Hq + 2 * Hkv) * D
    qkv = torch.randn(B * L, wide + 8, device=dev).to(bf16)[:, :wide]                   # strided views of a fused buffer
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    if pad == "right":
        for b in range(B): mask[b, L - 3 - (5 * b) % (L // 2):] = 0
    elif pad == "left":
        for b in range(B): mask[b, :4 + 3 * b] = 0
    d = ops.Drop(p_drop, 77, (5 << 8) | 9, None) if p_drop > 0 else None
    out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, drop=d)
    dm = None
    if d is not None:
        Lp = (L + 7) // 8 * 8
        dm = ops.dropout_scale(B * Hq * L * Lp, d, dev).view(B, Hq, L, Lp)[..., :L].double()
    qd, kd, vd = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _ref64(qd, kd, vd, mask, causal, B, L, Hq, Hkv, D, dm)
    rows = mask.bool().view(-1) if (causal and pad == "left") else torch.ones(B * L, dtype=torch.bool, device=dev)
    assert rel(out.float()[rows], ref[rows]) < 1.5e-2
    if causal and pad == "left":
        assert out.float()[~rows].abs().max().item() == 0.0
    # LSE against the mma.sync kernel's (same definition: natural log, +inf for fully masked rows)
    out2, lse2 = ops.attention_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, drop=d)
    fin = torch.isfinite(lse2)
    assert torch.equal(torch.isfinite(lse), fin) and (lse[fin] - lse2[fin]).abs().max().item() < 2e-2
    assert rel(out.float(), out2.float()) < 1.5e-2                                      # identical dropout masks in both kernels
    d_out = torch.randn(B * L, Hq * D, device=dev).to(bf16)
    d_out[~rows] = 0
    ref.backward(d_out.double())
    dqkv = torch.zeros(B * L, wide + 64, device=dev, dtype=bf16)
    dq, dk, dv = ops.attention_tc_bwd(q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq=dqkv[:, :Hq * D],
                                      dk=dqkv[:, Hq * D:(Hq + Hkv) * D], dv=dqkv[:, (Hq + Hkv) * D:wide], drop=d)
    tol = 3e-2 if Hq // Hkv < 8 else 4e-2                            # MQA sums 71 heads' bf16-rounded P / dS into one dK / dV
    assert rel(dq.float(), qd.grad) < tol
    assert rel(dk.float(), kd.grad) < tol
    assert rel(dv.float(), vd.grad) < tol
    assert dqkv[:, wide:].abs().max().item() == 0


def test_attention_tc_head_dim_64_speed_report(cuda_dev, capsys):
    """printed comparison (no assertion) at the cfg-2 encoder shapes (B 150, 16 x 64, dropout 0.1) and Falcon's (18 x 2048, 71q/1kv)"""
    from dalm_b200 import ops
    dev = cuda_dev

    def t(fn, n=10):
        for _ in range(2): fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n): fn()
        e.record(); torch.cuda.synchronize()
        return round(s.elapsed_time(e) / n * 1e3, 1)
    res = {}
    for tag, (B, L, Hq, Hkv, causal, p) in {"bge_q": (150, 50, 16, 16, False, 0.1), "bge_p": (150, 128, 16, 16, False, 0.1),
                                             "falcon": (4, 2048, 71, 1, True, 0.0)}.items():
        D = 64
        qkv = torch.randn(B * L, (Hq + 2 * Hkv) * D, device=dev).to(bf16)
        q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
        mask = torch.ones(B, L, dtype=torch.int64, device=dev)
        d = ops.Drop(p, 1, 2, None) if p > 0 else None
        out, lse = ops.attention_tc_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, drop=d)
        do = torch.randn_like(out); dq = torch.empty_like(q); dk = torch.empty_like(k); dv = torch.empty_like(v)
        res[tag] = {"fwd_tc_us": t(lambda: ops.attention_tc_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out, drop=d)),
                    "fwd_mma_us": t(lambda: ops.attention_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out, drop=d)),
                    "bwd_tc_us": t(lambda: ops.attention_tc_bwd(q, k, v, mask, out, lse, do, B, L, Hq, Hkv, D, causal, dq=dq, dk=dk, dv=dv, drop=d)),
                    "bwd_mma_us": t(lambda: ops.attention_bwd(q, k, v, mask, out, lse, do, B, L, Hq, Hkv, D, causal, dq=dq, dk=dk, dv=dv, drop=d))}
    with capsys.disabled():
        print("\nATTN_TC64_TIMING", res)
