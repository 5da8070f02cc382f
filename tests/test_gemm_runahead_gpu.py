"""-m gpu: the fused GEMM epilogues (SwiGLU, RoPE, NormRoPE, GELU pair) when every CTA carries several tiles.

The TMA producer loads a tile's first k-blocks while the consumers still run the previous tile's epilogue from their
registers, so each shape here has more tiles than the GPU has SMs, and more k-blocks than the stage ring is deep, so that
the ring's stage and phase carry over between tiles. Inputs and checks follow test_exact_tiles_gpu.py: integer operands,
NaN-poisoned padding, guarded outputs, fp64 references. The fused entry points launch one CTA per SM, so the tile count,
not a CTA cap, is what makes the CTAs walk several tiles.
"""
import pytest
import torch

from exact_helpers import (EPS, STAGES, Guarded, _expect_close, _expect_equal, _gelu64, _ints, _norm_w, _pick_block_n, _poisoned,
                           _ref_norm_rope, _tables, _ulp_bf16, _ulp_f32)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
K_RING = 64 * (STAGES[256] + 1)                 # one k-block more than the 256-wide ring holds


def _rows(ops, n_tiles):
    """rows giving more than 2 tiles per SM at n_tiles tiles per 128 rows, with a ragged last m-tile"""
    return 128 * (-(-2 * ops.num_sms() // n_tiles) + 3) + 1


def test_gemm_swiglu_runahead(cuda_dev):
    from dalm_b200 import ops
    dev = cuda_dev
    N = 512
    M = _rows(ops, N // 256)
    g = torch.Generator().manual_seed(2100)
    a = _poisoned(_ints((M, K_RING), g).to(dev, bf16))
    w = _poisoned(_ints((N, K_RING), g).to(dev, bf16))
    gu, act = Guarded(M, N, bf16, dev), Guarded(M, N // 2, bf16, dev)
    ops.gemm_swiglu(a, w, gu=gu.view, act=act.view)
    what = f"gemm_swiglu M {M} N {N} K {K_RING}"
    acc = a.double() @ w.double().t()
    _expect_equal(gu.view, acc.to(bf16), what + " gu", 128, 256)
    blk = acc.view(M, N // 256, 2, 128)
    gate, up = blk[:, :, 0].reshape(M, N // 2), blk[:, :, 1].reshape(M, N // 2)
    ref = gate * torch.sigmoid(gate) * up
    _expect_close(act.view, ref, _ulp_bf16(ref) + 2.0 ** -20 * ref.abs() + 2.0 ** -100, what + " act", 128, 128)
    gu.check(what + " gu"); act.check(what + " act")


@pytest.mark.parametrize("with_bias", [False, True])
def test_gemm_rope_runahead(cuda_dev, with_bias):
    from dalm_b200 import ops
    dev = cuda_dev
    Lr = 37
    cos_t, sin_t = _tables(dev, Lr)
    N, rope_cols = 768, 512                                       # two rotated tiles and one plain tile per 128 rows
    M = _rows(ops, N // 256)
    g = torch.Generator().manual_seed(2200 + with_bias)
    a = _poisoned(_ints((M, K_RING), g).to(dev, bf16))
    w = _poisoned(_ints((N, K_RING), g).to(dev, bf16))
    bias = _poisoned(_ints((N,), g, hi=64).to(dev)) if with_bias else None
    out = Guarded(M, N, bf16, dev)
    ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=out.view, bias=bias)
    what = f"gemm_rope M {M} N {N} K {K_RING} bias {with_bias}"
    y = a.double() @ w.double().t() + (0 if bias is None else bias.double()[None])
    pos = torch.arange(M, device=dev) % Lr
    c, s = cos_t.double()[pos][:, None], sin_t.double()[pos][:, None]
    h = y[:, :rope_cols].reshape(M, rope_cols // 128, 2, 64)
    x1, x2 = h[:, :, 0], h[:, :, 1]
    rot = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).view(M, rope_cols)
    terms = torch.stack([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], 2).view(M, rope_cols)
    _expect_close(out.view[:, :rope_cols], rot, _ulp_bf16(rot) + 2.0 ** -22 * terms, what + " rotated", 128, 256)
    _expect_equal(out.view[:, rope_cols:], y[:, rope_cols:].to(bf16), what + " plain", 128, 256)
    out.check(what)


def test_gemm_norm_rope_runahead(cuda_dev):
    from dalm_b200 import ops
    dev = cuda_dev
    Lr = 37
    cos_t, sin_t = _tables(dev, Lr)
    N, rope_cols = 768, 512
    M = _rows(ops, N // 256)
    g = torch.Generator().manual_seed(2300)
    a = _poisoned(_ints((M, K_RING), g).to(dev, bf16))
    w = _poisoned(_ints((N, K_RING), g).to(dev, bf16))
    bias = _poisoned(_ints((N,), g, hi=64).to(dev))
    wq, wk = _norm_w(g, dev), _norm_w(g, dev)
    nheads = rope_cols // 128
    nq = (nheads * 3) // 4
    out, pre, rstd = Guarded(M, N, bf16, dev), Guarded(M, rope_cols, bf16, dev), Guarded(M, nheads, f32, dev)
    ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=out.view, bias=bias, q_norm=wq, k_norm=wk, nq_heads=nq, eps=EPS,
                  pre_out=pre.view, rstd_out=rstd.view)
    what = f"gemm_rope+norm M {M} N {N} K {K_RING}"
    y = a.double() @ w.double().t() + bias.double()[None]
    pos = torch.arange(M, device=dev) % Lr
    rot, r64, terms = _ref_norm_rope(y, nheads, nq, wq, wk, cos_t, sin_t, pos)
    _expect_equal(pre.view, y[:, :rope_cols].to(bf16), what + " pre", 128, 256)
    _expect_close(rstd.view, r64, 4 * _ulp_f32(r64), what + " rstd", 128, 2)
    _expect_close(out.view[:, :rope_cols], rot, _ulp_bf16(rot) + 2.0 ** -20 * terms, what + " rotated", 128, 256)
    _expect_equal(out.view[:, rope_cols:], y[:, rope_cols:].to(bf16), what + " plain", 128, 256)
    out.check(what); pre.check(what + " pre"); rstd.check(what + " rstd")


@pytest.mark.parametrize("N", [136, 264, 520])
def test_gemm_gelu_runahead(cuda_dev, N):
    from dalm_b200 import ops
    dev = cuda_dev
    sms = ops.num_sms()
    M = _rows(ops, -(-N // 256))
    tn = _pick_block_n(M, N, sms)
    K = 64 * (STAGES[tn] + 1)
    g = torch.Generator().manual_seed(2400 + N)
    a = _poisoned(_ints((M, K), g).to(dev, bf16))
    w = _poisoned(_ints((N, K), g).to(dev, bf16))
    bv = _ints((N,), g, 4096).to(dev)
    pre, act = Guarded(M, N, bf16, dev), Guarded(M, N, bf16, dev)
    ops.gemm_gelu(a, w, bias=_poisoned(bv), pre=pre.view, act=act.view)
    what = f"gemm_gelu M {M} N {N} K {K} block_n {tn}"
    assert -(-M // 128) * -(-N // tn) > sms, what + ": fewer tiles than SMs"
    x = a.double() @ w.double().t() + bv.double()
    _expect_equal(pre.view, x.to(bf16), what + " pre", 128, tn)
    p = x.to(bf16).double()
    ref = _gelu64(p)
    _expect_close(act.view, ref, _ulp_bf16(ref) + 2.0 ** -21 * (ref.abs() + p.abs()), what + " act", 128, tn)
    pre.check(what + " pre"); act.check(what + " act")
