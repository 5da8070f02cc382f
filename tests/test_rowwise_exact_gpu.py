"""Element-wise checks of the row-wise, reduction, cast / pack and optimizer kernels at the widths, strides and alignments
that pick their code paths.

Every input is a view into a NaN-padded buffer and every output an interior view with sentinel guard bands
(exact_helpers). Where the result does not depend on the order of operations (column sums, scatter-adds, casts, packs,
masked_add at p = 0) the inputs are integers or the op is one rounding, and the check is bit equality. Everywhere else the
output is compared element by element with fp64, within a bound derived from the kernel's arithmetic and written next to
the check. U = 2^-24 is the fp32 unit roundoff: one correctly rounded fp32 operation is within U |result|.

Which LayerNorm kernel runs: the warp-per-row kernels when ln_warp_ok holds (H in {256, 512, 1024, 2048}, every bf16 row
stride a multiple of 8 and every pointer 16-byte aligned), else the CTA-per-row kernel, whose dropout path needs H % 8 == 0
and 16-byte aligned fp32 operands, whose vectorised path needs H % 4 == 0, bf16 strides % 4 == 0 and 8-byte aligned bf16
rows, and whose scalar path takes the rest.
"""
import itertools
import math

import numpy as np
import pytest
import torch

from exact_helpers import (PAD_R, Guarded, _ce_dlse, _dense_poisoned, _expect_close, _expect_equal, _gelu64, _gelu_grad64,
                           _gelu_grad_tol, _gelu_tol, _poisoned, _silu_tol, _ulp_bf16)

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
EPS = 1e-5


@pytest.fixture(scope="module")
def ops(cuda_dev):
    from dalm_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def Err(cuda_dev):
    from dalm_b200._lib import DalmB200Error
    return DalmB200Error


def _v(x):
    """1-D values through the 2-D comparisons"""
    return x.reshape(1, -1)


def _depth(H):
    """longest chain of fp32 additions a term of an H-wide row sum goes through: at most H / 32 serial adds per lane (warp
    kernels: 8 per 256-wide chunk; the CTA kernels do H / 1024) plus <= 24 for the pairwise float4 adds and the warp / block
    trees. A sum of such terms is within depth * U * sum |terms| of exact."""
    return H / 32 + 24


def _rows_with_offset(M, H, g, dev):
    """N(0, 1) rows; every odd row sits on a common offset of 1000, where a one-pass variance (E z^2 - (E z)^2) loses
    all of its digits"""
    z = torch.randn(M, H, generator=g, device=dev) * 1.5
    z[1::2] += 1000.0
    return z


def _drop_scale(ops, M, H, drop, dev):
    return ops.dropout_scale(M * H, drop, dev).view(M, H).double()


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm forward
# ----------------------------------------------------------------------------------------------------------------
# (H, M, dropout, want_f32, y16 shift, y16 extra row stride). Guarded row strides are cols + 512 (+ extra).
LN_FWD = [
    (256, 1, False, True, 0, 0), (512, 7, True, True, 0, 0),           # warp kernel; M tails at its 8-row CTA
    (1024, 9, False, False, 0, 0), (2048, 17, True, False, 0, 0),
    (768, 5, True, True, 0, 0),                                         # CTA dropout path, 16-byte y16 stores
    (768, 5, True, False, 0, 4),                                        # ... scalar y16 stores (ld16 % 8 == 4)
    (1024, 9, True, True, 4, 0),                                        # ... scalar y16 stores (y16 8- not 16-byte aligned)
    (384, 3, False, True, 0, 0), (4544, 3, False, True, 0, 0),          # CTA vectorised path
    (1024, 9, False, True, 0, 4), (2048, 17, False, True, 4, 0),        # warp widths sent to it by ld16 % 8 / alignment
    (1001, 3, False, True, 0, 0), (1001, 3, True, True, 0, 0),          # CTA scalar path: H % 4 != 0
    (388, 3, True, True, 0, 0),                                         # ... dropout with H % 8 != 0
    (768, 3, False, True, 0, 2), (1024, 9, False, False, 1, 0),         # ... ld16 % 4 != 0, y16 at an odd column
    (16384, 2, False, True, 0, 0),                                      # largest accepted width: 64 KB of shared memory
]


@pytest.mark.parametrize("H,M,drop,want_f32,shift,ld_extra", LN_FWD)
def test_layernorm_fwd(ops, cuda_dev, H, M, drop, want_f32, shift, ld_extra):
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(H * 31 + M)
    z = _rows_with_offset(M, H, g, dev)
    gam = torch.randn(H, generator=g, device=dev) * 0.5 + 1.0
    bet = torch.randn(H, generator=g, device=dev) * 0.5
    y16 = Guarded(M, H, bf16, dev, shift=shift, ld_extra=ld_extra)
    d = ops.Drop(0.1, seed=11 + H, stream=3) if drop else None
    y32, _, mean, rstd = ops.layernorm_fwd(_dense_poisoned(z), _poisoned(gam), _poisoned(bet), EPS, y16=y16.view,
                                           want_f32=want_f32, drop=d)
    what = f"layernorm_fwd H {H} M {M} drop {drop} y16 shift {shift} ld {y16.view.stride(0)}"
    y16.check(what)
    z64 = z.double()
    mu = z64.mean(1, keepdim=True)
    r64 = 1.0 / torch.sqrt(((z64 - mu) ** 2).mean(1, keepdim=True) + EPS)
    zh = (z64 - mu) * r64
    ref = zh * gam.double() + bet.double()
    dep = _depth(H)
    dmean = dep * U * z64.abs().mean(1, keepdim=True) + U * mu.abs()   # the row sum, then / H
    # sum of squares (depth + 2 roundings per term), squares about the kernel's mean (+ dmean^2), rsqrtf <= 2 ulp
    rel_rstd = (dep + 8) * U + 0.5 * dmean ** 2 * r64 ** 2
    _expect_close(_v(mean), _v(mu), _v(dmean), what + " mean")
    _expect_close(_v(rstd), _v(r64), _v(rel_rstd * r64), what + " rstd")
    # y = (z - mean) * rstd * gamma + beta: the mean's error scaled by rstd |gamma|, rstd's relative error, 3 roundings
    tol = dmean * r64 * gam.double().abs() + (zh * gam.double()).abs() * (rel_rstd + 3 * U) + U * ref.abs()
    if drop:
        sc = _drop_scale(ops, M, H, d, dev)
        ref, tol = ref * sc, tol * sc + U * (ref * sc).abs()           # one more rounding for the 1/(1-p) scale
    if want_f32:
        _expect_close(y32, ref, tol, what + " y32")
    else:
        assert y32 is None
    _expect_close(y16.view, ref, _ulp_bf16(ref) + tol, what + " y16")   # RNE: 1/2 ulp, 1 ulp across a binade edge


def test_layernorm_fwd_width_limit(ops, cuda_dev, Err):
    z = torch.zeros(2, 16385, device=cuda_dev)
    w = torch.ones(16385, device=cuda_dev)
    with pytest.raises(Err):
        ops.layernorm_fwd(z, w, w, EPS)


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm backward
# ----------------------------------------------------------------------------------------------------------------
def _ln_bwd_ref(z, gam, mean32, rstd32, dy, H):
    """fp64 LayerNorm input gradient from the saved (fp32) mean / rstd, and its element-wise bound"""
    z64, r = z.double(), rstd32.double()[:, None]
    zh = (z64 - mean32.double()[:, None]) * r
    gg = dy * gam.double()
    s1 = gg.mean(1, keepdim=True)
    s2 = (gg * zh).mean(1, keepdim=True)
    dz = r * (gg - s1 - zh * s2)
    dep = _depth(H)
    ds1 = (dep + 2) * U * gg.abs().mean(1, keepdim=True)                # g = (dy_a + dy_b) * gamma: 2 roundings, then the row sum
    ds2 = (dep + 4) * U * (gg * zh).abs().mean(1, keepdim=True)         # zhat: 2 roundings, g * zhat: 1
    tol = r * (ds1 + zh.abs() * ds2 + 6 * U * (gg.abs() + s1.abs() + (zh * s2).abs())) + U * dz.abs()
    return dz, tol


def _ln_stats(z):
    z64 = z.double()
    mu = z64.mean(1)
    rs = 1.0 / torch.sqrt(((z64 - mu[:, None]) ** 2).mean(1) + EPS)
    return mu.float(), rs.float()


# (H, M, inputs, want_f32, want_bf16, dropout, dz16 (shift, extra stride), dy_bf16 (col0, pad columns))
LN_BWD = [
    (256, 1, "ab", True, True, False, (0, 0), (0, 64)),                 # warp kernel
    (512, 7, "a", True, False, False, (0, 0), (0, 64)),
    (1024, 9, "b", False, True, True, (0, 0), (0, 64)),
    (2048, 17, "ab", True, True, True, (0, 0), (0, 64)),
    (768, 5, "ab", True, True, True, (0, 0), (0, 64)),                  # CTA dropout path, 16-byte dz16 stores
    (768, 5, "b", True, True, True, (0, 4), (0, 64)),                   # ... scalar dz16 stores (ld16 % 8 == 4)
    (1024, 9, "ab", True, True, True, (4, 0), (0, 64)),                 # ... scalar dz16 stores (8- not 16-byte aligned)
    (384, 3, "ab", True, True, False, (0, 0), (0, 64)),                 # CTA vectorised path
    (4544, 3, "b", True, True, False, (0, 0), (0, 64)),
    (1024, 9, "b", True, True, False, (0, 0), (0, 68)),                 # warp width, ldb % 8 == 4: CTA, vector loads
    (1024, 9, "ab", True, True, False, (0, 0), (0, 66)),                # CTA scalar loads: ldb % 4 != 0
    (768, 3, "b", True, True, False, (0, 0), (1, 64)),                  # ... dy_bf16 at an odd column
    (1001, 3, "ab", True, True, False, (0, 0), (0, 64)),                # CTA scalar path: H % 4 != 0
    (1001, 3, "b", False, True, True, (0, 0), (0, 64)),
    (768, 3, "ab", False, True, False, (0, 2), (0, 64)),                # ... ld16 % 4 != 0
    (1024, 9, "a", True, True, False, (1, 0), (0, 64)),                 # ... dz16 at an odd column
    (6144, 2, "ab", True, True, False, (0, 0), (0, 64)),                # largest accepted width (48 KB of shared memory)
]


@pytest.mark.parametrize("H,M,inputs,want_f32,want_bf16,drop,dz16_at,dyb_at", LN_BWD)
def test_layernorm_bwd(ops, cuda_dev, H, M, inputs, want_f32, want_bf16, drop, dz16_at, dyb_at):
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(H * 17 + M)
    z = _rows_with_offset(M, H, g, dev)
    gam = torch.randn(H, generator=g, device=dev) * 0.5 + 1.0
    mean, rstd = _ln_stats(z)
    dy_a = torch.randn(M, H, generator=g, device=dev) if "a" in inputs else None
    dy_b = (torch.randn(M, H, generator=g, device=dev) * 2).to(bf16) if "b" in inputs else None
    dz16 = Guarded(M, H, bf16, dev, shift=dz16_at[0], ld_extra=dz16_at[1]) if want_bf16 else None
    d = ops.Drop(0.1, seed=5 + H, stream=9) if drop else None
    dz32, _ = ops.layernorm_bwd(_dense_poisoned(z), _poisoned(gam), _poisoned(mean), _poisoned(rstd),
                                dy_f32=None if dy_a is None else _dense_poisoned(dy_a),
                                dy_bf16=None if dy_b is None else _poisoned(dy_b, col0=dyb_at[0], pad_c=dyb_at[1]),
                                want_f32=want_f32, dz16=None if dz16 is None else dz16.view, want_bf16=want_bf16, drop16=d)
    what = f"layernorm_bwd H {H} M {M} in {inputs} drop {drop} dz16 {dz16_at} dy_bf16 {dyb_at}"
    dy = (dy_a.double() if dy_a is not None else 0) + (dy_b.double() if dy_b is not None else 0)
    ref, tol = _ln_bwd_ref(z, gam, mean, rstd, dy, H)
    if want_f32:
        _expect_close(dz32, ref, tol, what + " dz32")
    else:
        assert dz32 is None
    if want_bf16:
        dz16.check(what)
        if drop:                                                        # only the bf16 (dense-branch) output is masked
            sc = _drop_scale(ops, M, H, d, dev)
            ref, tol = ref * sc, tol * sc + U * (ref * sc).abs()
        _expect_close(dz16.view, ref, _ulp_bf16(ref) + tol, what + " dz16")


# (H, M, dz16 (shift, extra stride), dres aliases dz32)
LN_BWD_RES = [(256, 9, (0, 0), True), (1024, 17, (0, 0), False), (768, 5, (0, 0), True), (1001, 3, (0, 0), True),
              (1024, 9, (1, 0), True), (768, 3, (0, 2), False)]


@pytest.mark.parametrize("H,M,dz16_at,alias", LN_BWD_RES)
def test_layernorm_bwd_res(ops, cuda_dev, H, M, dz16_at, alias):
    """pre-LN form: dz = LayerNorm-backward(dy_bf16) + dres, with dz32 either a fresh buffer or dres itself"""
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(H * 7 + M)
    z = _rows_with_offset(M, H, g, dev)
    gam = torch.randn(H, generator=g, device=dev) * 0.5 + 1.0
    mean, rstd = _ln_stats(z)
    dy_b = (torch.randn(M, H, generator=g, device=dev) * 2).to(bf16)
    dres = torch.randn(M, H, generator=g, device=dev)
    dres_in = _dense_poisoned(dres)
    dz16 = Guarded(M, H, bf16, dev, shift=dz16_at[0], ld_extra=dz16_at[1])
    dz32, _ = ops.layernorm_bwd_res(_dense_poisoned(z), _poisoned(gam), _poisoned(mean), _poisoned(rstd), _poisoned(dy_b),
                                    dres_in, dz32=dres_in if alias else None, dz16=dz16.view)
    what = f"layernorm_bwd_res H {H} M {M} dz16 {dz16_at} alias {alias}"
    dz16.check(what)
    if alias:
        assert dz32.data_ptr() == dres_in.data_ptr()
    ref, tol = _ln_bwd_ref(z, gam, mean, rstd, dy_b.double(), H)
    ref = ref + dres.double()
    tol = tol + U * ref.abs()                                           # the residual add: one rounding
    _expect_close(dz32, ref, tol, what + " dz32")
    _expect_close(dz16.view, ref, _ulp_bf16(ref) + tol, what + " dz16")


# ----------------------------------------------------------------------------------------------------------------
# RMSNorm
# ----------------------------------------------------------------------------------------------------------------
RMS_H = (4, 260, 896, 1024, 1536, 2048, 3584, 4096, 5120, 12288)


def _rms_rows(M, H, g, dev):
    """row 0 all zero, row 1 so small that eps dominates mean(x^2), the rest N(0, 1.7^2)"""
    x = torch.randn(M, H, generator=g, device=dev) * 1.7
    x[0] = 0.0
    x[1] *= 1e-4
    return x


@pytest.mark.parametrize("H", RMS_H)
def test_rmsnorm_fwd(ops, cuda_dev, H):
    dev, M = cuda_dev, 5
    g = torch.Generator(device=dev).manual_seed(H)
    x = _rms_rows(M, H, g, dev)
    w = torch.rand(H, generator=g, device=dev) + 0.5
    # h as the left columns of a wider (LoRA-augmented) activation buffer
    aug = Guarded(M, H + 16, bf16, dev)
    tail = aug.view[:, H:].clone()
    _, rstd = ops.rmsnorm_fwd(_dense_poisoned(x), _poisoned(w), EPS, h=aug.view[:, :H])
    what = f"rmsnorm_fwd H {H}"
    aug.check(what)
    assert torch.equal(aug.view[:, H:].view(torch.int16), tail.view(torch.int16)), what + ": columns right of h written"
    x64 = x.double()
    r64 = 1.0 / torch.sqrt((x64 ** 2).mean(1, keepdim=True) + EPS)
    ref = x64 * r64 * w.double()
    rel_rstd = (_depth(H) + 8) * U                                      # sum of squares, / H, + eps, rsqrtf <= 2 ulp
    _expect_close(_v(rstd), _v(r64), _v(rel_rstd * r64), what + " rstd")
    _expect_close(aug.view[:, :H], ref, _ulp_bf16(ref) + ref.abs() * (rel_rstd + 2 * U), what + " h")   # 2 products, RNE


@pytest.mark.parametrize("H", RMS_H)
@pytest.mark.parametrize("dres_mode", ["none", "given", "alias"])
def test_rmsnorm_bwd(ops, cuda_dev, H, dres_mode):
    dev, M = cuda_dev, 5
    g = torch.Generator(device=dev).manual_seed(H + 1)
    x = _rms_rows(M, H, g, dev)
    w = torch.rand(H, generator=g, device=dev) + 0.5
    x64 = x.double()
    rstd = (1.0 / torch.sqrt((x64 ** 2).mean(1) + EPS)).float()
    dh = (torch.randn(M, H, generator=g, device=dev) * 2).to(bf16)
    dres = torch.randn(M, H, generator=g, device=dev)
    dres_in = _dense_poisoned(dres) if dres_mode != "none" else None
    d16 = Guarded(M, H, bf16, dev, ld_extra=16)
    out32, _ = ops.rmsnorm_bwd(_dense_poisoned(x), _poisoned(w), _poisoned(rstd), _poisoned(dh), dres_in=dres_in,
                               dres_out=dres_in if dres_mode == "alias" else None, dres16=d16.view)
    what = f"rmsnorm_bwd H {H} dres {dres_mode}"
    d16.check(what)
    r = rstd.double()[:, None]
    xh = x64 * r
    gd = dh.double() * w.double()
    s = (gd * xh).mean(1, keepdim=True)
    ref = r * (gd - xh * s)
    ds = (_depth(H) + 3) * U * (gd * xh).abs().mean(1, keepdim=True)    # gd, xhat, their product: 3 roundings, then the sum
    tol = r * (xh.abs() * ds + 4 * U * (gd.abs() + (xh * s).abs())) + U * ref.abs()
    if dres_mode != "none":
        ref = ref + dres.double()
        tol = tol + U * ref.abs()
    _expect_close(out32, ref, tol, what + " dres_out")
    _expect_close(d16.view, ref, _ulp_bf16(ref) + tol, what + " dres16")


def test_norm_width_limits(ops, cuda_dev, Err):
    dev = cuda_dev
    for H in (12292,):
        x = torch.zeros(2, H, device=dev)
        w = torch.ones(H, device=dev)
        with pytest.raises(Err):
            ops.rmsnorm_fwd(x, w, EPS)
        with pytest.raises(Err):
            ops.rmsnorm_bwd(x, w, torch.ones(2, device=dev), torch.zeros(2, H, dtype=bf16, device=dev))
    z = torch.zeros(2, 6145, device=dev)
    with pytest.raises(Err):
        ops.layernorm_bwd(z, torch.ones(6145, device=dev), torch.zeros(2, device=dev), torch.ones(2, device=dev), dy_f32=z)


# ----------------------------------------------------------------------------------------------------------------
# wrappers refuse fp32 operands the kernels would read as dense rows when they are not
# ----------------------------------------------------------------------------------------------------------------
def test_row_strided_fp32_operands_are_refused(ops, cuda_dev, Err):
    """Each call passes one row-strided view (row stride H + 64; fp32 operands and bf16 embedding tables) where the kernel
    indexes dense rows ptr + r * H, or a transposed source where it needs contiguous rows. The buffers
    behind the views are larger than M * H, so a kernel that ignored the stride would still stay inside them."""
    dev, M, H = cuda_dev, 9, 256
    S = lambda: _poisoned(torch.randn(M, H, device=dev))                # noqa: E731  row-strided fp32 [M, H]
    D = lambda: torch.randn(M, H, device=dev)                           # noqa: E731  dense fp32 [M, H]
    w, mean, rstd = torch.ones(H, device=dev), torch.zeros(M, device=dev), torch.ones(M, device=dev)
    b16 = torch.randn(M, H, device=dev).to(bf16)
    ids = torch.zeros(M, dtype=torch.int64, device=dev)
    calls = {
        "layernorm_fwd z": lambda: ops.layernorm_fwd(S(), w, w, EPS),
        "layernorm_bwd z": lambda: ops.layernorm_bwd(S(), w, mean, rstd, dy_f32=D()),
        "layernorm_bwd dy_f32": lambda: ops.layernorm_bwd(D(), w, mean, rstd, dy_f32=S()),
        "layernorm_bwd_res z": lambda: ops.layernorm_bwd_res(S(), w, mean, rstd, b16, D()),
        "layernorm_bwd_res dres": lambda: ops.layernorm_bwd_res(D(), w, mean, rstd, b16, S()),
        "layernorm_bwd_res dz32": lambda: ops.layernorm_bwd_res(D(), w, mean, rstd, b16, D(), dz32=S()),
        "rmsnorm_fwd x": lambda: ops.rmsnorm_fwd(S(), w, EPS),
        "rmsnorm_bwd x": lambda: ops.rmsnorm_bwd(S(), w, rstd, b16),
        "rmsnorm_bwd dres_in": lambda: ops.rmsnorm_bwd(D(), w, rstd, b16, dres_in=S()),
        "rmsnorm_bwd dres_out": lambda: ops.rmsnorm_bwd(D(), w, rstd, b16, dres_out=S()),
        "masked_add a": lambda: ops.masked_add(S(), b16),
        "masked_add out": lambda: ops.masked_add(D(), b16, out=S()),
        "embed_scatter_add d": lambda: ops.embed_scatter_add_(S(), ids, torch.zeros(4, H, device=dev)),
        "embed_scatter_add dword": lambda: ops.embed_scatter_add_(D(), ids, _poisoned(torch.zeros(4, H, device=dev))),
        "embed_scatter_add dpos": lambda: ops.embed_scatter_add_(D(), ids, torch.zeros(4, H, device=dev),
                                                                 _poisoned(torch.zeros(4, H, device=dev)), 4),
        "col_reduce dy_f32": lambda: ops.col_reduce_(dy_f32=S(), out_sum=torch.zeros(H, device=dev)),
        "col_reduce z": lambda: ops.col_reduce_(dy_f32=D(), z=S(), rstd=rstd, out_prod=torch.zeros(H, device=dev)),
        "bert_embed out": lambda: ops.bert_embed(ids.view(1, M), b16, b16, b16[0], out=S()),
        "bert_embed word": lambda: ops.bert_embed(ids.view(1, M), _poisoned(b16), b16, b16[0]),
        "embed_gather table": lambda: ops.embed_gather(ids, _poisoned(b16)),
        "cast_f32_bf16 transposed src": lambda: ops.cast_f32_bf16(torch.randn(H, M, device=dev).t()),
    }
    for name, call in calls.items():
        with pytest.raises(Err):
            call()
            torch.cuda.synchronize()
            pytest.fail(f"{name}: a row-strided operand was accepted")


# ----------------------------------------------------------------------------------------------------------------
# embeddings: gathers and the scatter-add that must be their adjoint
# ----------------------------------------------------------------------------------------------------------------
def _ids_with_edges(M, V, g, dev):
    ids = torch.randint(0, V, (M,), generator=g, device=dev)
    edge = torch.tensor([0, V - 1, -1, V, V + 7, -(2 ** 40), 2 ** 40, 3, 3, 3, 3, V - 1], device=dev)
    ids[: edge.numel()] = edge
    return ids


def test_embedding_gathers(ops, cuda_dev):
    """ids at 0, V - 1 and out of range (read as row 0); M = B * L rows whose positions wrap L; integer tables make the
    fp32 sum exact, so the check is bit equality"""
    dev, B, L, V, H = cuda_dev, 3, 7, 50, 264
    g = torch.Generator(device=dev).manual_seed(21)
    ids = _ids_with_edges(B * L, V, g, dev).view(B, L)
    word = torch.randint(-100, 101, (V, H), generator=g, device=dev).to(bf16)
    pos = torch.randint(-100, 101, (L, H), generator=g, device=dev).to(bf16)
    typ = torch.randint(-100, 101, (H,), generator=g, device=dev).to(bf16)
    row = torch.where((ids >= 0) & (ids < V), ids, torch.zeros_like(ids)).view(-1)
    z = ops.bert_embed(ids, _dense_poisoned(word), _dense_poisoned(pos), _poisoned(typ))
    want = word.double()[row] + pos.double()[torch.arange(B * L, device=dev) % L] + typ.double()
    _expect_equal(z, want, "bert_embed")
    x = ops.embed_gather(ids, _dense_poisoned(word))
    _expect_equal(x, word.double()[row], "embed_gather")


def test_embed_scatter_is_the_gathers_adjoint(ops, cuda_dev):
    """integer gradients (exact fp32 sums whatever the atomic order), many repeats of one id, out-of-range ids, positions
    wrapping L, accumulation into non-zero tables. The row each token scatters into is the row embed_gather read for it
    (found by gathering from a table whose row v holds v)."""
    dev, L, V, H = cuda_dev, 6, 200, 132
    M = 4 * L
    g = torch.Generator(device=dev).manual_seed(22)
    ids = _ids_with_edges(M, V, g, dev)
    ident = torch.arange(V, device=dev, dtype=f32)[:, None].expand(V, 8).to(bf16).contiguous()
    read = ops.embed_gather(ids, ident)[:, 0].long()                    # the row the gather read for each token
    d = torch.randint(-8, 9, (M, H), generator=g, device=dev).float()
    w0 = torch.randint(-4, 5, (V, H), generator=g, device=dev).float()
    p0 = torch.randint(-4, 5, (L, H), generator=g, device=dev).float()
    dw_buf, dp_buf = w0.clone(), p0.clone()                             # the kernel needs dense tables
    ops.embed_scatter_add_(_dense_poisoned(d), ids, dw_buf, dp_buf, L)
    want_w = w0.double().index_add(0, read, d.double())
    want_p = p0.double().index_add(0, torch.arange(M, device=dev) % L, d.double())
    _expect_equal(dw_buf, want_w, "embed_scatter_add dword")
    _expect_equal(dp_buf, want_p, "embed_scatter_add dpos")
    dw2 = torch.zeros(V + PAD_R, H, device=dev)                         # without dpos; rows past V must stay untouched
    ops.embed_scatter_add_(_dense_poisoned(d), ids, dw2[:V])
    _expect_equal(dw2, torch.cat([torch.zeros(V, H, device=dev, dtype=f64).index_add(0, read, d.double()),
                                  torch.zeros(PAD_R, H, device=dev, dtype=f64)]), "embed_scatter_add dword only")


# ----------------------------------------------------------------------------------------------------------------
# col_reduce: column sums of the gradient and of gradient * zhat, accumulated into the outputs
# ----------------------------------------------------------------------------------------------------------------
CR_SHAPES = [(1, 4), (7, 124), (64, 128), (65, 132), (4608, 4544), (26700, 132), (26700, 4), (4608, 124), (65, 4544),
             (1, 132), (7, 4544), (64, 4)]
CR_VARIANTS = [  # inputs, outputs, mean given
    ("a", "sp", True), ("b", "s", False), ("ab", "p", True), ("ab", "sp", False), ("a", "p", False), ("b", "sp", True)]


@pytest.mark.parametrize("si", range(len(CR_SHAPES)))
def test_col_reduce(ops, cuda_dev, si):
    """integer dy, z and mean with power-of-two rstd: every partial sum is an integer multiple of 1/4 below 2^21, so the
    result is exact whatever the split-row grid and the atomic order, and the check is bit equality"""
    M, H = CR_SHAPES[si]
    dev = cuda_dev
    for vi, (inputs, outs, with_mean) in enumerate(CR_VARIANTS):
        if (si + vi) % 2:                                               # every variant meets half of the shapes
            continue
        g = torch.Generator(device=dev).manual_seed(si * 10 + vi)
        dy_a = torch.randint(-2, 3, (M, H), generator=g, device=dev).float() if "a" in inputs else None
        dy_b = torch.randint(-2, 3, (M, H), generator=g, device=dev).to(bf16) if "b" in inputs else None
        z = torch.randint(-4, 5, (M, H), generator=g, device=dev).float()
        mean = torch.randint(-2, 3, (M,), generator=g, device=dev).float()
        rstd = 2.0 ** torch.randint(-2, 2, (M,), generator=g, device=dev).float()
        s0 = torch.randint(-50, 51, (H,), generator=g, device=dev).float()   # accumulate into non-zero outputs
        p0 = torch.randint(-50, 51, (H,), generator=g, device=dev).float()
        osum = Guarded(1, H, f32, dev, init=s0[None]) if "s" in outs else None
        oprod = Guarded(1, H, f32, dev, init=p0[None]) if "p" in outs else None
        ops.col_reduce_(dy_f32=None if dy_a is None else _dense_poisoned(dy_a),
                        dy_bf16=None if dy_b is None else _poisoned(dy_b),
                        z=_dense_poisoned(z) if oprod else None, mean=_poisoned(mean) if with_mean and oprod else None,
                        rstd=_poisoned(rstd) if oprod else None,
                        out_sum=None if osum is None else osum.view[0], out_prod=None if oprod is None else oprod.view[0])
        what = f"col_reduce M {M} H {H} in {inputs} out {outs} mean {with_mean}"
        dy = (dy_a.double() if dy_a is not None else 0) + (dy_b.double() if dy_b is not None else 0)
        if osum:
            osum.check(what)
            _expect_equal(osum.view, _v(s0.double() + dy.sum(0)), what + " sum")
        if oprod:
            oprod.check(what)
            zh = (z.double() - (mean.double()[:, None] if with_mean else 0)) * rstd.double()[:, None]
            _expect_equal(oprod.view, _v(p0.double() + (dy * zh).sum(0)), what + " prod")


# ----------------------------------------------------------------------------------------------------------------
# masked_add
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["ab", "a", "b", "ab_inplace", "a_inplace"])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_masked_add(ops, cuda_dev, mode, p):
    """out = (a + b) * mask / (1 - p): integer a, b make the sum exact, so p = 0 is bit-exact and p > 0 is one fp32
    rounding of the exact (a + b) * scale (within 1/2 fp32 ulp of fp64)"""
    dev, M, H = cuda_dev, 37, 264
    g = torch.Generator(device=dev).manual_seed(int(p * 10) + len(mode))
    a = torch.randint(-300, 301, (M, H), generator=g, device=dev).float() if "a" in mode else None
    b = torch.randint(-200, 201, (M, H), generator=g, device=dev).to(bf16) if "b" in mode.split("_")[0] else None
    d = ops.Drop(p, seed=3, stream=4)
    a_in = None if a is None else _dense_poisoned(a)
    out = ops.masked_add(a_in, None if b is None else _poisoned(b), drop=d, out=a_in if "inplace" in mode else None)
    if "inplace" in mode:
        assert out.data_ptr() == a_in.data_ptr()
    s = (a.double() if a is not None else 0) + (b.double() if b is not None else 0)
    what = f"masked_add {mode} p {p}"
    if p == 0:
        _expect_equal(out, s, what)
    else:
        ref = s * _drop_scale(ops, M, H, d, dev)
        _expect_close(out, ref, 2.0 ** -24 * ref.abs(), what)


# ----------------------------------------------------------------------------------------------------------------
# Adam
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,shadow", [(1, False), (255, False), (257, False), (10007, False), (4, True), (1020, True),
                                      (1028, True), (10004, True)])
def test_adam(ops, cuda_dev, n, shadow):
    """20 steps against torch.optim.Adam in fp64 (same fp32 hyper-parameters), grad_scale 0.5. The bound is carried along
    the steps: m and v take 3-4 roundings per step and inherit beta times the previous error; the step takes m's and
    v's errors, the fp32 bias corrections (powf within 8 ulp; 1 - beta^t loses beta^t / (1 - beta^t) of relative accuracy)
    and 4 roundings; p one more. The bf16 shadow must be bit-equal to p.to(bf16)."""
    dev = cuda_dev
    lr, b1, b2, eps, gs = (float(np.float32(v)) for v in (1e-3, 0.9, 0.999, 1e-8, 0.5))
    g = torch.Generator(device=dev).manual_seed(n)
    p0 = torch.randn(n, generator=g, device=dev)
    P, Mo, Vo = (Guarded(1, n, f32, dev, init=t[None]) for t in (p0, torch.zeros(n, device=dev), torch.zeros(n, device=dev)))
    S = Guarded(1, n, bf16, dev) if shadow else None
    ref = p0.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps)
    m64 = torch.zeros(n, dtype=f64, device=dev); v64 = torch.zeros_like(m64)
    tm = torch.zeros_like(m64); tv = torch.zeros_like(m64); tp = torch.zeros_like(m64)
    what = f"adam n {n} shadow {shadow}"
    for k in range(1, 21):
        grad = torch.randn(n, generator=g, device=dev)
        if shadow:
            ops.adam_step_shadow_(P.view[0], _poisoned(grad), Mo.view[0], Vo.view[0], S.view[0], lr, b1, b2, eps, k, gs)
        else:
            ops.adam_step_(P.view[0], _poisoned(grad), Mo.view[0], Vo.view[0], lr, b1, b2, eps, k, gs)
        gi = grad.double() * gs
        ref.grad = gi.clone()
        opt.step()
        m64 = b1 * m64 + (1 - b1) * gi
        v64 = b2 * v64 + (1 - b2) * gi * gi
        bc1, bc2 = 1 - b1 ** k, 1 - b2 ** k
        den = v64.sqrt() / math.sqrt(bc2) + eps
        step = lr / bc1 * m64 / den
        tm = b1 * tm + 3 * U * m64.abs()
        tv = b2 * tv + 4 * U * v64
        rb1 = (8 * U * b1 ** k + U) / bc1
        rb2 = 0.5 * (8 * U * b2 ** k + U) / bc2 + U
        rden = (0.5 * tv / v64.clamp_min(1e-300) + rb2 + 3 * U) * (den - eps) / den
        tp = tp + lr / bc1 * tm / den + step.abs() * (rden + rb1 + 4 * U) + U * ref.detach().abs()
        _expect_close(_v(P.view[0]), _v(ref.detach()), _v(tp), f"{what} step {k} p")
        if shadow:
            _expect_equal(S.view, P.view.to(bf16), f"{what} step {k} shadow")
    _expect_close(_v(Mo.view[0]), _v(m64), _v(tm), what + " m")
    _expect_close(_v(Vo.view[0]), _v(v64), _v(tv), what + " v")
    for gd in (P, Mo, Vo) + ((S,) if shadow else ()):
        gd.check(what)


# ----------------------------------------------------------------------------------------------------------------
# casts and packs: one rounding (RNE), bit-exact against torch
# ----------------------------------------------------------------------------------------------------------------
def _special_f32(rows, cols, g, dev):
    """random values over many binades, exact bf16 halfway points (ties to even both ways), values one fp32 ulp either
    side of a tie, +-inf, NaN, the largest finite fp32 (rounds to inf) and subnormals"""
    x = torch.randn(rows, cols, generator=g, device=dev) * torch.exp2(torch.randint(-20, 20, (rows, cols), generator=g, device=dev).float())
    bits = x.view(torch.int32)
    sel = torch.randint(0, 6, (rows, cols), generator=g, device=dev)
    hi = bits & ~0xFFFF
    bits = torch.where(sel == 1, hi | 0x8000, bits)                       # exact tie
    bits = torch.where(sel == 2, hi | 0x7FFF, bits)                       # just below
    bits = torch.where(sel == 3, hi | 0x8001, bits)                       # just above
    x = bits.view(f32).clone()
    flat = x.view(-1)
    sp = torch.tensor([float("inf"), float("-inf"), float("nan"), 3.4028234663852886e38, -3.4028234663852886e38, 1e-40,
                       -1e-40, 0.0, -0.0], device=dev)
    k = min(sp.numel(), flat.numel())
    flat[:k] = sp[:k]
    return x


def _expect_bits(got, want, what):
    """bf16 bit patterns equal; NaN where and only where want is NaN (NaN payloads may differ)"""
    gn, wn = torch.isnan(got), torch.isnan(want)
    bad = ((got.view(torch.int16) != want.view(torch.int16)) & ~(gn & wn)) | (gn != wn)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} wrong; first at ({r}, {c}): got "
                    f"{got[r, c].item()!r}, want {want[r, c].item()!r}")


@pytest.mark.parametrize("rows,cols", [(3, 8), (37, 1028), (70000, 8)])
def test_cast_f32_bf16(ops, cuda_dev, rows, cols):
    """strided source and destination; 70 000 rows is more than one grid dimension of 65 535 CTAs"""
    dev = cuda_dev
    x = _special_f32(rows, cols, torch.Generator(device=dev).manual_seed(rows), dev)
    dst = Guarded(rows, cols, bf16, dev)
    ops.cast_f32_bf16(_poisoned(x), dst.view)
    what = f"cast_f32_bf16 [{rows}, {cols}]"
    dst.check(what)
    _expect_bits(dst.view, x.to(bf16), what)


def _pack_ref(src_rc, scale):
    """bf16 RNE of the fp32 product (fp64 holds the product of two fp32 values exactly)"""
    return (src_rc.double() * float(np.float32(scale))).float().to(bf16)


@pytest.mark.parametrize("transposed", [False, True])
def test_pack_scaled_bf16(ops, cuda_dev, transposed):
    dev, rows, cols, scale = cuda_dev, 24, 520, 0.3
    x = _special_f32(rows, cols, torch.Generator(device=dev).manual_seed(7), dev)
    src = _poisoned(x.t().contiguous()) if transposed else _poisoned(x)
    si_r, si_c = (1, src.stride(0)) if transposed else (src.stride(0), 1)
    dst = Guarded(rows, cols, bf16, dev)
    ops.pack_scaled_bf16_(src, si_r, si_c, dst.view, rows, cols, scale)
    what = f"pack_scaled_bf16 transposed {transposed}"
    dst.check(what)
    _expect_bits(dst.view, _pack_ref(x, scale), what)


def test_pack_table(ops, cuda_dev):
    """one launch over several entries, two of them larger than the 32 x 256-thread grid-stride of an entry"""
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(8)
    specs = [(8, 520, True, 2.0), (16, 4096, False, 0.3), (24, 40, True, -1.5), (520, 24, False, 0.125)]
    entries, outs = [], []
    for rows, cols, tr, sc in specs:
        x = _special_f32(rows, cols, g, dev)
        src = _poisoned(x.t().contiguous()) if tr else _poisoned(x)
        si_r, si_c = (1, src.stride(0)) if tr else (src.stride(0), 1)
        dst = Guarded(rows, cols, bf16, dev)
        entries.append((src, si_r, si_c, dst.view, rows, cols, sc))
        outs.append((dst, x, sc, src))
    table = ops.build_pack_table(entries, dev)
    ops.pack_table_(table)
    for i, (dst, x, sc, _) in enumerate(outs):
        what = f"pack_table entry {i} {specs[i]}"
        dst.check(what)
        _expect_bits(dst.view, _pack_ref(x, sc), what)


# ----------------------------------------------------------------------------------------------------------------
# RoPE, SwiGLU, GELU: within one bf16 ulp of fp64
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [32, 64, 128])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 33])
def test_rope(ops, cuda_dev, D, M):
    dev, L, nh = cuda_dev, 3, 2
    col0 = 8 * (M % 3)                                                  # 0, 8 or 16 columns into the row
    W = col0 + nh * D + 24
    g = torch.Generator(device=dev).manual_seed(D * 100 + M)
    x = torch.randn(M, W, generator=g, device=dev).to(bf16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=f64, device=dev) / D))
    fr = torch.outer(torch.arange(L, dtype=f64, device=dev), inv)
    cos_t, sin_t = fr.cos().float(), fr.sin().float()
    for backward in (False, True):
        buf = Guarded(M, W, bf16, dev, init=x, ld_extra=8)
        ops.rope_(buf.view, col0, nh, D, _dense_poisoned(cos_t), _dense_poisoned(sin_t), L, backward=backward)
        what = f"rope D {D} M {M} col0 {col0} backward {backward}"
        buf.check(what)
        h = x[:, col0:col0 + nh * D].double().view(M, nh, 2, D // 2)
        pos = torch.arange(M, device=dev) % L
        c, s = cos_t.double()[pos][:, None, :], sin_t.double()[pos][:, None, :] * (-1 if backward else 1)
        x1, x2 = h[:, :, 0], h[:, :, 1]
        ref = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).view(M, nh * D)
        mag = torch.stack([(x1 * c).abs() + (x2 * s).abs()] * 2, 2).view(M, nh * D)
        _expect_close(buf.view[:, col0:col0 + nh * D], ref, _ulp_bf16(ref) + 2 * U * mag, what)   # 2 fp32 roundings, RNE
        _expect_equal(buf.view[:, :col0], x[:, :col0], what + " left of the heads")
        _expect_equal(buf.view[:, col0 + nh * D:], x[:, col0 + nh * D:], what + " right of the heads")


@pytest.mark.parametrize("F,il", [(8, 0), (264, 0), (256, 128), (384, 128)])
def test_swiglu(ops, cuda_dev, F, il):
    dev, M = cuda_dev, 5
    gen = torch.Generator(device=dev).manual_seed(F + il)
    gu = (torch.randn(M, 2 * F, generator=gen, device=dev) * 2).to(bf16)
    if il:
        gcols = (torch.arange(F, device=dev) // il) * 2 * il + torch.arange(F, device=dev) % il
        ucols = gcols + il
    else:
        gcols, ucols = torch.arange(F, device=dev), torch.arange(F, device=dev) + F
    g, u = gu.double()[:, gcols], gu.double()[:, ucols]
    sg = torch.sigmoid(g)
    act = Guarded(M, F, bf16, dev)
    ops.swiglu_fwd(_poisoned(gu), F, act=act.view, interleave=il)
    what = f"swiglu F {F} interleave {il}"
    act.check(what)
    ref = g * sg * u
    _expect_close(act.view, ref, _ulp_bf16(ref) + _silu_tol(g) * ref.abs(), what + " fwd")
    dact = (torch.randn(M, F, generator=gen, device=dev)).to(bf16)
    work = Guarded(M, 2 * F, bf16, dev, init=gu)
    ops.swiglu_bwd_(work.view, _poisoned(dact), F, interleave=il)
    work.check(what)
    d = dact.double()
    dg = d * u * sg * (1 + g * (1 - sg))
    du = d * g * sg
    # dgate: sigmoid's error enters 1 + g (1 - sg) times |g| sg (no cancellation bound is needed: the error is absolute)
    tol_dg = _ulp_bf16(dg) + _silu_tol(g) * (d * u * sg).abs() * (1 + g.abs()) * 4
    _expect_close(work.view[:, gcols], dg, tol_dg, what + " dgate")
    _expect_close(work.view[:, ucols], du, _ulp_bf16(du) + _silu_tol(g) * du.abs(), what + " dup")


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 9])
@pytest.mark.parametrize("F", [8, 264, 2056])
def test_gelu(ops, cuda_dev, M, F):
    """M = 1..5 and 9 cover the 4-row unroll's tails"""
    dev = cuda_dev
    gen = torch.Generator(device=dev).manual_seed(M * 1000 + F)
    pre = (torch.randn(M, F, generator=gen, device=dev) * 2).to(bf16)
    act = Guarded(M, F, bf16, dev)
    ops.gelu_fwd(_poisoned(pre), act=act.view)
    what = f"gelu M {M} F {F}"
    act.check(what)
    x = pre.double()
    ref = _gelu64(x)
    _expect_close(act.view, ref, _ulp_bf16(ref) + _gelu_tol(x), what + " fwd")
    d = torch.randn(M, F, generator=gen, device=dev).to(bf16)
    work = Guarded(M, F, bf16, dev, init=d)
    ops.gelu_bwd_(_poisoned(pre), work.view)
    work.check(what)
    gg = _gelu_grad64(x)
    ref = d.double() * gg
    _expect_close(work.view, ref, _ulp_bf16(ref) + d.double().abs() * _gelu_grad_tol(x), what + " bwd")


# ----------------------------------------------------------------------------------------------------------------
# LoRA input-dropout backward
# ----------------------------------------------------------------------------------------------------------------
LORA_DX = [(8, 8, 1), (16, 248, 15), (24, 264, 17), (8, 1024, 33), (16, 4096, 16), (24, 56, 2)]


@pytest.mark.parametrize("R,K,M", LORA_DX)
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_lora_dx(ops, cuda_dev, R, K, M, p):
    """dh += mask / (1 - p) * G A. K < 256 columns gives fewer than 32 eight-column groups (a CTA narrower than a warp
    multiple of the row); M tails at the 16-row blocks. Integer G, A, dh keep every value an integer below 256, so p = 0
    is bit-exact; p > 0 is one fp32 fma and one bf16 rounding of the exact value."""
    dev = cuda_dev
    gen = torch.Generator(device=dev).manual_seed(R * K + M)
    G = torch.randint(-2, 3, (M, R), generator=gen, device=dev).to(bf16)
    A = torch.randint(-2, 3, (R, K), generator=gen, device=dev).to(bf16)
    dh0 = torch.randint(-4, 5, (M, K), generator=gen, device=dev).to(bf16)
    dh = Guarded(M, K, bf16, dev, init=dh0)
    d = ops.Drop(p, seed=12, stream=34)
    ops.lora_dx_(dh.view, _poisoned(G, col0=8), _poisoned(A), K, R, d)
    what = f"lora_dx R {R} K {K} M {M} p {p}"
    dh.check(what)
    acc = G.double() @ A.double()
    if p == 0:
        _expect_equal(dh.view, dh0.double() + acc, what)
    else:
        sc = _drop_scale(ops, M, K, d, dev)
        ref = dh0.double() + sc * acc
        _expect_close(dh.view, ref, _ulp_bf16(ref) + U * ref.abs(), what)


# ----------------------------------------------------------------------------------------------------------------
# small fp32 matmul of the similarity API
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ta,tb", list(itertools.product([False, True], repeat=2)))
def test_small_matmul(ops, cuda_dev, ta, tb):
    """integer operands and a power-of-two alpha: exact, whatever the summation order"""
    dev = cuda_dev
    for (M, N, K) in ((17, 33, 40), (5, 3, 1), (64, 16, 48)):
        gen = torch.Generator(device=dev).manual_seed(M + N + K)
        a = torch.randint(-3, 4, (K, M) if ta else (M, K), generator=gen, device=dev).float()
        b = torch.randint(-3, 4, (N, K) if tb else (K, N), generator=gen, device=dev).float()
        c = ops.small_matmul(_poisoned(a), _poisoned(b), trans_a=ta, trans_b=tb, alpha=0.5)
        ref = 0.5 * ((a.double().t() if ta else a.double()) @ (b.double().t() if tb else b.double()))
        _expect_equal(c, ref, f"small_matmul ta {ta} tb {tb} [{M}, {N}, {K}]")


# ----------------------------------------------------------------------------------------------------------------
# cross-entropy rows at the Llama-3 / Qwen vocabularies: bf16 rows above the 200 KB shared-memory cache
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [128256, 151936, 152064])
@pytest.mark.parametrize("inplace", [False, True])
def test_ce_rows_large_vocab(ops, cuda_dev, V, inplace):
    dev, B, L, ld = cuda_dev, 2, 4, V + 64
    gen = torch.Generator(device=dev).manual_seed(V + int(inplace))
    x = (torch.randn(B * L, V, generator=gen, device=dev) * 3).to(bf16)
    base = torch.full((B * L, ld), float("nan"), dtype=bf16, device=dev)
    base[:, :V] = x
    logits = base.view(B, L, ld)[:, :, :V]
    ids = torch.randint(0, V, (B, L), generator=gen, device=dev)
    ids[0, 1], ids[1, 2] = V - 1, 0
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    mask[1, 1] = 0                                                      # a masked token: the row before it is zeroed
    nsum = mask[:, 1:].sum().float().view(1)
    tok_lp, dl = ops.ce_marginal(logits, ids, mask, nsum, need_grad=True, inplace=inplace, grad_out=1.5)
    what = f"ce V {V} inplace {inplace}"
    x64 = x.double()
    lse = torch.logsumexp(x64, 1, keepdim=True)
    t = torch.arange(B * L, device=dev) % L
    nxt = torch.arange(B * L, device=dev) + 1
    valid = t < L - 1
    w = torch.where(valid, mask.view(-1)[nxt.clamp_max(B * L - 1)], torch.zeros_like(t)).double()
    label = torch.where(valid, ids.view(-1)[nxt.clamp_max(B * L - 1)], torch.zeros_like(t))
    lp = (x64.gather(1, label[:, None]) - lse)[:, 0] * (w > 0)
    mx = x64.max(1, keepdim=True).values
    span = mx - x64.min(1, keepdim=True).values
    dlse = _ce_dlse(V, lse, mx, span)
    _expect_close(tok_lp.view(1, -1), lp.view(1, -1), (dlse[:, 0] + U * lp.abs()).view(1, -1) * (w > 0), what + " tok_lp")
    prob = torch.exp(x64 - lse)
    onehot = torch.zeros_like(prob).scatter_(1, label[:, None], 1.0)
    coef = (1.5 * w / nsum.double())[:, None]
    ref = coef * (prob - onehot)
    # p = exp(x - lse): lse's error, the rounding of x - lse and __expf; then - 1, * coef (itself 2 roundings), RNE
    tol = _ulp_bf16(ref) + coef.abs() * (prob * (dlse + 2.0 ** -23 * (3 + 1.2 * (x64 - lse).abs())) + 4 * U * (prob - onehot).abs())
    got = dl.reshape(B * L, V)
    _expect_close(got, ref, tol, what + " dlogits")
    assert torch.equal(got[w == 0].double(), torch.zeros_like(ref[w == 0])), what + ": masked rows not zeroed"
    if inplace:
        assert dl.data_ptr() == logits.data_ptr()
        assert torch.isnan(base[:, V:]).all(), what + ": padding columns written"
