"""Poisoned inputs, guarded outputs, element-wise comparisons and the fp64 references shared by the exact kernel tests. The
module-scoped `dev` and `ops` fixtures are used by importing them into a test module.

Every operand is a view into a larger buffer whose padding columns and trailing rows hold NaN, so a kernel that reads past
a row or ignores the row stride picks up NaN. Every output is an interior view surrounded by sentinel guard bands that must
come back bit-unchanged, so a kernel that writes past its view is caught.
"""
import math

import pytest
import torch

bf16, f32 = torch.bfloat16, torch.float32

GUARD_R, GUARD_C = 128, 256                      # guard band around every output: one tile of rows / a 256-wide tile of columns
PAD_R, PAD_C = 128, 64                           # NaN rows after / NaN columns right of every input view
_SENTINEL_BITS = {bf16: (torch.int16, 0x7FA5), f32: (torch.int32, 0x7FA5A5A5)}   # NaN payloads no kernel writes


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from dalm_b200 import _lib
    _lib.call("dalm_b200_probe_device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ops(dev):
    from dalm_b200 import ops as _ops
    return _ops


def _poisoned(x: torch.Tensor, col0: int = 0, pad_c: int = PAD_C) -> torch.Tensor:
    """x [r, c] copied into a NaN buffer [r + 128, col0 + c + pad_c] at column col0: a view whose row stride runs into NaN
    columns and whose rows are followed by NaN rows (1-D: N values followed by 256 NaNs)"""
    if x.dim() == 1:
        buf = torch.full((x.shape[0] + 256,), float("nan"), dtype=x.dtype, device=x.device)
        buf[: x.shape[0]] = x
        return buf[: x.shape[0]]
    r, c = x.shape
    buf = torch.full((r + PAD_R, col0 + c + pad_c), float("nan"), dtype=x.dtype, device=x.device)
    buf[:r, col0:col0 + c] = x
    return buf[:r, col0:col0 + c]


def _dense_poisoned(x: torch.Tensor) -> torch.Tensor:
    """x [r, c] as dense rows (row stride c, the layout the fp32 row kernels index) followed by 128 NaN rows"""
    r, c = x.shape
    buf = torch.full(((r + PAD_R) * c,), float("nan"), dtype=x.dtype, device=x.device)
    buf[: r * c] = x.reshape(-1)
    return buf[: r * c].view(r, c)


class Guarded:
    """an output view [rows, cols] inside a sentinel-filled buffer with GUARD_R rows above / below and GUARD_C columns left /
    right (16-byte aligned: the view starts 256 elements into a row and the row stride is cols + 512). `shift` moves the view
    that many elements right (a start that is not 16-byte aligned) and `ld_extra` widens the row stride."""

    def __init__(self, rows, cols, dtype, dev, init=None, shift=0, ld_extra=0):
        itype, bits = _SENTINEL_BITS[dtype]
        self.buf = torch.full((rows + 2 * GUARD_R, cols + 2 * GUARD_C + ld_extra), bits, dtype=itype, device=dev).view(dtype)
        self.rows, self.cols, self.itype, self.bits, self.c0 = rows, cols, itype, bits, GUARD_C + shift
        self.view = self.buf[GUARD_R:GUARD_R + rows, self.c0:self.c0 + cols]
        if init is not None:
            self.view.copy_(init)

    def check(self, what):
        """the four bands around the view, each compared in place (no copy of the whole buffer: some outputs are GBs)"""
        b = self.buf.view(self.itype)
        r1, c0, c1 = GUARD_R + self.rows, self.c0, self.c0 + self.cols
        for rs, cs in ((slice(0, GUARD_R), slice(None)), (slice(r1, None), slice(None)),
                       (slice(GUARD_R, r1), slice(0, c0)), (slice(GUARD_R, r1), slice(c1, None))):
            bad = b[rs, cs] != self.bits
            if bad.any():
                r, c = bad.nonzero()[0].tolist()
                r += rs.start
                c += cs.start or 0
                pytest.fail(f"{what}: {int(bad.sum())} guard elements overwritten in one band; first at buffer ({r}, {c}) = "
                            f"output ({r - GUARD_R}, {c - self.c0}) of a [{self.rows}, {self.cols}] view")


class Guarded1d:
    """a flat output view of n elements between two sentinel bands of GUARD_C elements (16-byte aligned start): for outputs
    the kernels index by explicit strides (a transposed gradient, a padded KV cache viewed with as_strided)"""

    def __init__(self, n, dtype, dev, init=None):
        itype, bits = _SENTINEL_BITS[dtype]
        self.buf = torch.full((n + 2 * GUARD_C,), bits, dtype=itype, device=dev).view(dtype)
        self.n, self.itype, self.bits = n, itype, bits
        self.view = self.buf[GUARD_C:GUARD_C + n]
        if init is not None:
            self.view.copy_(init.reshape(-1))

    def check(self, what):
        b = self.buf.view(self.itype)
        bad = torch.cat([b[:GUARD_C], b[GUARD_C + self.n:]]) != self.bits
        if bad.any():
            i = int(bad.nonzero()[0])
            at = i - GUARD_C if i < GUARD_C else self.n + i - GUARD_C
            pytest.fail(f"{what}: {int(bad.sum())} guard elements overwritten; first at output offset {at} of {self.n}")


def _ulp_bf16(x):
    """spacing of bf16 numbers at |x| (fp64), normal range"""
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def _ulp_f32(x):
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 23)


def _where(bad, what, tile_m=128, tile_n=None):
    r, c = bad.nonzero()[0].tolist()
    tile = f" = tile (m {r // tile_m}, n {c // tile_n})" if tile_n else ""
    return f"{what}: {int(bad.sum())} of {bad.numel()} elements wrong; first at (row {r}, col {c}){tile}"


def _expect_equal(got, want, what, tile_m=128, tile_n=None):
    """got (kernel output, any float dtype) == want (same dtype) element for element (+0 == -0), no NaN"""
    g, w = got.double(), want.double()
    bad = (g != w) | torch.isnan(g)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n) + f": got {g[r, c].item()!r}, want {w[r, c].item()!r}")


def _expect_close(got, ref, tol, what, tile_m=128, tile_n=None):
    """|got - ref| <= tol element-wise (fp64), no NaN"""
    g = got.double()
    bad = ~((g - ref).abs() <= tol)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n) + f": got {g[r, c].item()!r}, ref {ref[r, c].item()!r}, "
                    f"tol {tol[r, c].item() if torch.is_tensor(tol) else tol!r}")


# ----------------------------------------------------------------------------------------------------------------
# GEMM: integer operands and the tile geometry
# ----------------------------------------------------------------------------------------------------------------
STAGES = {64: 8, 128: 6, 256: 4}                 # GemmCfg<BN>::STAGES: depth of the shared-memory ring
M_EDGE = (1, 127, 128, 129, 255, 256, 257)       # 128 = the CTA tile's rows, 256 = the cluster's


def _ints(shape, g, hi=2):
    return torch.randint(-hi, hi + 1, shape, generator=g).to(f32)


def _gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# erff in fp32: a few ulps, plus the cancellation in 1 + erf(x / sqrt 2) for negative x (~|x| 2^-23): gelu_erf(x) is within
# _gelu_tol(x) of fp64, its derivative within _gelu_grad_tol(x)
def _gelu_tol(x):
    return 2.0 ** -21 * (_gelu64(x).abs() + x.abs())


def _gelu_grad_tol(x):
    return 2.0 ** -20 * (_gelu_grad64(x).abs() + 1)


# __expf is within (2 + 1.16 |x|) ulp (CUDA programming guide); with the IEEE division and products that follow, silu(g)
# and sigmoid(g) are within 2^-19 (1 + |g|) relative
def _silu_tol(g):
    return 2.0 ** -19 * (1 + g.abs())


def _ce_dlse(V, lse, mx, span):
    """bound on |lse - fp64| of a cross-entropy row of V logits (fp32, ce_rows_kernel): the sum of V exponentials has chain
    depth V / 512 + 24, each __expf within (2 + 1.16 |x - max|) ulp; __logf within 2^-21.4 absolute on [0.5, 2] and 3 ulp
    elsewhere; lse and the difference one rounding each. lse, mx (row max), span (max - min): fp64 [rows, 1]"""
    U = 2.0 ** -24
    return (V / 512 + 24) * U + 2.0 ** -23 * (2 + 1.2 * span) + 2.0 ** -21 + 3 * 2.0 ** -23 * (lse - mx) + U * lse.abs()


def _pick_block_n(M, N, sms):
    """the tile width gemm_gelu takes (pick_block_n in gemm_wgmma.cu)"""
    m1, best, bn = -(-M // 128), 1e30, 64
    for cand, pen in ((256, 1.0), (128, 1.55), (64, 2.7)):
        if cand > 64 and N < cand:
            continue
        cost = -(-(m1 * -(-N // cand)) // sms) * cand * pen
        if cost < best:
            best, bn = cost, cand
    return bn


# ----------------------------------------------------------------------------------------------------------------
# attention against fp64
# ----------------------------------------------------------------------------------------------------------------
def _attn_fns(ops, kind):
    return (ops.attention_tc_fwd, ops.attention_tc_bwd) if kind == "wg" else (ops.attention_fwd, ops.attention_bwd)


def _row_mask(B, L, pattern, g):
    mask = torch.ones(B, L, dtype=torch.int64)
    if pattern == "right64":                              # >= 64 pad tokens: a fully masked second KV tile
        mask[0, max(1, L - 70):] = 0
        mask[1, 64:] = 0
        mask[2, L - 5:] = 0
    elif pattern == "left64":
        mask[0, : min(L - 1, max(64, L - 10))] = 0
        mask[1, :64] = 0
        mask[2, :3] = 0
    elif pattern == "holes":
        mask = (torch.rand(B, L, generator=g) > 0.3).long()
        mask[1, 10:min(L - 1, 74)] = 0
        mask[:, 0] = 1
    elif pattern == "empty":                              # sample 1: every key masked
        mask[0, L - 7:] = 0
        mask[1] = 0
    return mask


def _attn_ref64(q, k, v, vis, B, L, Hq, Hkv, D, scale):
    """fp64 attention with an explicit safe softmax: rows without a visible key give zero output, lse -inf, zero gradient"""
    qh = q.view(B, L, Hq, D).transpose(1, 2)
    kh = k.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, 1)
    vh = v.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, 1)
    s = (qh @ kh.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    m = s.amax(-1, keepdim=True).detach()
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    o = (e / torch.where(l > 0, l, torch.ones_like(l))) @ vh
    return o.transpose(1, 2).reshape(B * L, Hq * D), (m + torch.log(l)).squeeze(-1).detach()


def _attn_bwd64(q, k, v, d_out, o, vis, B, L, Hq, Hkv, D, scale):
    """fp64 flash-attention backward: P from fp64 scores, delta = rowsum(dO * O) from the given output,
    dS = P (dP - delta) scale; -> dq [B*L, Hq*D], dk / dv [B*L, Hkv*D] (summed over the q heads of each kv head)"""
    G = Hq // Hkv
    qh = q.view(B, L, Hq, D).transpose(1, 2)
    kh = k.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(G, 1)
    vh = v.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(G, 1)
    doh = d_out.view(B, L, Hq, D).transpose(1, 2)
    oh = o.view(B, L, Hq, D).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    dp = doh @ vh.transpose(-1, -2)
    delta = (doh * oh).sum(-1, keepdim=True)
    ds = p * (dp - delta) * scale
    dq = ds @ kh
    dk = (ds.transpose(-1, -2) @ qh).view(B, Hkv, G, L, D).sum(2)
    dv = (p.transpose(-1, -2) @ doh).view(B, Hkv, G, L, D).sum(2)
    flat = lambda t, H: t.transpose(1, 2).reshape(B * L, H * D)
    return flat(dq, Hq), flat(dk, Hkv), flat(dv, Hkv)


# ----------------------------------------------------------------------------------------------------------------
# Qwen3's q / k RMSNorm before RoPE (head_dim 128, theta 1e6)
# ----------------------------------------------------------------------------------------------------------------
NORM_STD = 0.5                                   # q / k norm weights are drawn 1 + N(0, NORM_STD)
EPS = 1e-6                                       # rms_norm_eps


def _tables(dev, T, poison=True):
    inv = 1.0 / (1e6 ** (torch.arange(0, 128, 2, dtype=f32) / 128))
    fr = torch.outer(torch.arange(T, dtype=f32), inv)
    if not poison:
        return fr.cos().to(dev).contiguous(), fr.sin().to(dev).contiguous()
    cbuf = torch.full((T + 128, 64), float("nan"), device=dev); cbuf[:T] = fr.cos().to(dev)
    sbuf = torch.full((T + 128, 64), float("nan"), device=dev); sbuf[:T] = fr.sin().to(dev)
    return cbuf[:T], sbuf[:T]


def _norm_w(g, dev):
    return _poisoned((1 + torch.randn(128, generator=g) * NORM_STD).to(dev))


def _ref_norm_rope(y, nheads, nq, wq, wk, cos_t, sin_t, pos):
    """fp64 Qwen3 q/k path on y[:, :128 nheads]: (rotated, rstd, magnitude terms of the rotation)"""
    M = y.shape[0]
    h = y[:, :128 * nheads].double().reshape(M, nheads, 128)
    rstd = 1.0 / torch.sqrt((h * h).mean(-1) + EPS)
    w = torch.stack([wq.double() if i < nq else wk.double() for i in range(nheads)])[None]
    xn = h * rstd[..., None] * w
    c, s = cos_t.double()[pos][:, None], sin_t.double()[pos][:, None]
    x1, x2 = xn[..., :64], xn[..., 64:]
    rot = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).reshape(M, 128 * nheads)
    terms = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1).reshape(M, 128 * nheads)
    return rot, rstd, terms
