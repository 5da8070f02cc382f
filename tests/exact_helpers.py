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


def _where(bad, what, tile_m=128, tile_n=None, row0=0):
    r, c = bad.nonzero()[0].tolist()
    r += row0
    tile = f" = tile (m {r // tile_m}, n {c // tile_n})" if tile_n else ""
    rows = f" of rows from {row0}" if row0 else ""
    return f"{what}: {int(bad.sum())} of {bad.numel()} elements{rows} wrong; first at (row {r}, col {c}){tile}"


def _expect_equal(got, want, what, tile_m=128, tile_n=None, row0=0):
    """got (kernel output, any float dtype) == want (same dtype) element for element (+0 == -0), no NaN. row0: the row of
    the full output where these rows start (a chunk of a large output), for the failure message"""
    g, w = got.double(), want.double()
    bad = (g != w) | torch.isnan(g)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n, row0) + f": got {g[r, c].item()!r}, want {w[r, c].item()!r}")


def _expect_close(got, ref, tol, what, tile_m=128, tile_n=None, row0=0):
    """|got - ref| <= tol element-wise (fp64), no NaN"""
    g = got.double()
    bad = ~((g - ref).abs() <= tol)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n, row0) + f": got {g[r, c].item()!r}, ref {ref[r, c].item()!r}, "
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
# routed experts: the grouped GEMM over padded expert segments, and the routing's definition
# ----------------------------------------------------------------------------------------------------------------
def _segments(counts):
    """padded row offsets of segments with these row counts"""
    off, o = [], 0
    for c in counts:
        off.append(o)
        o += -(-c // 128) * 128
    return off, o


def _grouped_case(ops, dev, counts, extra, layout, swiglu, N, K, max_ctas, seed, experts=None, E=None, device_ref=False):
    """gemm_grouped on segments of counts[i] rows (padded to the 128-row tile, in this order) with segment i on expert
    experts[i] (default i) of an E-expert stack (default len(counts)), `extra` unused tiles after the live ones. Integer
    operands in [-2, 2]: every row of every segment bit-exact against fp64, the rows past the live tiles untouched.
    device_ref: operands drawn on the device and the fp64 reference computed there, one segment at a time (production
    widths); otherwise drawn from a host generator and checked on the host."""
    experts = list(range(len(counts))) if experts is None else list(experts)
    E = len(counts) if E is None else E
    off, live_rows = _segments(counts)
    n_tiles = live_rows // 128 + extra
    rows = 128 * n_tiles
    wshape = (E, N, K) if layout == 0 else (E, K, N)
    wbuf = torch.full((E + 1,) + wshape[1:], float("nan"), dtype=bf16, device=dev)   # a NaN expert after the last one
    if device_ref:
        g = torch.Generator(device=dev).manual_seed(seed)
        buf = torch.full((rows + PAD_R, K + PAD_C), float("nan"), dtype=bf16, device=dev)
        a = buf[:rows, :K]
        a.copy_(torch.randint(-2, 3, (rows, K), generator=g, device=dev, dtype=torch.int8))
        live_row = torch.zeros(rows, dtype=torch.bool, device=dev)
        for o, c in zip(off, counts):
            live_row[o:o + c] = True
        a.masked_fill_(~live_row[:, None], float("nan"))            # padding rows of every segment and the tail: NaN
        wbuf[:E].copy_(torch.randint(-2, 3, wshape, generator=g, device=dev, dtype=torch.int8))
        a_ref = a
    else:
        g = torch.Generator().manual_seed(seed)
        a_host = torch.full((rows, K), float("nan"))
        for o, c in zip(off, counts):
            a_host[o:o + c] = _ints((c, K), g)
        a = _poisoned(a_host.to(dev, bf16))
        wbuf[:E] = _ints(wshape, g).to(dev, bf16)
        a_ref = a_host
    w = wbuf[:E]
    tiles = torch.full((n_tiles,), -1, dtype=torch.int32)
    for o, c, e in zip(off, counts, experts):
        tiles[o // 128:(o + -(-c // 128) * 128) // 128] = e
    tile_expert = tiles.to(dev)
    live = torch.tensor([live_rows // 128], dtype=torch.int32, device=dev)
    out = Guarded(rows, N, bf16, dev)
    act = Guarded(rows, N // 2, bf16, dev) if swiglu else None
    ops.gemm_grouped(a, w, tile_expert, live, out=out.view, layout=layout, swiglu=swiglu, act=act.view if swiglu else None,
                     max_ctas=max_ctas)
    segs = counts if len(counts) <= 12 else f"{len(counts)} segments, {sum(counts)} rows"
    what = f"gemm_grouped layout {layout} swiglu {swiglu} counts {segs} +{extra} tiles N {N} K {K} max_ctas {max_ctas}"
    if device_ref:
        got, got_act = out.view, act.view if swiglu else None
    else:
        w64 = w.double().cpu()
        got, got_act = out.view.cpu(), act.view.cpu() if swiglu else None
    for i, (o, c, e) in enumerate(zip(off, counts, experts)):
        if c == 0:
            continue
        x = a_ref[o:o + c].double()
        we = w[e].double() if device_ref else w64[e]
        acc = x @ (we.t() if layout == 0 else we)
        _expect_equal(got[o:o + c], acc.to(bf16), f"{what} segment {i} (expert {e}, rows from {o})", 128, 256)
        if swiglu:
            blk = acc.view(c, N // 256, 2, 128)
            gate, up = blk[:, :, 0].reshape(c, N // 2), blk[:, :, 1].reshape(c, N // 2)
            ref = gate * torch.sigmoid(gate) * up
            _expect_close(got_act[o:o + c], ref, _ulp_bf16(ref) + 2.0 ** -20 * ref.abs() + 2.0 ** -100,
                          f"{what} act segment {i} (expert {e})", 128, 128)
    # the tail tiles past the live count are not computed: their rows keep the sentinel
    for v, nm in ((out, "out"), (act, "act")):
        if v is None:
            continue
        tail = v.view[live_rows:].contiguous().view(torch.int16)
        assert bool((tail == v.bits).all()), f"{what}: {nm} rows past the live tiles were written"
        v.check(f"{what} {nm}")


def _check_routing(r, ids, E):
    """a moe_permute result against its definition: counts, padded segment offsets, the tile -> expert table, the live tile
    count, and the pair <-> row maps (within a segment, pairs by token, then by slot)"""
    ids = ids.cpu().long().view(-1)
    P = ids.numel()
    counts = torch.bincount(ids, minlength=E)
    assert torch.equal(r.counts.cpu().long(), counts)
    pad = (counts + 127) // 128 * 128
    off = torch.cat([torch.zeros(1, dtype=torch.long), pad.cumsum(0)])
    assert torch.equal(r.seg_off.cpu().long(), off)
    live = int(off[-1]) // 128
    assert int(r.live.item()) == live
    te = torch.full((r.n_tiles,), -1, dtype=torch.long)
    for e in range(E):
        te[int(off[e]) // 128:int(off[e + 1]) // 128] = e
    assert torch.equal(r.tile_expert.cpu().long(), te)
    pr = r.pair_row.cpu().long()
    want = torch.empty(P, dtype=torch.long)
    for e in range(E):
        sel = (ids == e).nonzero().view(-1)                 # pair order: by token, then slot
        want[sel] = off[e] + torch.arange(sel.numel())
    assert torch.equal(pr, want), "pair -> row map"
    rp = r.row_pair.cpu().long()[:live * 128]
    wrp = torch.full((live * 128,), -1, dtype=torch.long)
    wrp[want] = torch.arange(P)
    assert torch.equal(rp, wrp), "row -> pair map"


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
