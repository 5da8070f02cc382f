"""Element-wise checks of the wgmma GEMM and the attention kernels at the tile edges where they go wrong.

GEMM: operands are small integers, so every product and partial sum is exact in fp32 whatever the accumulation order, and
the kernels' outputs can be compared with an fp64 reference bit for bit (fp32 outputs) or with its round-to-nearest-even
bf16 image (bf16 outputs). Activations, which no exact reference exists for, are compared element by element within a stated
number of ulps of fp64 applied to the exact pre-activation.

Attention: "selector" inputs make the softmax one-hot to far below an fp32 ulp, so `out` must equal V[target] bit for bit
and `lse` must equal the fp64 log-sum-exp; higher-scoring "attractor" keys sit everywhere a kernel must not look (masked
keys, keys after the diagonal, the next sample's rows inside the last tile). Random inputs are checked per row against fp64.

Every operand is a view into a larger buffer whose padding columns and trailing rows hold NaN, and every output is an
interior view surrounded by sentinel guard bands (128 rows, 256 columns) that must come back bit-unchanged.
"""
import math
import random

import pytest
import torch

from exact_helpers import (M_EDGE, PAD_R, STAGES, Guarded, _attn_fns, _attn_ref64, _expect_close, _expect_equal,  # noqa: F401
                           _gelu64, _ints, _pick_block_n, _poisoned, _row_mask, _ulp_bf16, _ulp_f32, dev, ops)

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64


# ----------------------------------------------------------------------------------------------------------------
# 1. GEMM: integer operands, exact comparison
# ----------------------------------------------------------------------------------------------------------------
M_EDGE_WGRAD = (8, 120, 128, 136, 248, 256, 264)  # the wgrad layout needs M % 8 == 0
K_EDGE = (8, 56, 64, 72)                         # 64 = one k-block
T_EDGE = (1, 7, 63, 65)                          # wgrad contraction over token rows: no multiple-of-8 requirement

# epilogue variants, cycled over the shapes so that each kernel instance meets each of them. Bias and residual values are
# integers in +-4096 / +-2048, so bf16 outputs are large enough for round-to-nearest-even to matter; alpha is a power of two.
VARIANTS = (
    dict(out=f32),
    dict(out=bf16, alpha=0.5, bias=True),
    dict(out=f32, alpha=0.25, bias=True, resid=f32),
    dict(out=bf16, bias=True, resid=bf16),
    dict(out=f32, bias=True, act=1),
    dict(out=bf16, alpha=2.0, act=1),
    dict(out=f32, alpha=2.0, resid=f32, inplace=True),
    dict(out=f32, bias=True, resid=f32, drop=0.1),
    dict(out=bf16, bias=True, act=2),
    dict(out=bf16, alpha=4.0, resid=bf16, inplace=True),
)


def _gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def _run_gemm(ops, dev, layout, bn, M, N, K, var, max_ctas=0, seed=0):
    """one ops.gemm call on poisoned operands into a guarded output, checked element-wise against fp64"""
    g = torch.Generator().manual_seed(seed)
    ash, bsh = {0: ((M, K), (N, K)), 1: ((M, K), (K, N)), 2: ((K, M), (K, N))}[layout]
    a = _poisoned(_ints(ash, g).to(dev, bf16))
    b = _poisoned(_ints(bsh, g).to(dev, bf16))
    a64, b64 = a.double(), b.double()
    acc = a64 @ b64.t() if layout == 0 else (a64 @ b64 if layout == 1 else a64.t() @ b64)
    alpha = var.get("alpha", 1.0)
    x = alpha * acc
    bias = None
    if var.get("bias"):
        bv = _ints((N,), g, 4096).to(dev)
        bias = _poisoned(bv)
        x = x + bv.double()
    odt, act = var["out"], var.get("act", 0)
    rdt = var.get("resid")
    resid_vals = None
    if act == 2:
        resid_vals = (torch.randn(M, N, generator=g) * 2).to(dev, bf16)
    elif rdt is not None:
        resid_vals = _ints((M, N), g, 2048 if rdt == f32 else 256).to(dev, rdt)
    out = Guarded(M, N, odt, dev, init=resid_vals if var.get("inplace") else None)
    if var.get("inplace"):
        resid = out.view
    elif resid_vals is not None:
        resid = _poisoned(resid_vals)
    else:
        resid = None
    drop = ops.Drop(var["drop"], seed=77 + seed, stream=5) if var.get("drop") else None
    ops.gemm(a, b, out=out.view, out_dtype=odt, alpha=alpha, bias=bias, act=act, resid=resid, block_n=bn,
             max_ctas=max_ctas, drop=drop, layout=layout)
    what = f"gemm layout {layout} block_n {bn} M {M} N {N} K {K} max_ctas {max_ctas} {var}"
    tm, tn = (256, bn % 1000) if bn > 1000 else (128, bn)
    got = out.view
    if act == 0 and drop is None:
        want = x + (resid_vals.double() if resid_vals is not None else 0)
        _expect_equal(got, want.to(odt), what, tm, tn)            # exact: fp32 bit for bit, bf16 = RNE of the exact value
    elif act == 1:
        ref = _gelu64(x)
        # erff in fp32: a few ulps of the result, plus the cancellation in 1 + erf(x / sqrt 2) for negative x (~|x| 2^-23)
        slack = 2.0 ** -21 * (ref.abs() + x.abs())
        tol = (_ulp_bf16(ref) if odt == bf16 else 0) + slack
        _expect_close(got, ref, tol, what, tm, tn)
    elif act == 2:
        d = x.to(bf16).double()                                   # the dgrad value is rounded to bf16 before the product
        gg = _gelu_grad64(resid_vals.double())
        ref = d * gg
        tol = _ulp_bf16(ref) + 2.0 ** -20 * d.abs() * (gg.abs() + 1)
        _expect_close(got, ref, tol, what, tm, tn)
    else:
        # dropout on act(alpha acc + bias) before the residual: the scale 1/(1-p) is not a power of two, so the product is
        # rounded once in fp32 (possibly fused with the residual add): within one fp32 ulp of the larger term
        sc = ops.dropout_scale(M * N, drop, dev).view(M, N).double()
        xs = x * sc
        ref = xs + (resid_vals.double() if resid_vals is not None else 0)
        tol = _ulp_f32(torch.maximum(ref.abs(), xs.abs()))
        _expect_close(got, ref, tol, what, tm, tn)
    out.check(what)


def _n_edges(bn):
    t = bn % 1000
    return (t - 8, t, t + 8)


@pytest.mark.gpu
@pytest.mark.parametrize("layout,bn", [(l, b) for l in (0, 1, 2) for b in (64, 128, 256)] + [(0, 2128), (0, 2256)])
def test_gemm_exact_edges(ops, dev, layout, bn):
    """every plain / cluster kernel instance at M, N and K (or T) on and around its tile edges"""
    ms = M_EDGE_WGRAD if layout == 2 else M_EDGE
    ks = T_EDGE if layout == 2 else K_EDGE
    i = 0
    for M in ms:
        for N in _n_edges(bn):
            for K in ks:
                _run_gemm(ops, dev, layout, bn, M, N, K, VARIANTS[i % len(VARIANTS)], seed=i)
                i += 1


@pytest.mark.gpu
@pytest.mark.parametrize("layout,bn", [(l, b) for l in (0, 1, 2) for b in (64, 128, 256)] + [(0, 2128), (0, 2256)])
def test_gemm_exact_ring_depth(ops, dev, layout, bn):
    """k-block counts just below, at and above the ring depth with 1-3 CTAs (clusters) walking 9 tiles each, so that the
    ring's stage / phase carry over from one tile to the next"""
    tn = bn % 1000
    S = STAGES[tn]
    M = 264 if layout == 2 else (513 if bn > 1000 else 257)
    N = 2 * tn + 8
    i = 0
    for nkb in (S - 1, S, S + 1):
        K = 64 * nkb - (0 if layout != 2 else 3)                 # wgrad: a ragged last k-block of token rows
        for ctas in (1, 2, 3):
            _run_gemm(ops, dev, layout, bn, M, N, K, VARIANTS[(i + 3 * layout) % len(VARIANTS)],
                      max_ctas=ctas * (2 if bn > 1000 else 1), seed=100 + i)
            i += 1


def _gelu_shapes(sms):
    small = [(M, N, K) for M in M_EDGE for N in (56, 64, 72, 120, 128, 136, 248, 256, 264) for K in (8, 72)]
    big = [(M, N, 8) for M in (128 * sms, 128 * sms + 1) for N in (128, 136, 248, 256, 264)]   # multi-wave: wider tiles pay
    return small + big


@pytest.mark.gpu
def test_gemm_gelu_exact(ops, dev):
    """gemm_gelu (pre-activation and gelu(pre), one launch) at every tile width its heuristic picks"""
    sms = ops.num_sms()
    shapes = _gelu_shapes(sms)
    assert {_pick_block_n(M, N, sms) for M, N, _ in shapes} == {64, 128, 256}
    for i, (M, N, K) in enumerate(shapes):
        g = torch.Generator().manual_seed(i)
        a = _poisoned(_ints((M, K), g).to(dev, bf16))
        w = _poisoned(_ints((N, K), g).to(dev, bf16))
        bv = _ints((N,), g, 4096).to(dev) if i % 2 else None
        pre, act = Guarded(M, N, bf16, dev), Guarded(M, N, bf16, dev)
        ops.gemm_gelu(a, w, bias=None if bv is None else _poisoned(bv), pre=pre.view, act=act.view)
        tn = _pick_block_n(M, N, sms)
        what = f"gemm_gelu M {M} N {N} K {K} block_n {tn} bias {bv is not None}"
        x = a.double() @ w.double().t() + (0 if bv is None else bv.double())
        _expect_equal(pre.view, x.to(bf16), what + " pre", 128, tn)
        p = x.to(bf16).double()                                   # gelu is taken of the rounded pre-activation
        ref = _gelu64(p)
        _expect_close(act.view, ref, _ulp_bf16(ref) + 2.0 ** -21 * (ref.abs() + p.abs()), what + " act", 128, tn)
        pre.check(what + " pre"); act.check(what + " act")


@pytest.mark.gpu
def test_gemm_swiglu_exact(ops, dev):
    """gate|up projection with SiLU(gate) * up in the epilogue: gu bit-exact, act within one bf16 ulp of fp64"""
    i = 0
    for M in M_EDGE:
        for N in (256, 512):
            for K in K_EDGE:
                g = torch.Generator().manual_seed(200 + i)
                a = _poisoned(_ints((M, K), g).to(dev, bf16))
                w = _poisoned(_ints((N, K), g).to(dev, bf16))
                gu, act = Guarded(M, N, bf16, dev), Guarded(M, N // 2, bf16, dev)
                ops.gemm_swiglu(a, w, gu=gu.view, act=act.view)
                what = f"gemm_swiglu M {M} N {N} K {K}"
                acc = a.double() @ w.double().t()
                _expect_equal(gu.view, acc.to(bf16), what + " gu", 128, 256)
                blk = acc.view(M, N // 256, 2, 128)
                gate, up = blk[:, :, 0].reshape(M, N // 2), blk[:, :, 1].reshape(M, N // 2)
                ref = gate * torch.sigmoid(gate) * up                 # from the fp32 accumulators, not the rounded gu
                # __expf and the division: a few fp32 ulps before the bf16 rounding; 2^-100 absorbs silu(g) of very negative g
                # (exp overflows to inf in fp32 and the kernel returns -0 where fp64 has a sub-bf16-denormal value)
                _expect_close(act.view, ref, _ulp_bf16(ref) + 2.0 ** -20 * ref.abs() + 2.0 ** -100, what + " act", 128, 128)
                gu.check(what + " gu"); act.check(what + " act")
                i += 1


@pytest.mark.gpu
def test_gemm_rope_exact(ops, dev):
    """q|k|v projection with RoPE in the epilogue: rotated columns within one bf16 ulp, the rest bit-exact"""
    Lr = 37                                               # rows wrap around the position table
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, dtype=f32) / 128))
    fr = torch.outer(torch.arange(Lr, dtype=f32), inv)
    # the tables must be contiguous [L, 64]: poisoned by NaN rows after them only
    cbuf = torch.full((Lr + PAD_R, 64), float("nan"), device=dev); cbuf[:Lr] = fr.cos().to(dev)
    sbuf = torch.full((Lr + PAD_R, 64), float("nan"), device=dev); sbuf[:Lr] = fr.sin().to(dev)
    cos_t, sin_t = cbuf[:Lr], sbuf[:Lr]
    i = 0
    for M in M_EDGE:
        for N, rope_cols in ((256, 256), (264, 256), (504, 256), (512, 512), (520, 512)):
            for K in (8, 72):
                g = torch.Generator().manual_seed(300 + i)
                a = _poisoned(_ints((M, K), g).to(dev, bf16))
                w = _poisoned(_ints((N, K), g).to(dev, bf16))
                out = Guarded(M, N, bf16, dev)
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=out.view)
                what = f"gemm_rope M {M} N {N} K {K} rope_cols {rope_cols}"
                y = a.double() @ w.double().t()
                pos = torch.arange(M, device=dev) % Lr
                c, s = cos_t.double()[pos], sin_t.double()[pos]                  # [M, 64]
                h = y[:, :rope_cols].reshape(M, rope_cols // 128, 2, 64)
                x1, x2 = h[:, :, 0], h[:, :, 1]
                c, s = c[:, None], s[:, None]
                rot = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).view(M, rope_cols)
                terms = torch.stack([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], 2).view(M, rope_cols)
                # fmaf(own, cos, -oth * sin): the sin product is rounded in fp32 before the fused add
                _expect_close(out.view[:, :rope_cols], rot, _ulp_bf16(rot) + 2.0 ** -22 * terms, what + " rotated", 128, 256)
                _expect_equal(out.view[:, rope_cols:], y[:, rope_cols:].to(bf16), what + " plain", 128, 256)
                out.check(what)
                i += 1


# ----------------------------------------------------------------------------------------------------------------
# 2. attention: selector inputs (exact) and per-row checks of random inputs
# ----------------------------------------------------------------------------------------------------------------
TARGET_AMP, ATTRACT_AMP = 4.0, 8.0
MIN_MARGIN = 104.0          # nats: exp(-104) < 2^-149, so every non-target weight underflows to exactly 0 in fp32


def _hadamard(n):
    h = torch.ones(1, 1, dtype=f64)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


def _selector_mask(B, L):
    """sample 0: right padding, 1: left padding, 2: interior holes; every sample keeps at least one key"""
    mask = torch.ones(B, L, dtype=torch.int64)
    n = max(1, L // 3) if L > 1 else 0
    if n:
        mask[0, L - n:] = 0
        if B > 1:
            mask[1, :n] = 0
        if B > 2:
            mask[2, 1::3] = 0
    return mask


def _selector_case(B, L, Hq, Hkv, D, causal, scale, seed):
    """Inputs whose softmax is one-hot. Keys are sums of Hadamard rows, k_j = sum_c amp[j, c] H[c]; query i is aq H[cls_i], so
    its score against key j is scale * aq * D * amp[j, cls_i] and zero for every class it does not carry. Each sample uses its
    own half of the classes. Targets carry amplitude 4 in distinct classes; attractors carry 8 in a target's class at masked
    keys, at keys after the diagonal that only queries of later targets can see (causal), and in the first rows of the next
    sample that fall into this sample's last 64-row tile (in a class of this sample, invisible to the next one's queries).
    aq makes the target score at least 110 nats. Returns fp64 CPU q, k, v [B*L, H*D], the mask and target[b, h, i] (-1: no
    visible key)."""
    g = torch.Generator().manual_seed(seed)
    rng = random.Random(seed)
    mask = _selector_mask(B, L)
    H = _hadamard(D)
    half = D // 2
    aq = 2.0 ** math.ceil(math.log2(110.0 / (TARGET_AMP * D * scale)))
    over = (-L) % 64
    amp = torch.zeros(B, Hkv, L, D, dtype=f64)
    target = torch.full((B, Hq, L), -1, dtype=torch.int64)
    qcls = torch.zeros(B, Hq, L, dtype=torch.int64)
    group = Hq // Hkv
    des_cls = {}
    for b in range(B):
        own = list(range(0, half)) if b % 2 == 0 else list(range(half, D))
        vis = [j for j in range(L) if mask[b, j]]
        for hk in range(Hkv):
            if causal:
                step = max(2, -(-len(vis) // half))
                des = vis[::step]
            else:
                des = sorted(set(rng.sample(vis, min(len(vis), 5))) | {vis[-1]})
            perm = rng.sample(range(half), half)
            cls = {j: own[perm[n]] for n, j in enumerate(des)}
            dc = list(cls.values())
            des_cls[b, hk] = dc
            for j, c in cls.items():
                amp[b, hk, j, c] += TARGET_AMP
            for j in range(L):
                if not mask[b, j]:
                    amp[b, hk, j, rng.choice(dc)] += ATTRACT_AMP
                elif causal and j not in cls:
                    retired = [cls[des[n]] for n in range(len(des) - 1) if des[n + 1] <= j]
                    if retired:
                        amp[b, hk, j, rng.choice(retired)] += ATTRACT_AMP
            if b > 0 and over and des_cls[b - 1, hk]:
                prev = des_cls[b - 1, hk]
                for j in range(min(over, L)):
                    amp[b, hk, j, rng.choice(prev)] += ATTRACT_AMP
            for h in range(hk * group, (hk + 1) * group):
                for i in range(L):
                    if causal:
                        seen = [t for t in des if t <= i]
                        t = seen[-1] if seen else -1
                    else:
                        t = rng.choice(des) if des else -1
                    target[b, h, i] = t
                    qcls[b, h, i] = cls[t] if t >= 0 else own[0]
    q = (aq * H[qcls]).permute(0, 2, 1, 3).reshape(B * L, Hq * D)               # [B, Hq, L, D] -> token-major
    k = (amp @ H).permute(0, 2, 1, 3).reshape(B * L, Hkv * D)
    sign = torch.where(torch.rand(B * L, Hkv * D, generator=g) < 0.5, -1.0, 1.0)
    v = (sign * (0.25 + 2 * torch.rand(B * L, Hkv * D, generator=g))).to(bf16).to(f64)   # no zeros
    return dict(q=q, k=k, v=v, mask=mask, target=target, B=B, L=L, Hq=Hq, Hkv=Hkv, D=D, causal=causal, scale=scale)


def _visible(mask, L, causal):
    vis = mask.bool()[:, None, None, :].expand(-1, 1, L, L)                        # [B, 1, Lq, Lk]
    if causal:
        vis = vis & torch.ones(L, L, dtype=torch.bool, device=mask.device).tril()
    return vis


def _scores(c):
    B, L, Hq, Hkv, D = c["B"], c["L"], c["Hq"], c["Hkv"], c["D"]
    qh = c["q"].view(B, L, Hq, D).transpose(1, 2)
    kh = c["k"].view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, 1)
    return c["scale"] * (qh @ kh.transpose(-1, -2))


# (kind, D, dropout, L, causal, Hq, Hkv, scale); Hq / Hkv = 1, 2 and 71 (Falcon-7B's multi-query attention)
def _selector_params():
    out = []
    kinds = (("wg", 64, False), ("wg", 64, True), ("wg", 128, False), ("mma", 32, False), ("mma", 32, True),
             ("mma", 64, False), ("mma", 128, False))
    for L in (1, 2, 31, 32, 33, 63, 64, 65, 127, 129):
        for n, (kind, D, drop) in enumerate(kinds):
            for causal in ((False,) if drop else (False, True)):
                hq, hkv = ((2, 2), (4, 2), (71, 1))[(L + n + causal) % 3]
                scale = 0.05 if (L + n) % 4 == 3 else 1.0 / math.sqrt(D)
                out.append(pytest.param(kind, D, drop, L, causal, hq, hkv, scale,
                                        id=f"{kind}{D}{'-drop' if drop else ''}-L{L}-{'causal' if causal else 'bidir'}-h{hq}x{hkv}"
                                           f"{'-scale' if scale == 0.05 else ''}"))
    return out


SELECTOR_PARAMS = _selector_params()


@pytest.mark.parametrize("kind,D,drop,L,causal,Hq,Hkv,scale", SELECTOR_PARAMS)
def test_selector_construction(kind, D, drop, L, causal, Hq, Hkv, scale):
    """CPU: the fp64 reference of every selector case picks the intended key for every row, with a margin that makes all
    other weights vanish in fp32, and attractors outrank the target where the kernel must not look"""
    B = 3
    c = _selector_case(B, L, Hq, Hkv, D, causal, scale, seed=L * 7 + D)
    s = _scores(c)
    vis = _visible(c["mask"], L, causal)
    tgt = c["target"]
    valid = vis.expand(B, Hq, L, L).any(-1)
    assert torch.equal(valid, tgt >= 0)
    sv = s.masked_fill(~vis, float("-inf"))
    best, arg = sv.max(-1)
    assert torch.equal(arg[valid], tgt[valid])
    assert (best[valid] >= 110.0).all()
    second = sv.scatter(-1, arg[..., None], float("-inf")).max(-1).values
    assert ((best - second)[valid] >= MIN_MARGIN).all()
    hidden = s.masked_fill(vis, float("-inf")).max(-1).values
    if (c["mask"] == 0).any() or (causal and L > 2):
        assert (hidden[valid] > best[valid]).any(), "no attractor hidden behind a mask"
    over = (-L) % 64
    if over:                                              # the next sample's rows in this sample's last tile outrank the target
        kh = c["k"].view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, 1)
        qh = c["q"].view(B, L, Hq, D).transpose(1, 2)
        leak = c["scale"] * (qh[:-1] @ kh[1:, :, : min(over, L)].transpose(-1, -2))
        assert (leak.max(-1).values > best[:-1])[valid[:-1]].any(), "no attractor in the next sample's rows"


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,drop,L,causal,Hq,Hkv,scale", SELECTOR_PARAMS)
def test_attention_selector_exact(ops, dev, kind, D, drop, L, causal, Hq, Hkv, scale):
    """out == V[target] bit for bit (times the bf16-rounded dropout scale), lse == fp64 log-sum-exp within 1e-4"""
    B = 3
    c = _selector_case(B, L, Hq, Hkv, D, causal, scale, seed=L * 7 + D)
    q, k, v = (_poisoned(c[n].to(dev, bf16)) for n in ("q", "k", "v"))
    mask = c["mask"].to(dev)
    out = Guarded(B * L, Hq * D, bf16, dev)
    dr = ops.Drop(0.1, seed=1234 + L, stream=9) if drop else None
    fwd, _ = _attn_fns(ops, kind)
    _, lse = fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out.view, scale=scale, drop=dr)
    tgt = c["target"].to(dev)
    valid = tgt >= 0
    vh = c["v"].to(dev).view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, 1)     # [B, Hq, L, D]
    want = torch.gather(vh, 2, tgt.clamp_min(0)[..., None].expand(-1, -1, -1, D))
    if drop:
        Lp = (L + 7) // 8 * 8
        sc = ops.dropout_scale(B * Hq * L * Lp, dr, dev).view(B, Hq, L, Lp)[..., :L]
        # the kernel rounds the dropped probability (1 or 0 times 1/(1-p)) to bf16 before P V
        want = want * torch.gather(sc, 3, tgt.clamp_min(0)[..., None]).to(bf16).double()
    want = torch.where(valid[..., None], want, torch.zeros((), dtype=f64, device=dev))
    what = f"{kind} attention D {D} L {L} causal {causal} Hq {Hq} Hkv {Hkv} drop {drop}"
    got = out.view.view(B, L, Hq, D).transpose(1, 2)
    bad = ((got.double() != want.to(bf16).double()) | torch.isnan(got)).any(-1)
    if bad.any():
        b, h, i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} wrong output rows; first (sample {b}, head {h}, query {i}), target key "
                    f"{tgt[b, h, i].item()}, 64-row tile {i // 64}")
    s = _scores({**c, "q": c["q"].to(dev), "k": c["k"].to(dev)})
    ref = torch.logsumexp(s.masked_fill(~_visible(mask, L, causal), float("-inf")), -1)
    assert torch.isinf(lse[~valid]).all() and (lse[~valid] > 0).all(), f"{what}: rows without a visible key need lse = +inf"
    err = (lse.double() - ref).abs()[valid]
    print(f"[selector] {what}: max |lse - fp64| = {err.max().item() if err.numel() else 0.0:.3e}")
    if err.numel() and err.max() > 1e-4:
        b, h, i = torch.nonzero(valid)[err.argmax()].tolist()
        pytest.fail(f"{what}: lse off by {err.max().item():.3e} at (sample {b}, head {h}, query {i})")
    out.check(what + " out")


ROW_PARAMS = [
    ("wg", 64, 128, False, "right64", 4, 2, None), ("wg", 128, 128, False, "right64", 2, 2, None),
    ("mma", 32, 128, False, "right64", 4, 4, None), ("mma", 64, 128, False, "right64", 4, 1, None),
    ("wg", 64, 128, False, "left64", 4, 4, None), ("wg", 128, 100, False, "left64", 4, 2, None),
    ("mma", 32, 128, False, "left64", 2, 2, None),
    ("wg", 64, 129, False, "holes", 4, 2, None), ("wg", 128, 97, True, "holes", 4, 1, None),
    ("mma", 64, 129, True, "holes", 2, 2, None), ("mma", 32, 65, False, "holes", 4, 4, None),
    ("wg", 64, 128, False, "empty", 4, 4, None), ("wg", 128, 65, False, "empty", 2, 1, None),
    ("mma", 32, 128, False, "empty", 2, 2, None), ("mma", 128, 63, False, "empty", 2, 2, None),
    ("wg", 64, 96, True, "right64", 4, 2, 0.07), ("wg", 128, 130, False, "holes", 2, 2, 0.2),
    ("mma", 32, 77, False, "right64", 4, 4, 0.3),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,L,causal,pattern,Hq,Hkv,scale", ROW_PARAMS)
def test_attention_rows_vs_fp64(ops, dev, kind, D, L, causal, pattern, Hq, Hkv, scale):
    """random inputs, forward and backward, every row against fp64: fully masked KV tiles, >= 64 left-pad tokens, interior
    holes, a sample with every key masked (zero output, lse = +inf, zero gradients) and non-default scales"""
    B = 3
    g = torch.Generator().manual_seed(L * 31 + D)
    mask = _row_mask(B, L, pattern, g)
    sc = 1.0 / math.sqrt(D) if scale is None else scale
    q0 = torch.randn(B * L, Hq * D, generator=g).to(bf16)
    k0 = torch.randn(B * L, Hkv * D, generator=g).to(bf16)
    v0 = torch.randn(B * L, Hkv * D, generator=g).to(bf16)
    do0 = torch.randn(B * L, Hq * D, generator=g).to(bf16)
    q, k, v, d_out = (_poisoned(t.to(dev)) for t in (q0, k0, v0, do0))
    mask = mask.to(dev)
    fwd, bwd = _attn_fns(ops, kind)
    out = Guarded(B * L, Hq * D, bf16, dev)
    _, lse = fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out.view, scale=sc)
    dq, dk, dv = Guarded(B * L, Hq * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev)
    bwd(q, k, v, mask, out.view, lse, d_out, B, L, Hq, Hkv, D, causal, dq=dq.view, dk=dk.view, dv=dv.view, scale=sc)
    what = f"{kind} attention D {D} L {L} causal {causal} {pattern} Hq {Hq} Hkv {Hkv} scale {sc:.4g}"
    vis = _visible(mask, L, causal)
    qd, kd, vd = (t.double().requires_grad_(True) for t in (q, k, v))
    ref, lse_ref = _attn_ref64(qd, kd, vd, vis, B, L, Hq, Hkv, D, sc)
    ref.backward(d_out.double())
    for name, t in (("out", out.view), ("lse", lse), ("dq", dq.view), ("dk", dk.view), ("dv", dv.view)):
        assert not torch.isnan(t).any(), f"{what}: NaN in {name}"
    # forward, element-wise: bf16 P and the bf16 output each cost 2^-9 relative; bound 2^-7 of the largest |v| of the head
    vmax = v.double().abs().view(B, L, Hkv, D).amax((1, 3)).repeat_interleave(Hq // Hkv, 1)   # [B, Hq]
    tol = (vmax[:, None, :, None] / 128).expand(B, L, Hq, D).reshape(B * L, Hq * D)
    _expect_close(out.view, ref.detach(), tol, what + " out", 64)
    valid = vis.expand(B, Hq, L, L).any(-1)
    assert (torch.isinf(lse[~valid]) & (lse[~valid] > 0)).all(), f"{what}: rows without a visible key need lse = +inf"
    lerr = (lse.double() - lse_ref).abs()[valid]
    print(f"[rows] {what}: max |lse - fp64| = {lerr.max().item():.3e}")
    assert lerr.max() < 1e-4, f"{what}: lse off by {lerr.max().item():.3e}"
    # backward, per row (a token's gradient for one head): error norm <= 4% of the row's norm + 1% of the median row norm.
    # Rows that no visible (query, key) pair reaches must be exactly zero: dq of a query without a visible key, dk / dv of a
    # masked key.
    no_query = (~valid).permute(0, 2, 1).reshape(B * L, Hq)
    masked_key = (mask == 0).reshape(B * L, 1).expand(B * L, Hkv)
    for name, got, want, H, zero in (("dq", dq.view, qd.grad, Hq, no_query), ("dk", dk.view, kd.grad, Hkv, masked_key),
                                     ("dv", dv.view, vd.grad, Hkv, masked_key)):
        gr, wr = got.double().view(B * L, H, D), want.view(B * L, H, D)
        err, nrm = (gr - wr).norm(dim=-1), wr.norm(dim=-1)
        med = nrm[~zero].median()
        lim = 0.04 * nrm + 0.01 * med
        bad = err > lim
        print(f"[rows] {what}: {name} max row error / bound = {(err / lim).max().item():.3e}")
        if bad.any():
            r, h = bad.nonzero()[0].tolist()
            pytest.fail(f"{what}: {name} {int(bad.sum())} bad rows; first token {r} (sample {r // L}, position {r % L}) head {h}: "
                        f"error {err[r, h].item():.3e} vs row norm {nrm[r, h].item():.3e}")
        assert (gr[zero] == 0).all(), f"{what}: {name} nonzero where every contribution is masked"
    for name, gd in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
        gd.check(f"{what} {name}")
