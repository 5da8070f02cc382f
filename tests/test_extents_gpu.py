"""The kernels at the extents production reaches: row, batch and query counts past the grid's 65535 limit on y / z, one
logits buffer past 2^31 elements, and attention at 8192 tokens.

A. A launcher that puts a count on grid.y or grid.z either launches it in chunks or refuses it by name. The chunked ones are
   called just below, at and just above the limit and at about twice it with a ragged tail, with narrow rows, and every
   element is checked (the chunk seams separately: a wrong chunk base shows up only there).
B. The unchunked lm_head (DALM_B200_CHUNKED_HEAD=0) materialises [B*L, V] logits: at the Llama 3 vocabulary 16768 rows pass
   2^31 elements. The GEMM epilogue and the cross-entropy rows must index them with 64-bit offsets.
C. Attention at L = 8192 (128 key tiles), every row of out / lse / dq / dk / dv against fp64, within bounds derived from the
   kernels' arithmetic. Each case carries a control: the fp64 reference with the last visible key tile of every query dropped
   must miss the forward bound on at least one row that sees at least half as many keys as the longest row, so the bound can
   see a one-tile error at this length.

Inputs are NaN-poisoned views and outputs sit inside sentinel guard bands (exact_helpers). The fp64 references run on the
GPU, in row, chunk or head pieces. U = 2^-24 is the fp32 unit roundoff, 2^-8 the bf16 one (8 significant bits).
"""
import math

import pytest
import torch

from exact_helpers import (Guarded, _ce_dlse, _dense_poisoned, _expect_close, _expect_equal, _gelu64, _gelu_grad64,
                           _gelu_grad_tol, _gelu_tol, _poisoned, _silu_tol, _ulp_bf16)

pytestmark = pytest.mark.gpu
bf16, f32, f64, i64 = torch.bfloat16, torch.float32, torch.float64, torch.int64
U = 2.0 ** -24
GRID_Y = 65535                                   # largest grid.y / grid.z extent


@pytest.fixture(scope="module")
def ops(cuda_dev):
    from dalm_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def Err(cuda_dev):
    from dalm_b200._lib import DalmB200Error
    return DalmB200Error


@pytest.fixture(autouse=True)
def _free(cuda_dev):
    """the buffers here are large: give them back to the allocator between tests"""
    yield
    torch.cuda.empty_cache()


def _rows(view, rows):
    return view[[r for r in rows if 0 <= r < view.shape[0]]]


# ----------------------------------------------------------------------------------------------------------------
# A. counts past 65535 on grid.y: SwiGLU / GeGLU (one CTA row per token row, chunks of 65535 rows), GELU (4 rows per CTA
# row, chunks of 262140 rows), top-k (8 queries per CTA row, chunks of 16384 queries)
# ----------------------------------------------------------------------------------------------------------------
GLU_M = (GRID_Y, GRID_Y + 1, 2 * GRID_Y + 5)
GLU_SEAMS = (0, GRID_Y - 1, GRID_Y, GRID_Y + 1, 2 * GRID_Y - 1, 2 * GRID_Y, 2 * GRID_Y + 1)   # rows around the chunk bases


def _glu_cols(F, il, dev):
    if il:
        gcols = (torch.arange(F, device=dev) // il) * 2 * il + torch.arange(F, device=dev) % il
        return gcols, gcols + il
    return torch.arange(F, device=dev), torch.arange(F, device=dev) + F


@pytest.mark.parametrize("M", GLU_M)
@pytest.mark.parametrize("act,F,il", [("swiglu", 24, 0), ("swiglu", 128, 128), ("geglu", 24, 0)])
def test_glu_rows_past_grid_y(ops, cuda_dev, act, F, il, M):
    """SwiGLU fwd / bwd (both gate|up layouts) and GeGLU fwd / bwd on M token rows; bounds as in the row-wise tests: one bf16
    rounding of the output plus the activation's fp32 error"""
    dev = cuda_dev
    gen = torch.Generator(device=dev).manual_seed(M + F + il)
    gu = (torch.randn(M, 2 * F, generator=gen, device=dev) * 2).to(bf16)
    dact = torch.randn(M, F, generator=gen, device=dev).to(bf16)
    gcols, ucols = _glu_cols(F, il, dev)
    g, u, d = gu.double()[:, gcols], gu.double()[:, ucols], dact.double()
    what = f"{act} M {M} F {F} interleave {il}"
    out = Guarded(M, F, bf16, dev)
    work = Guarded(M, 2 * F, bf16, dev, init=gu)
    if act == "swiglu":
        ops.swiglu_fwd(_poisoned(gu), F, act=out.view, interleave=il)
        ops.swiglu_bwd_(work.view, _poisoned(dact), F, interleave=il)
        sg = torch.sigmoid(g)
        ref = g * sg * u
        tol = _ulp_bf16(ref) + _silu_tol(g) * ref.abs()
        dg = d * u * sg * (1 + g * (1 - sg))
        du = d * g * sg
        tol_dg = _ulp_bf16(dg) + _silu_tol(g) * (d * u * sg).abs() * (1 + g.abs()) * 4
        tol_du = _ulp_bf16(du) + _silu_tol(g) * du.abs()
    else:
        ops.geglu_fwd(_poisoned(gu), F, act=out.view)
        ops.geglu_bwd_(work.view, _poisoned(dact), F)
        ref = _gelu64(g) * u
        tol = _ulp_bf16(ref) + _gelu_tol(g) * u.abs() + U * ref.abs()              # gelu_erf, then one fp32 product
        dg = d * u * _gelu_grad64(g)
        du = d * _gelu64(g)
        tol_dg = _ulp_bf16(dg) + (d * u).abs() * _gelu_grad_tol(g) + 2 * U * dg.abs()
        tol_du = _ulp_bf16(du) + d.abs() * _gelu_tol(g) + U * du.abs()
    out.check(what + " fwd")
    work.check(what + " bwd")
    for name, got, want, t in (("fwd", out.view, ref, tol), ("dgate", work.view[:, gcols], dg, tol_dg),
                               ("dup", work.view[:, ucols], du, tol_du)):
        _expect_close(_rows(got, GLU_SEAMS), _rows(want, GLU_SEAMS), _rows(t, GLU_SEAMS), f"{what} {name} at the chunk seams")
        _expect_close(got, want, t, f"{what} {name}")


GELU_M = (4 * GRID_Y, 4 * GRID_Y + 1, 4 * GRID_Y + 3)           # M % 4 = 0, 1, 3 around the 262140-row chunk


@pytest.mark.parametrize("M", GELU_M)
def test_gelu_rows_past_grid_y(ops, cuda_dev, M):
    dev, F = cuda_dev, 8
    gen = torch.Generator(device=dev).manual_seed(M)
    pre = (torch.randn(M, F, generator=gen, device=dev) * 2).to(bf16)
    d = torch.randn(M, F, generator=gen, device=dev).to(bf16)
    act = Guarded(M, F, bf16, dev)
    ops.gelu_fwd(_poisoned(pre), act=act.view)
    work = Guarded(M, F, bf16, dev, init=d)
    ops.gelu_bwd_(_poisoned(pre), work.view)
    what = f"gelu M {M}"
    act.check(what + " fwd")
    work.check(what + " bwd")
    x = pre.double()
    ref = _gelu64(x)
    seams = (4 * GRID_Y - 1, 4 * GRID_Y, 4 * GRID_Y + 1, 4 * GRID_Y + 2)
    _expect_close(_rows(act.view, seams), _rows(ref, seams), _rows(_ulp_bf16(ref) + _gelu_tol(x), seams), what + " fwd at the seam")
    _expect_close(act.view, ref, _ulp_bf16(ref) + _gelu_tol(x), what + " fwd")
    dref = d.double() * _gelu_grad64(x)
    _expect_close(work.view, dref, _ulp_bf16(dref) + d.double().abs() * _gelu_grad_tol(x), what + " bwd")


TOPK_NQ = (8 * GRID_Y, 8 * GRID_Y + 1, 8 * GRID_Y + 17)         # 65535, 65536 and 65538 query tiles of 8


@pytest.mark.parametrize("nq", TOPK_NQ)
@pytest.mark.parametrize("D", [64, 128])                         # D 64: register kernel, D 128: pipelined kernel
def test_topk_queries_past_grid_y(ops, cuda_dev, D, nq):
    """integer Q / P in [-2, 2]: every score is exact, so scores and indices are bit-equal to the fp64 order (higher score
    first, lower index on ties; with 300 passages most rows tie) and to the nq = 8 result of the same rows"""
    dev, N, K = cuda_dev, 300, 3
    g = torch.Generator(device=dev).manual_seed(nq + D)
    Q = torch.randint(-2, 3, (nq, D), generator=g, device=dev).float()
    P = torch.randint(-2, 3, (N, D), generator=g, device=dev).float()
    P[7] = P[250]                                                    # an exact tie for every query
    scores, idx = ops.topk_ip(_dense_poisoned(Q), _poisoned(P), K)
    what = f"topk D {D} N {N} nq {nq} K {K}"
    step = 65536
    for r0 in range(0, nq, step):
        ref = Q[r0:r0 + step].double() @ P.double().t()
        vals, order = torch.sort(ref, dim=1, descending=True, stable=True)
        _expect_equal(idx[r0:r0 + step], order[:, :K], f"{what} indices, rows from {r0}")
        _expect_equal(scores[r0:r0 + step], vals[:, :K], f"{what} scores, rows from {r0}")
    for r0 in (0, 16384 - 8, 16384, 8 * GRID_Y - 8, nq - 8):          # first rows, the first query chunk seam, the last tiles
        s8, i8 = ops.topk_ip(Q[r0:r0 + 8].contiguous(), P, K)
        assert torch.equal(i8, idx[r0:r0 + 8]) and torch.equal(s8.view(torch.int32), scores[r0:r0 + 8].view(torch.int32)), \
            f"{what}: rows {r0}..{r0 + 7} differ from their nq = 8 result"


# ----------------------------------------------------------------------------------------------------------------
# A. counts that are refused by name: B sequences / samples on grid.y or grid.z
# ----------------------------------------------------------------------------------------------------------------
def _attn_call(ops, kind, bwd):
    fwd_f, bwd_f = (ops.attention_tc_fwd, ops.attention_tc_bwd) if kind == "wg" else (ops.attention_fwd, ops.attention_bwd)
    dev, B, L, D = "cuda", GRID_Y + 1, 2, 64
    q = torch.zeros(B * L, D, dtype=bf16, device=dev)
    mask = torch.ones(B, L, dtype=i64, device=dev)
    if not bwd:
        return lambda: fwd_f(q, q, q, mask, B, L, 1, 1, D, True)
    lse = torch.zeros(B, 1, L, dtype=f32, device=dev)
    return lambda: bwd_f(q, q, q, mask, q, lse, q, B, L, 1, 1, D, True)


@pytest.mark.parametrize("kind", ["mma", "wg"])
@pytest.mark.parametrize("bwd", [False, True])
def test_attention_refuses_batches_past_grid_z(ops, Err, kind, bwd):
    with pytest.raises(Err, match="65535"):
        _attn_call(ops, kind, bwd)()
    torch.cuda.synchronize()


@pytest.mark.parametrize("H", [128, 100])                        # pool_sum path / one-CTA-per-sample path
def test_pool_norm_refuses_batches_past_grid_y(ops, Err, cuda_dev, H):
    B = GRID_Y + 1
    with pytest.raises(Err, match="65535"):
        ops.pool_norm_fwd(torch.zeros(B, 2, H, device=cuda_dev), torch.ones(B, 2, dtype=i64, device=cuda_dev))
    # the largest accepted batch: every sample's mean is 1, its normalised embedding 1 / sqrt(H) within a few fp32 roundings
    emb, _ = ops.pool_norm_fwd(torch.ones(GRID_Y, 2, H, device=cuda_dev), torch.ones(GRID_Y, 2, dtype=i64, device=cuda_dev))
    err = (emb.double() - 1 / math.sqrt(H)).abs()
    assert err.max() <= 4 * U, f"pool_norm_fwd at B = 65535: sample {int(err.amax(1).argmax())} off by {err.max().item():.3e}"


def test_embed_and_dequant_refuse_rows_past_grid_y(ops, Err, cuda_dev):
    dev, B = cuda_dev, GRID_Y + 1
    word = torch.zeros(16, 8, dtype=bf16, device=dev)
    with pytest.raises(Err, match="65535"):
        ops.roberta_embed(torch.full((B, 1), 2, dtype=i64, device=dev), word, word, word[:1], 1)
    packed = torch.zeros(B * 64 // 2, dtype=torch.uint8, device=dev)
    with pytest.raises(Err, match="65535"):
        ops.nf4_dequant_(packed, torch.ones(B, device=dev), B, 64, torch.zeros(B, 64, dtype=bf16, device=dev))
    M = 16 * GRID_Y + 1                                              # lora_dx: 16 rows per CTA row
    with pytest.raises(Err, match="65535"):
        ops.lora_dx_(torch.zeros(M, 8, dtype=bf16, device=dev), torch.zeros(M, 8, dtype=bf16, device=dev),
                     torch.zeros(8, 8, dtype=bf16, device=dev), 8, 8, ops.Drop(0.0, 0, 0))
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------
# B. one logits buffer past 2^31 elements: the unchunked lm_head at the Llama 3 vocabulary
# ----------------------------------------------------------------------------------------------------------------
def test_logits_past_2_31_elements(ops, cuda_dev):
    """GEMM [16768, 64] x [128256, 64]^T into a guarded bf16 buffer: integer operands in [-2, 2], every product sum an integer
    of magnitude <= 256, so the bf16 output is the exact product. Then the cross-entropy pass on those logits in place, and
    ce_marginal_rows_ on a chunk whose first row lies past element 2^31 of the buffer, against fp64 with the loss bounds."""
    dev, B, L, V, K = cuda_dev, 2, 8384, 128256, 64
    M = B * L
    g = torch.Generator(device=dev).manual_seed(31)
    a = torch.randint(-2, 3, (M, K), generator=g, device=dev).to(bf16)
    w = torch.randint(-2, 3, (V, K), generator=g, device=dev).to(bf16)
    w[V - 1] = 2 * torch.sign(a[M - 2].float()).to(bf16)             # row M - 2's label logit is its row maximum
    out = Guarded(M, V, bf16, dev)
    ld = out.view.stride(0)
    assert M * ld > 2 ** 31
    ops.gemm(_poisoned(a), _poisoned(w), out=out.view)
    out.check("gemm [16768, 128256]")
    ids = torch.randint(0, V, (B, L), generator=g, device=dev)
    ids[1, L - 1] = V - 1
    mask = torch.ones(B, L, dtype=i64, device=dev)
    mask[1, 5] = 0
    nsum = mask[:, 1:].sum().float().view(1)
    t = torch.arange(M, device=dev) % L
    nxt = (torch.arange(M, device=dev) + 1).clamp_max(M - 1)
    valid = t < L - 1
    wt = torch.where(valid, mask.view(-1)[nxt], torch.zeros_like(t)).double()
    label = torch.where(valid, ids.view(-1)[nxt], torch.zeros_like(t))
    a64, w64 = a.double(), w.double()
    lse, mx, span, xl = (torch.empty(M, 1, dtype=f64, device=dev) for _ in range(4))
    step = 512
    for r0 in range(0, M, step):
        x = a64[r0:r0 + step] @ w64.t()
        _expect_equal(out.view[r0:r0 + step], x, f"gemm rows from {r0}")
        lse[r0:r0 + step] = torch.logsumexp(x, 1, keepdim=True)
        mx[r0:r0 + step] = x.amax(1, keepdim=True)
        span[r0:r0 + step] = mx[r0:r0 + step] - x.amin(1, keepdim=True)
        xl[r0:r0 + step] = x.gather(1, label[r0:r0 + step, None])
    del x
    dlse = _ce_dlse(V, lse, mx, span)
    boundary = {2 ** 31 // V, 2 ** 31 // ld}                         # first row past element 2^31 at the dense / guarded stride
    check_rows = sorted({0, 1, M - 2, M - 1} | {r + d for r in boundary for d in (-1, 0, 1)})

    def expect_ce(tok_lp, rows_got, rows, what):
        lp = ((xl - lse)[:, 0] * (wt > 0)).view(1, -1)
        tol = ((dlse[:, 0] + U * lp.abs()) * (wt > 0)).view(1, -1)
        _expect_close(tok_lp.reshape(1, -1), lp, tol, what + " tok_lp")
        rs = torch.tensor(rows, device=dev)
        x = a64[rs] @ w64.t()
        prob = torch.exp(x - lse[rs])
        onehot = torch.zeros_like(prob).scatter_(1, label[rs, None], 1.0)
        coef = (wt[rs] / nsum.double())[:, None]
        ref = coef * (prob - onehot)
        tol = _ulp_bf16(ref) + coef.abs() * (prob * (dlse[rs] + 2.0 ** -23 * (3 + 1.2 * (x - lse[rs]).abs())) +
                                             4 * U * (prob - onehot).abs())
        _expect_close(rows_got, ref, tol, f"{what} dlogits rows {rows}")

    logits = torch.as_strided(out.view, (B, L, V), (L * ld, ld, 1))
    tok_lp, dl = ops.ce_marginal(logits, ids, mask, nsum, need_grad=True, inplace=True)
    assert dl.data_ptr() == out.view.data_ptr()
    out.check("ce_marginal in place")
    expect_ce(tok_lp, out.view[check_rows], check_rows, "ce_marginal")
    # the rows from r0 on again, as one chunk of the chunked head: row0 * V and row0 * ld both pass 2^31
    r0 = 2 ** 31 // V + 1
    ops.gemm(a[r0:], w, out=out.view[r0:])
    tok_lp2 = torch.zeros(B, L, dtype=f32, device=dev)
    tok_lp2.view(-1)[:r0] = tok_lp.view(-1)[:r0]
    ops.ce_marginal_rows_(out.view[r0:], ids, mask, nsum, tok_lp2, r0, V)
    out.check("ce_marginal_rows_")
    rows = [r0, r0 + 1, r0 + 2, M - 2, M - 1]
    expect_ce(tok_lp2, out.view[rows], rows, f"ce_marginal_rows_ row0 {r0}")


# ----------------------------------------------------------------------------------------------------------------
# C. attention at 8192 tokens
# ----------------------------------------------------------------------------------------------------------------
# (name, D, Hq, Hkv, B, causal, window, bidirectional, padding): padding "left3000" gives sample 1 3000 left pad tokens,
# "rl100" gives sample 0 100 right and sample 1 100 left pad tokens, "r100" sample 0 100 right pad tokens
ATTN_8K = [
    ("qwen2_group7", 128, 7, 1, 1, True, 0, False, None),
    ("mistral_window4096", 128, 4, 1, 2, True, 4096, False, "left3000"),
    ("modernbert_local65", 64, 2, 2, 2, False, 65, True, "rl100"),
    ("modernbert_global", 64, 2, 2, 1, False, 0, False, "r100"),
]
L8K = 8192


def _vis(mask_b, L, causal, window, bidirectional, dev):
    """[L, L] bool: query i sees key j"""
    i = torch.arange(L, device=dev)[:, None]
    j = torch.arange(L, device=dev)[None, :]
    vis = mask_b.bool()[None, :].expand(L, L)
    if causal:
        vis = vis & (j <= i)
        if window:
            vis = vis & (i - j < window)
    elif window:
        vis = vis & ((i - j).abs() < window)
    return vis


def _drop_last_tile(vis):
    """the visibility with the last visible 64-key tile of every query removed"""
    j = torch.arange(vis.shape[1], device=vis.device)
    last = torch.where(vis, j[None, :], -1).amax(1, keepdim=True)
    return vis & ~((j[None, :] // 64 == last // 64) & (last >= 0))


@pytest.mark.parametrize("name,D,Hq,Hkv,B,causal,window,bidir,pad", ATTN_8K, ids=[c[0] for c in ATTN_8K])
def test_attention_8k_vs_fp64(ops, cuda_dev, name, D, Hq, Hkv, B, causal, window, bidir, pad):
    """Forward and backward of every kernel built for the case (mma.sync at D 64 / 128, wgmma at D 64 / 128), every row.

    Arithmetic of the kernels and the bound it gives (fp64 values: s scores, p probabilities, per query row i, key j):
    - s in fp32 from bf16 q, k (exact products, fp32 tensor-core sums of D terms): |ds| <= e_s_i = 2 (D + 8) U scale
      |q_i| max_j |k_j| (Cauchy-Schwarz on sum |q_id k_jd|; 2 U per add covers the tensor core's accumulation).
    - p = exp2 of a rounded argument (|s - m| < 64: 2^-16 relative covers the argument rounding and ex2.approx); in the
      backward p is recomputed from s and the forward's lse, whose error is measured: eps_i = e_s_i + |dlse_i| + 2^-16.
    - out = sum_j bf16(p_ij) v_j / l_i, l_i summed from the fp32 p: the bf16 rounding of P costs 2^-8 per term, plus the fp32
      chains over the key (and, in the backward, G query heads') tiles and the online softmax's 128 rescales by __expf
      (g = (G L / 64 + 64) U + (L / 64) 2^-21): |dout_id| <= (2^-8 + 2 e_s_i + 2^-15 + g) sum_j p_ij |v_jd| + 1 ulp.
    - lse = m + log l: |dlse_i| <= e_s_i + g + 2^-20 + U |lse_i|.
    - dv_jd = sum_i bf16(p_ij) do_id: |ddv_jd| <= sum_i (2^-8 + eps_i + g) p_ij |do_id| + 1 ulp.
    - ds_ij = p_ij (dp_ij - delta_i) scale, rounded to bf16; dp from bf16 do, v (|ddp_ij| <= 2 (D + 8) U |do_i| |v_j|),
      delta_i = sum_d do_id o_id over the kernel's own o (|ddelta_i| <= 2 (D + 8) U sum_d |do_id o_id|):
      |dds_ij| <= scale A_ij, A_ij = p_ij |dp_ij - delta_i| (eps_i + 2^-8 + 3 U + g) + p_ij (|ddp_ij| + |ddelta_i|), and
      |ddq_id| <= scale sum_j A_ij |k_jd| + 1 ulp, |ddk_jd| <= scale sum_i A_ij |q_id| + 1 ulp.
    Rows no visible pair reaches (a query without a visible key, a masked key) get a bound of 0 + ulp(0): exact zeros."""
    dev, L = cuda_dev, L8K
    G = Hq // Hkv
    scale = 1.0 / math.sqrt(D)
    gen = torch.Generator(device=dev).manual_seed(D * 1000 + Hq * 10 + B)
    # q twice as wide as k: scores of standard deviation 2, so a few keys carry a visible share of each row's weight and a
    # one-tile error stays visible next to the 2^-8 bound at 8192 keys
    q0 = (torch.randn(B * L, Hq * D, generator=gen, device=dev) * 2).to(bf16)
    k0 = torch.randn(B * L, Hkv * D, generator=gen, device=dev).to(bf16)
    v0 = torch.randn(B * L, Hkv * D, generator=gen, device=dev).to(bf16)
    do0 = torch.randn(B * L, Hq * D, generator=gen, device=dev).to(bf16)
    mask = torch.ones(B, L, dtype=i64, device=dev)
    if pad == "left3000":
        mask[1, :3000] = 0
    elif pad == "rl100":
        mask[0, L - 100:] = 0
        mask[1, :100] = 0
    elif pad == "r100":
        mask[0, L - 100:] = 0
    q, k, v, d_out = (_poisoned(t) for t in (q0, k0, v0, do0))
    kinds = ["mma", "wg"]
    res = {}
    for kind in kinds:
        fwd, bwd = (ops.attention_tc_fwd, ops.attention_tc_bwd) if kind == "wg" else (ops.attention_fwd, ops.attention_bwd)
        out = Guarded(B * L, Hq * D, bf16, dev)
        _, lse = fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out.view, scale=scale, window=window, bidirectional=bidir)
        dq, dk, dv = Guarded(B * L, Hq * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev)
        bwd(q, k, v, mask, out.view, lse, d_out, B, L, Hq, Hkv, D, causal, dq=dq.view, dk=dk.view, dv=dv.view, scale=scale,
            window=window, bidirectional=bidir)
        for nm, gd in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
            gd.check(f"{kind} {name} {nm}")
        res[kind] = (out.view, lse, dq.view, dk.view, dv.view)
    g_acc = (G * L / 64 + 64) * U + L / 64 * 2.0 ** -21            # fp32 chains over G * 128 query / key tiles, 128 rescales
    gam_d = 2 * (D + 8) * U
    for b in range(B):
        vis = _vis(mask[b], L, causal, window, bidir, dev)
        has = vis.any(1)
        nvis = vis.sum(1)
        ctl_vis = _drop_last_tile(vis)
        long_rows = nvis >= nvis.max() // 2
        rows = slice(b * L, (b + 1) * L)
        for hk in range(Hkv):
            kh, vh = k0[rows, hk * D:(hk + 1) * D].double(), v0[rows, hk * D:(hk + 1) * D].double()
            kn, vn = kh.norm(dim=1), vh.norm(dim=1)
            dk_ref = torch.zeros(L, D, dtype=f64, device=dev)
            dv_ref = torch.zeros_like(dk_ref)
            dk_tol = {kd: torch.zeros_like(dk_ref) for kd in kinds}
            dv_tol = {kd: torch.zeros_like(dk_ref) for kd in kinds}
            for hq in range(hk * G, (hk + 1) * G):
                cols = slice(hq * D, (hq + 1) * D)
                qh, doh = q0[rows, cols].double(), do0[rows, cols].double()
                e_s = gam_d * scale * qh.norm(dim=1) * kn.max()                           # [L]
                s = (qh @ kh.t() * scale).masked_fill_(~vis, float("-inf"))
                lse_ref = torch.logsumexp(s, 1)                                          # -inf without a visible key
                p = torch.exp(s - torch.where(has, lse_ref, torch.zeros_like(lse_ref))[:, None])
                del s
                o_ref = p @ vh
                pv = p @ vh.abs()
                what = f"{name} sample {b} head {hq}"
                # control: the last visible key tile of every query dropped must break the forward bound on a long row
                pc = p * ctl_vis
                lc = pc.sum(1, keepdim=True)
                o_ctl = (pc / torch.where(lc > 0, lc, torch.ones_like(lc))) @ vh
                del pc
                tol_fwd = (2.0 ** -8 + 2 * e_s[:, None] + 2.0 ** -15 + g_acc) * pv
                miss = ((o_ctl - o_ref).abs() > tol_fwd + _ulp_bf16(o_ref)).any(1) & long_rows
                assert miss.any(), f"{what}: control (last visible key tile dropped) stays within the bound on every long row"
                dp = doh @ vh.t()
                for kind in kinds:
                    out, lse, dq, dk, dv = res[kind]
                    kw = f"{kind} {what}"
                    got_o = out[rows, cols]
                    _expect_close(got_o, o_ref, tol_fwd + _ulp_bf16(o_ref), kw + " out", 64)
                    lk = lse[b, hq].double()
                    assert (torch.isinf(lk[~has]) & (lk[~has] > 0)).all(), f"{kw}: rows without a visible key need lse = +inf"
                    lse_tol = e_s + g_acc + 2.0 ** -20 + U * lse_ref.abs()
                    _expect_close(lk[has].view(1, -1), lse_ref[has].view(1, -1), lse_tol[has].view(1, -1), kw + " lse")
                    dlse = torch.where(has, (lk - lse_ref).abs(), torch.zeros_like(lk))
                    eps = e_s + dlse + 2.0 ** -16
                    oh = got_o.double()
                    delta = (doh * oh).sum(1, keepdim=True)
                    d_delta = gam_d * (doh * oh).abs().sum(1, keepdim=True)
                    dpd = dp - delta
                    ds = p * dpd * scale
                    A = p * (dpd.abs() * (eps[:, None] + 2.0 ** -8 + 3 * U + g_acc) + gam_d * doh.norm(dim=1)[:, None] * vn[None, :]
                             + d_delta)
                    dq_ref = ds @ kh
                    _expect_close(dq[rows, cols], dq_ref, scale * (A @ kh.abs()) + _ulp_bf16(dq_ref), kw + " dq", 64)
                    dk_tol[kind] += scale * (A.t() @ qh.abs())
                    dv_tol[kind] += ((2.0 ** -8 + eps[:, None] + g_acc) * p).t() @ doh.abs()
                    if kind == kinds[0]:
                        dk_ref += ds.t() @ qh
                        dv_ref += p.t() @ doh
                    del A, ds, dpd
                del p, dp
            for kind in kinds:
                _, _, _, dk, dv = res[kind]
                kw = f"{kind} {name} sample {b} kv head {hk}"
                kc = slice(hk * D, (hk + 1) * D)
                _expect_close(dk[rows, kc], dk_ref, dk_tol[kind] + _ulp_bf16(dk_ref), kw + " dk", 64)
                _expect_close(dv[rows, kc], dv_ref, dv_tol[kind] + _ulp_bf16(dv_ref), kw + " dv", 64)
    print(f"[8k] {name}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
