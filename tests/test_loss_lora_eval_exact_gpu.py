"""Element-wise checks of the loss, pooling, LoRA, top-k and decode-step kernels at the shapes, strides and alignments that
pick their code paths, and of the wrapper checks in front of them.

Every strided input is a view into a NaN-padded buffer and every output the wrappers let the caller place is an interior
view with sentinel guard bands (exact_helpers). Integer inputs make the result exact: the LoRA operands (skinny_gemm,
lora_wgrad: integers in [-2, 2], so every fp32 partial sum and atomic add is an integer below 2^24 and the check is bit
equality after the one bf16 rounding), the top-k operands (integer scores: the indices must equal a stable fp64 sort),
marginal_counts (integer counts) and the greedy step (an argmax and integer bookkeeping). Everything else is compared
with fp64 element by element, within a bound derived from the kernel's arithmetic and written next to the check.
U = 2^-24 is the fp32 unit roundoff, gamma_n = n U / (1 - n U) bounds an n-term fp32 sum or dot product relative to the sum
of the magnitudes of its terms. __expf is within 2 + floor(1.173 |x|) ulp of exp(x) (one ulp <= 2^-23 of the result) and
__logf within 2^-21.41 absolute on [0.5, 2], 3 ulp elsewhere (CUDA programming guide, intrinsic functions); where the
kernels apply them to a difference computed in fp32, that difference carries one more rounding, U |x|.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from exact_helpers import GUARD_C, Guarded, Guarded1d, _dense_poisoned, _expect_close, _expect_equal, _ints, _poisoned, _ulp_bf16

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
EXP_ULP = 2.0 ** -23                              # one ulp of an fp32 result, relative, at most
LOGF_ABS = 2.0 ** -21.41
EPS9, EPS12 = float(torch.tensor(1e-9, dtype=f32)), float(torch.tensor(1e-12, dtype=f32))   # the kernels' fp32 clamps


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


def _gamma(n):
    return n * U / (1 - n * U)


def _expf_rel(x):
    """relative error of __expf of an fp32 difference x (x itself one rounding from exact)"""
    return (2 + 1.173 * x.abs()) * EXP_ULP + U * x.abs()


def _logf_abs(s):
    return torch.where((s >= 0.5) & (s <= 2), torch.full_like(s, LOGF_ABS), 3 * EXP_ULP * torch.log(s).abs())


def _lse(S, dim, depth):
    """fp64 log-sum-exp of the kernel's fp32 scores along `dim`, and the bound on the kernel's mx + __logf(sum __expf(s - mx))
    whose sum is a chain of at most `depth` fp32 additions"""
    m = S.amax(dim, keepdim=True)
    x = S - m
    e = torch.exp(x)
    s = e.sum(dim, keepdim=True)
    ds = (e * _expf_rel(x)).sum(dim, keepdim=True) + depth * U * s
    lse = m + torch.log(s)
    return lse, ds / s + _logf_abs(s) + U * lse.abs()


# ----------------------------------------------------------------------------------------------------------------
# marginal counts
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [2, 37])
@pytest.mark.parametrize("pad", ["left", "right"])
def test_marginal_counts(ops, cuda_dev, L, pad):
    """integer counts: bit-equal to the oracle, with qlen 1, L - 1, L, L + 3, 0 and a negative one (python slice wrap)"""
    from oracle import losses
    g = torch.Generator().manual_seed(L)
    qlen = torch.tensor([1, L - 1, L, L + 3, 0, -3], dtype=torch.int64)
    B = qlen.numel()
    mask = torch.ones(B, L, dtype=torch.int64)
    for b in range(B):
        n = int(torch.randint(0, L, (1,), generator=g)) if b else L - 1
        if pad == "right":
            mask[b, L - n:] = 0
        else:
            mask[b, :n] = 0
    cvec, nsum = ops.marginal_counts(mask.to(cuda_dev), qlen.to(cuda_dev))
    c_ref, n_ref = losses.marginal_counts(mask, qlen)
    what = f"marginal_counts L {L} {pad}"
    _expect_equal(_v(cvec.cpu()), _v(c_ref), what + " cvec")
    _expect_equal(_v(nsum.cpu()), _v(n_ref), what + " nsum")


# ----------------------------------------------------------------------------------------------------------------
# fused in-batch similarity + contrastive loss + marginal coupling
# ----------------------------------------------------------------------------------------------------------------
INBATCH = [(1, 64), (7, 1030), (18, 1024), (150, 1024), (36, 4096)]   # 1030: scalar P loads; 150 > SMs: CTAs loop over rows
VARIANTS = [(True, True, 0.75), (False, True, 1.0), (True, False, 1.0)]   # (cvec / nsum, need_grad, grad_out)
SCALE = 100.0


def _inbatch_inputs(B, D, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    q = F.normalize(torch.randn(B, D, generator=g, device=dev), dim=1)
    p = F.normalize(torch.randn(B, D, generator=g, device=dev) + 0.5 * q, dim=1)
    c = torch.randint(0, 60, (B,), generator=g, device=dev).float()
    return q, p, c


def _check_inbatch(r, q, p, c, N, need_grad, gout, what):
    B, D = q.shape
    q64, p64 = q.double(), p.double()
    ref = SCALE * q64 @ p64.t()
    # B x B dot products of D fp32 FMAs (lane chains + the warp tree), then one rounding for * scale
    _expect_close(r["S"], ref, SCALE * _gamma(D) * (q64.abs() @ p64.abs().t()) + U * ref.abs(), what + " S")
    S = r["S"].double()                              # everything downstream starts from the kernel's scores
    rl, drl = _lse(S, 1, B + 5)                      # rows: B / 32 per lane + the warp tree; columns: B per thread
    cl, dcl = _lse(S, 0, B + 5)
    d = S.diagonal() - rl[:, 0]
    dd = drl[:, 0] + U * d.abs()                     # s_ii - lse: one rounding
    _expect_close(_v(r["dlp"]), _v(d), _v(dd), what + " dlp")
    e = S.diagonal() - cl[0]
    de = dcl[0] + U * e.abs()
    terms = d + e
    lc = -(terms.sum() * 0.5 / B).item()
    # B terms (one rounding each) summed per thread and over the block (<= B + 10 additions), * 0.5 / B (two roundings)
    tol_lc = 0.5 / B * ((dd + de + U * terms.abs()).sum() + (B + 10) * U * terms.abs().sum()).item() + 2 * U * abs(lc)
    if c is not None:
        c64 = c.double()
        doc = -((c64 * d).sum() / N).item()
        # integer weights times dlp (one rounding), the block sum, * (1 / N) (two roundings)
        tol_doc = (((c64 * dd).sum() + (B + 12) * U * (c64 * d).abs().sum()) / N).item() + 2 * U * abs(doc)
    else:
        doc, tol_doc = 0.0, 0.0
    want = torch.tensor([lc, doc, lc + doc, N if c is not None else 0.0], dtype=f64)
    tol = torch.tensor([tol_lc, tol_doc, tol_lc + tol_doc + U * abs(lc + doc), 0.0], dtype=f64)
    _expect_close(_v(r["losses"].cpu()), _v(want), _v(tol), what + " losses {Lc, doc, Lc + doc, N}")
    if not need_grad:
        assert r["dQ"] is None and r["dP"] is None, what
        return
    eye = torch.eye(B, dtype=f64, device=S.device)
    xr, xc = S - rl, S - cl
    pr, pc = torch.exp(xr), torch.exp(xc)
    epr = pr * (drl + _expf_rel(xr))                 # the lse's error moves the __expf argument
    epc = pc * (dcl + _expf_rel(xc))
    a = 0.5 / B
    cw = (c.double() / N)[:, None] if c is not None else 0.0
    G = a * ((pr - eye) + (pc - eye)) + cw * (pr - eye)
    mag = a * ((pr - eye).abs() + (pc - eye).abs()) + cw * (pr - eye).abs()
    k = gout * SCALE
    dS = k * G
    # <= 8 roundings forming g (the subtractions, 0.5 / B, c / N and their products / sums), then * gout and * scale
    ddS = abs(k) * (a * (epr + epc) + cw * epr + 10 * U * mag)
    # dQ = dS P and dP = dS^T Q: chains of B fp32 FMAs per element
    _expect_close(r["dQ"], dS @ p64, ddS @ p64.abs() + _gamma(B + 1) * (dS.abs() @ p64.abs()), what + " dQ")
    _expect_close(r["dP"], dS.t() @ q64, ddS.t() @ q64.abs() + _gamma(B + 1) * (dS.abs().t() @ q64.abs()), what + " dP")


@pytest.mark.parametrize("B,D", INBATCH)
@pytest.mark.parametrize("marg,need_grad,gout", VARIANTS)
def test_inbatch_loss(ops, cuda_dev, B, D, marg, need_grad, gout):
    q, p, c = _inbatch_inputs(B, D, cuda_dev, B * 131 + D)
    N = 700.0
    cvec = _poisoned(c) if marg else None
    nsum = _poisoned(torch.tensor([N], device=cuda_dev)) if marg else None
    r = ops.inbatch_loss(_dense_poisoned(q), _dense_poisoned(p), SCALE, cvec, nsum, need_grad=need_grad, grad_out=gout)
    _check_inbatch(r, q, p, c if marg else None, N, need_grad, gout, f"inbatch B {B} D {D} marg {marg} grad {need_grad}")


@pytest.mark.parametrize("B,D", [(18, 1024), (36, 4096)])
def test_inbatch_loss_misaligned(ops, cuda_dev, B, D):
    """contiguous Q / P views that start 4 bytes past a 16-byte boundary: P's float4 loads must give way to scalar ones"""
    q, p, c = _inbatch_inputs(B, D, cuda_dev, B + D)
    views = []
    for t in (q, p):
        buf = torch.full((B * D + 64,), float("nan"), device=cuda_dev)
        v = buf[1:1 + B * D].view(B, D)
        v.copy_(t)
        views.append(v)
    nsum = torch.tensor([700.0], device=cuda_dev)
    r = ops.inbatch_loss(views[0], views[1], SCALE, c, nsum, grad_out=1.0)
    _check_inbatch(r, q, p, c, 700.0, True, 1.0, f"inbatch misaligned B {B} D {D}")


# ----------------------------------------------------------------------------------------------------------------
# vocabulary cross-entropy rows: the fp32 and scalar paths (the bf16 large-vocabulary rows: test_rowwise_exact_gpu)
# ----------------------------------------------------------------------------------------------------------------
CE_B, CE_L = 3, 5
CE_CASES = [
    # (dtype, V, row stride, mode): "out" / "inplace" through ce_marginal, "rows" through ce_marginal_rows_ from row 3
    (f32, 32000, 32000, "out"), (f32, 32000, 32064, "inplace"),          # fp32 rows cached in shared memory (125 KB)
    (f32, 65024, 65024, "inplace"), (f32, 65024, 65088, "out"),          # above the 200 KB cache: read from global
    (f32, 1001, 1005, "out"), (f32, 1001, 1005, "inplace"),              # scalar path: V % 4 != 0
    (bf16, 1001, 1005, "out"), (bf16, 1001, 1005, "inplace"),            # bf16 scalar path
    (bf16, 32000, 32000, "rows"), (f32, 65024, 65024, "rows"), (f32, 1001, 1005, "rows"),
]


def _ce_run(ops, dev, dtype, V, ld, mode, shift=0):
    B, L = CE_B, CE_L
    g = torch.Generator(device=dev).manual_seed(V + ld + len(mode) + shift)
    x = (torch.randn(B * L, V, generator=g, device=dev) * 3).to(dtype)
    base = torch.full((B * L, ld), float("nan"), dtype=dtype, device=dev)
    base[:, shift:shift + V] = x
    ids = torch.randint(0, V, (B, L), generator=g, device=dev)
    ids[0, 1], ids[1, 2] = V - 1, 0
    mask = torch.ones(B, L, dtype=torch.int64, device=dev)
    mask[1, 1] = 0                                                      # masked tokens: the rows before them get no gradient
    mask[2, 3] = 0
    nsum = mask[:, 1:].sum().float().view(1)
    what = f"ce {str(dtype)[6:]} V {V} ld {ld} {mode} shift {shift}"
    itype = torch.int16 if dtype == bf16 else torch.int32
    if mode == "rows":
        r0, n = 3, 9                                                    # starts mid-sequence, spans three sequences
        tok = Guarded1d(B * L, f32, dev)
        chunk = base[r0:r0 + n, shift:shift + V]
        ops.ce_marginal_rows_(chunk, ids, mask, nsum, tok.view.view(B, L), r0, V, grad_out=1.5)
        tok.check(what + " tok_lp")
        rows = torch.arange(r0, r0 + n, device=dev)
        untouched = torch.ones(B * L, dtype=torch.bool, device=dev)
        untouched[r0:r0 + n] = False
        assert (tok.view.view(torch.int32)[untouched] == tok.bits).all(), what + ": tok_lp written outside the chunk's rows"
        assert torch.equal(base[untouched, shift:shift + V].view(itype), x[untouched].view(itype)), what + ": rows outside the chunk written"
        got_lp, got_dl = tok.view[r0:r0 + n], chunk
    else:
        logits = base.view(B, L, ld)[:, :, shift:shift + V]
        tok_lp, dl = ops.ce_marginal(logits, ids, mask, nsum, need_grad=True, inplace=mode == "inplace", grad_out=1.5)
        if mode == "inplace":
            assert dl.data_ptr() == logits.data_ptr()
        rows = torch.arange(B * L, device=dev)
        got_lp, got_dl = tok_lp.reshape(-1), dl.reshape(B * L, V)
    assert torch.isnan(base[:, :shift]).all() and torch.isnan(base[:, shift + V:]).all(), what + ": padding columns written"
    _ce_check(x[rows], ids, mask, nsum, rows, got_lp, got_dl, dtype, what)


def _ce_check(x, ids, mask, nsum, rows, got_lp, got_dl, dtype, what):
    B, L = ids.shape
    V = x.shape[1]
    x64 = x.double()
    t = rows % L
    valid = t < L - 1
    nxt = (rows + 1).clamp_max(B * L - 1)
    w = torch.where(valid, mask.view(-1)[nxt], torch.zeros_like(t)).double()
    label = torch.where(valid, ids.view(-1)[nxt], torch.zeros_like(t))
    lse = torch.logsumexp(x64, 1, keepdim=True)
    lp = (x64.gather(1, label[:, None]) - lse)[:, 0] * (w > 0)
    mx = x64.max(1, keepdim=True).values
    span = mx - x64.min(1, keepdim=True).values
    # V exponentials summed in chains of V / 512 per thread + 24 for the block tree, each __expf of a difference <= span;
    # __logf of a sum in [1, V] (2^-21.41 absolute or 3 ulp of lse - max); mx + log one rounding
    dlse = ((V / 512 + 24) * U + (2 + 1.173 * span) * EXP_ULP + U * span + LOGF_ABS + 3 * EXP_ULP * (lse - mx) + U * lse.abs())
    _expect_close(_v(got_lp), _v(lp), _v((dlse[:, 0] + U * lp.abs()) * (w > 0)), what + " tok_lp")
    prob = torch.exp(x64 - lse)
    onehot = torch.zeros_like(prob).scatter_(1, label[:, None], 1.0)
    coef = (1.5 * w / nsum.double())[:, None]
    ref = coef * (prob - onehot)
    # p = __expf(x - lse): lse's error, the difference's rounding and the __expf ulps; - 1, * coef (itself 2 roundings); the
    # store rounds to bf16 (RNE: within one ulp) or is exact (fp32)
    tol = coef.abs() * (prob * (dlse + _expf_rel(x64 - lse)) + 4 * U * (prob - onehot).abs())
    tol = tol + (_ulp_bf16(ref) if dtype == bf16 else U * ref.abs())
    _expect_close(got_dl, ref, tol, what + " dlogits")
    assert torch.equal(got_dl[w == 0].double(), torch.zeros_like(ref[w == 0])), what + ": rows with mask 0 not zeroed"
    assert torch.equal(got_lp[w == 0].double(), torch.zeros_like(lp[w == 0])), what + ": tok_lp of rows with mask 0"


@pytest.mark.parametrize("dtype,V,ld,mode", CE_CASES)
def test_ce_rows_paths(ops, cuda_dev, dtype, V, ld, mode):
    _ce_run(ops, cuda_dev, dtype, V, ld, mode)


@pytest.mark.parametrize("dtype", [bf16, f32])
@pytest.mark.parametrize("mode", ["out", "inplace", "rows"])
def test_ce_rows_misaligned(ops, cuda_dev, dtype, mode):
    """logits[..., 1:1 + V] of rows padded to a multiple of 16 bytes: ld and V allow 16-byte vectors, the pointer does not"""
    _ce_run(ops, cuda_dev, dtype, 4096, 4104, mode, shift=1)


@pytest.mark.parametrize("with_inbatch", [True, False])
def test_finalize_loss(ops, cuda_dev, with_inbatch):
    dev, B, L = cuda_dev, 72, 512                                       # B * L = 36 864 token rows
    g = torch.Generator(device=dev).manual_seed(5)
    tok = -torch.rand(B, L, generator=g, device=dev) * 12
    mask = (torch.rand(B, L, generator=g, device=dev) < 0.8).long()
    nsum = mask[:, 1:].sum().float().view(1)
    inb = torch.tensor([1.25, -0.375, 0.875, 700.0], device=dev) if with_inbatch else None
    out = ops.finalize_loss(_dense_poisoned(tok), mask, nsum, inb).cpu().double()
    terms = (mask[:, 1:].double() * tok[:, :-1].double())
    N = nsum.item()
    lm = -(terms.sum() / N).item()
    # 36 864 / 512 = 72 additions per thread + 10 for the block tree, then / N (one rounding)
    tol_lm = ((72 + 10) * U * terms.abs().sum() / N).item() + U * abs(lm)
    lc, doc = (1.25, -0.375) if with_inbatch else (0.0, 0.0)
    want = torch.tensor([lc, lm + doc, lc + lm + doc, N], dtype=f64)
    tol = torch.tensor([0.0, tol_lm + U * abs(lm + doc), tol_lm + 2 * U * (abs(lc + lm) + abs(lc + lm + doc)), 0.0], dtype=f64)
    _expect_close(_v(out), _v(want), _v(tol), f"finalize_loss inbatch {with_inbatch}")


# ----------------------------------------------------------------------------------------------------------------
# masked mean-pool + L2 normalise, forward and backward
# ----------------------------------------------------------------------------------------------------------------
POOL = [(384, 0), (1024, 0), (4096, 0),       # two-launch pool_sum path (H % 128 == 0, hidden 16-byte aligned)
        (72, 0), (1001, 0), (1024, 1),        # per-sample kernel: H % 128 != 0, or hidden 4 bytes past alignment
        (12288, 0)]                           # the widest d_pooled pool_norm_bwd holds in shared memory
POOL_B, POOL_L = 4, 40


def _pool_mask(dev):
    m = torch.ones(POOL_B, POOL_L, dtype=torch.int64)
    m[0, ::3] = 0                             # holes
    m[1] = 0
    m[1, POOL_L - 3] = 1                      # one valid token
    m[2] = 0                                  # every token masked: count clamped to 1e-9, zero norm
    return m.to(dev)                          # sample 3: every token, on an offset of 1000


@pytest.mark.parametrize("H,shift", POOL)
@pytest.mark.parametrize("normalize", [True, False])
def test_pool_norm(ops, cuda_dev, H, shift, normalize):
    dev, B, L = cuda_dev, POOL_B, POOL_L
    g = torch.Generator(device=dev).manual_seed(H + shift)
    mask = _pool_mask(dev)
    hidden = torch.randn(B, L, H, generator=g, device=dev)
    hidden[3] += 1000.0
    hidden[mask == 0] = float("nan")                                   # masked rows must not leak into the sums
    buf = torch.full((B * L * H + 64,), float("nan"), device=dev)
    hv = buf[shift:shift + B * L * H].view(B, L, H)
    hv.copy_(hidden)
    emb, norm = ops.pool_norm_fwd(hv, mask, normalize)
    what = f"pool_norm H {H} shift {shift} normalize {normalize}"
    m = mask.double()
    h64 = torch.where(mask[..., None] > 0, hidden.double(), torch.zeros((), dtype=f64, device=dev))
    inv = 1.0 / m.sum(1).clamp_min(EPS9)
    hs = h64.sum(1)
    pooled = hs * inv[:, None]
    # L masked rows summed (<= L / 8 per warp + 8 partials, or L per thread), then * (1 / count): two roundings
    tol_p = ((L + 8) * U * h64.abs().sum(1) + 2 * U * hs.abs()) * inv[:, None]
    nrm = pooled.norm(dim=1)
    # squares of values within tol_p; H / 256 per thread + 10 tree additions; sqrtf one rounding
    tol_n = (pooled.abs() * tol_p).sum(1) / nrm.clamp_min(1e-300) + ((H / 256 + 12) * U + U) * nrm
    _expect_close(_v(norm), _v(nrm), _v(tol_n), what + " norm")
    if normalize:
        s = 1.0 / nrm.clamp_min(EPS12)
        ref = pooled * s[:, None]
        tol = tol_p * s[:, None] + ref.abs() * (tol_n * s + 3 * U)[:, None]
    else:
        ref, tol = pooled, tol_p
    _expect_close(emb, ref, tol, what + " emb")

    d_emb = torch.randn(B, H, generator=g, device=dev)
    dh = ops.pool_norm_bwd(emb, norm, _dense_poisoned(d_emb), mask, L, normalize)
    e, n, de = emb.double(), norm.double(), d_emb.double()
    if normalize:
        dot = (e * de).sum(1, keepdim=True)
        tol_dot = (H / 256 + 12) * U * (e * de).abs().sum(1, keepdim=True)
        big = (n > EPS12)[:, None]
        d = torch.where(big, (de - e * dot) / n[:, None], de / EPS12)
        # (d_emb - emb * dot) / norm: dot's error times |emb|, three roundings; or d_emb / 1e-12: one
        tol_d = torch.where(big, (e.abs() * tol_dot + 3 * U * (de.abs() + (e * dot).abs())) / n[:, None], U * d.abs())
    else:
        d, tol_d = de, torch.zeros_like(de)
    dp = d * inv[:, None]
    tol_dp = tol_d * inv[:, None] + 2 * U * dp.abs()                   # * (1 / count): two roundings
    _expect_close(dh.reshape(B * L, H), (m[..., None] * dp[:, None]).reshape(B * L, H),
                  (m[..., None] * tol_dp[:, None]).reshape(B * L, H), what + " d_hidden")
    assert (dh[mask == 0] == 0).all(), what + ": masked rows of d_hidden not exactly 0"


# ----------------------------------------------------------------------------------------------------------------
# LoRA: skinny GEMM (u = x A^T, g = dY B) and the token-contracting weight gradient
# ----------------------------------------------------------------------------------------------------------------
SKINNY = [(1, 8, 8), (31, 136, 16), (33, 120, 24), (65, 1032, 32),    # M tails at the 32-row CTA, K tails at the 128 chunk
          (96, 256, 16), (200, 4096, 8), (64, 128, 32)]


@pytest.mark.parametrize("M,K,R", SKINNY)
def test_skinny_gemm(ops, cuda_dev, M, K, R):
    """x and out share one augmented buffer (the engine's [x | u] layout): out is its tail columns"""
    dev = cuda_dev
    g = torch.Generator().manual_seed(M * K + R)
    x = _ints((M, K), g).to(dev, bf16)
    w = _ints((R, K), g).to(dev, bf16)
    aug = Guarded(M, K + R, bf16, dev)
    aug.view[:, :K] = x
    ops.skinny_gemm(aug.view[:, :K], _poisoned(w), aug.view[:, K:], K=K, R=R)
    what = f"skinny_gemm M {M} K {K} R {R}"
    aug.check(what)
    _expect_equal(aug.view[:, :K], x, what + " (input columns)")
    _expect_equal(aug.view[:, K:], (x.double() @ w.double().t()).to(bf16), what)   # exact integers, one bf16 rounding


LORA_WGRAD = [  # (M, K, R, transposed output)
    (1, 8, 8, False), (63, 120, 16, False), (65, 136, 8, True),          # M tails at the 64-row chunk, K tails at 128
    (511, 264, 16, True), (513, 128, 16, False), (1100, 136, 8, False),   # ... and at the 512-token slab
    (1100, 264, 16, True),
]


@pytest.mark.parametrize("M,K,R,transposed", LORA_WGRAD)
def test_lora_wgrad(ops, cuda_dev, M, K, R, transposed):
    """out[r, k] += scale sum_m g[m, r] x[m, k] over two calls (scales 1 and 0.5): integer sums, exact whatever the atomics'
    order. transposed: a dense [K, 8] output (so_r = 1, so_k = 8, dB^T's layout); else [8, K] rows at a guarded stride."""
    dev = cuda_dev
    gen = torch.Generator().manual_seed(M + K + R)
    xs = [_ints((M, K), gen).to(dev, bf16) for _ in range(2)]
    gs = [_ints((M, R), gen).to(dev, bf16) for _ in range(2)]
    inits = [_ints((8, K), gen, hi=3).to(dev) for _ in range(R // 8)]
    outs, views = [], []
    for init in inits:
        if transposed:
            o = Guarded1d(K * 8, f32, dev, init=init.t().contiguous())
            views.append((o.view, o.view.view(K, 8).t()))
            so_r, so_k = 1, 8
        else:
            o = Guarded(8, K, f32, dev, init=init)
            views.append((o.view, o.view))
            so_r, so_k = o.view.stride(0), 1
        outs.append(o)
    for x, gg, scale in zip(xs, gs, (1.0, 0.5)):
        ops.lora_wgrad_(_poisoned(x), _poisoned(gg), views[0][0], so_r, so_k, K, R, scale,
                        out1=views[1][0] if R == 16 else None)
    ref = (gs[0].double().t() @ xs[0].double()) + 0.5 * (gs[1].double().t() @ xs[1].double())
    what = f"lora_wgrad M {M} K {K} R {R} transposed {transposed}"
    for j, (o, (_, logical)) in enumerate(zip(outs, views)):
        o.check(what + f" out{j}")
        _expect_equal(logical, inits[j].double() + ref[8 * j:8 * j + 8], what + f" out{j}")


# ----------------------------------------------------------------------------------------------------------------
# exact inner-product top-k
# ----------------------------------------------------------------------------------------------------------------
TOPK = [  # (D, N, nq, K)
    (4, 5000, 9, 32), (96, 3000, 17, 32),                 # register kernel, small D
    (128, 20000, 1, 1), (1024, 4099, 9, 32),              # pipelined kernel
    (4096, 3001, 17, 32), (6400, 1500, 9, 8),             # register kernel past the pipelined one's D; 6400: largest tile
    (128, 20, 3, 32), (4096, 1, 1, 32), (1024, 1, 2, 1),  # N < K (-1 padding), N = 1
]


@pytest.mark.parametrize("D,N,nq,K", TOPK)
def test_topk_ip(ops, cuda_dev, D, N, nq, K):
    """integer Q / P: every score exact. Query 0's best row is copied to ~40 passages spread over the whole matrix (ties
    across warps, CTAs and the merge); at D = 4 most scores tie. Order: higher score first, lower index on ties."""
    dev = cuda_dev
    g = torch.Generator().manual_seed(D * 7 + N + nq + K)
    Q = _ints((nq, D), g)
    P = _ints((N, D), g)
    hot = torch.arange(3, max(3, N), max(1, N // 40))
    P[hot] = 2 * torch.sign(Q[0])
    Q, P = Q.to(dev), P.to(dev)
    scores, idx = ops.topk_ip(_dense_poisoned(Q), _poisoned(P), K)
    ref = Q.double() @ P.double().t()
    vals, order = torch.sort(ref, dim=1, descending=True, stable=True)
    kk = min(K, N)
    what = f"topk D {D} N {N} nq {nq} K {K}"
    _expect_equal(idx[:, :kk], order[:, :kk], what + " indices")
    _expect_equal(scores[:, :kk], vals[:, :kk], what + " scores")
    if kk < K:
        assert (idx[:, kk:] == -1).all() and (scores[:, kk:] == float("-inf")).all(), what + ": padding past N"


# ----------------------------------------------------------------------------------------------------------------
# decode step: attention against the KV cache, RoPE at position ids, greedy argmax + bookkeeping
# ----------------------------------------------------------------------------------------------------------------
DECODE = [  # (D, Hq, Hkv, T, cur, window, device columns)
    (32, 4, 4, 300, 257, 0, False), (64, 8, 2, 1000, 999, 0, True), (128, 8, 1, 520, 300, 0, True),
    (128, 32, 4, 8192, 8191, 0, False),                   # the largest cache the kernel accepts, full
    (64, 4, 1, 700, 650, 128, False), (128, 8, 8, 400, 399, 100, True),
]


def _decode_ref(q, Kc, Vc, valid, Hq, Hkv, D, scale):
    """fp64 attention of one query row over n cached columns -> (out [Hq, D], bound before the bf16 store)"""
    n = Kc.shape[0]
    G = Hq // Hkv
    qs = q.view(Hq, D) * scale
    Kh = Kc.view(n, Hkv, D).repeat_interleave(G, 1)
    Vh = Vc.view(n, Hkv, D).repeat_interleave(G, 1)
    s = torch.einsum("hd,nhd->hn", qs, Kh).masked_fill(~valid[None], float("-inf"))
    P = torch.softmax(s, 1)
    o = torch.einsum("hn,nhd->hd", P, Vh)
    # scores: q * scale (one rounding) and D-term sums; each p = __expf(s - m) then carries the score errors and its own
    # ulps; a relative error eps_t of p_t moves the normalised output by at most sum_t P_t eps_t (|V_t| + |o|)
    ds = (D + 2) * U * torch.einsum("hd,nhd->hn", qs.abs(), Kh.abs())
    x = (s - s.amax(1, keepdim=True)).masked_fill(~valid[None], 0.0)
    eps = (ds + _expf_rel(x)) * P
    Va = Vh.abs()
    tol = torch.einsum("hn,nhd->hd", eps, Va) + eps.sum(1, keepdim=True) * o.abs()
    # P V sums (n / key groups per thread + the 16 group partials), sum of p (n / 128 + the block tree), the division
    tol = tol + (n + 16) * U * torch.einsum("hn,nhd->hd", P, Va) + (n / 128 + 14) * U * o.abs()
    return o.reshape(-1), tol.reshape(-1)


@pytest.mark.parametrize("D,Hq,Hkv,T,cur,window,device_cols", DECODE)
def test_attention_decode(ops, cuda_dev, D, Hq, Hkv, T, cur, window, device_cols):
    """padded cache rows (row stride Hkv D + 16) and sequences (T rows + 64 elements) inside guarded buffers; masked
    columns <= cur hold +-1e4 (they must get probability exactly 0), columns > cur hold NaN"""
    dev, B = cuda_dev, 3
    scale = 0.7 / math.sqrt(D)
    curs = [cur, cur - 37, cur // 2] if device_cols else [cur] * B
    W = Hkv * D
    st, sb = W + 16, T * (W + 16) + 64
    g = torch.Generator(device=dev).manual_seed(D + Hq + T + cur)
    mask = torch.ones(B, T + 24, dtype=torch.int64, device=dev)[:, :T]
    mask.copy_((torch.rand(B, T, generator=g, device=dev) > 0.25).long())
    mask[:, 0] = 1
    mask[0, curs[0]] = 0                                                # column cur is the new token: visible regardless
    caches, vals = [], []
    for _ in range(2):
        cb = Guarded1d(B * sb, bf16, dev)
        cb.view.fill_(float("nan"))
        c = torch.as_strided(cb.view, (B, T, W), (sb, st, 1))
        v = torch.randn(B, T, W, generator=g, device=dev)
        junk = torch.where(torch.rand(B, T, W, generator=g, device=dev) > 0.5, 1e4, -1e4)
        v = torch.where(mask[..., None] > 0, v, junk)
        for b in range(B):
            v[b, curs[b] + 1:] = float("nan")
        c.copy_(v.to(bf16))
        caches.append((cb, c))
        vals.append(c.clone())
    q_col, k_col = 0, Hq * D + 8
    v_col = k_col + W + 8
    qkv = torch.full((B, v_col + W + 24), float("nan"), dtype=bf16, device=dev)
    for c0, w in ((q_col, Hq * D), (k_col, W), (v_col, W)):
        qkv[:, c0:c0 + w] = torch.randn(B, w, generator=g, device=dev).to(bf16)
    before = [cb.buf.clone() for cb, _ in caches]
    out = Guarded(B, Hq * D, bf16, dev)
    cur_arg = torch.tensor(curs, dtype=torch.int32, device=dev) if device_cols else cur
    ops.attention_decode(qkv, q_col, k_col, v_col, caches[0][1], caches[1][1], mask, cur_arg, Hq, Hkv, D, out=out.view,
                         scale=scale, window=window)
    what = f"attention_decode D {D} Hq {Hq} Hkv {Hkv} T {T} cur {curs} window {window}"
    out.check(what + " out")
    for (cb, _), exp, col, name in zip(caches, before, (k_col, v_col), ("K", "V")):
        ev = torch.as_strided(exp[GUARD_C:GUARD_C + B * sb], (B, T, W), (sb, st, 1))
        for b in range(B):
            ev[b, curs[b]] = qkv[b, col:col + W]                        # the appended row, bit for bit
        bad = cb.buf.view(torch.int16) != exp.view(torch.int16)
        assert not bad.any(), f"{what}: cache {name}: {int(bad.sum())} elements differ, first at {int(bad.nonzero()[0])}"
    worst_shifted = 0.0
    for b in range(B):
        c = curs[b]
        t0 = max(0, c - window + 1) if window else 0
        cols = torch.arange(t0, c + 1, device=dev)
        Kc, Vc = vals[0][b, t0:c + 1].double(), vals[1][b, t0:c + 1].double()
        Kc[-1], Vc[-1] = qkv[b, k_col:k_col + W].double(), qkv[b, v_col:v_col + W].double()
        q = qkv[b, q_col:q_col + Hq * D].double()
        valid = mask[b, cols] != 0
        valid[-1] = True
        o, tol = _decode_ref(q, Kc, Vc, valid, Hq, Hkv, D, scale)
        tol = tol + _ulp_bf16(o)                                        # the bf16 store
        _expect_close(out.view[b:b + 1], o[None], tol[None], what + f" row {b}")
        # control: the mask one column off must miss this bound by far, so the bound would catch a mask / column slip
        vs = mask[b, (cols - 1).clamp_min(0)] != 0
        vs[-1] = True
        Ks, Vs = Kc.clone(), Vc.clone()
        Ks[:-1], Vs[:-1] = torch.nan_to_num(Ks[:-1]), torch.nan_to_num(Vs[:-1])
        os_, _ = _decode_ref(q, Ks, Vs, vs, Hq, Hkv, D, scale)
        worst_shifted = max(worst_shifted, ((out.view[b].double() - os_).abs() / tol).max().item())
    assert worst_shifted > 10, f"{what}: a mask shifted by one column stays within {worst_shifted:.2f}x of the bound"



@pytest.mark.parametrize("D", [64, 128])
def test_rope_pos(ops, cuda_dev, D):
    """heads at column 24 of a wider guarded row; positions < 0 and >= T clamp to [0, T - 1]; table rows past T are NaN"""
    dev, M, nheads, col0, T = cuda_dev, 12, 3, 24, 50
    half, W = D // 2, 24 + 3 * D + 40
    g = torch.Generator(device=dev).manual_seed(D)
    pos = torch.tensor([-5, -1, 0, 1, 7, 23, T - 2, T - 1, T, T + 1, T + 100, 2 ** 40], dtype=torch.int64, device=dev)
    inv = 1.0 / (10000.0 ** (torch.arange(half, dtype=f32) / half))
    fr = torch.outer(torch.arange(T, dtype=f32), inv).to(dev)
    tabs = []
    for t in (fr.cos(), fr.sin()):
        tb = torch.full((T + 64, half), float("nan"), device=dev)
        tb[:T] = t
        tabs.append(tb[:T])
    x = torch.randn(M, W, generator=g, device=dev).to(bf16)
    buf = Guarded(M, W, bf16, dev, init=x)
    ops.rope_pos_(buf.view, col0, nheads, D, tabs[0], tabs[1], pos)
    what = f"rope_pos D {D}"
    buf.check(what)
    c1 = col0 + nheads * D
    _expect_equal(buf.view[:, :col0], x[:, :col0], what + " columns before the heads")
    _expect_equal(buf.view[:, c1:], x[:, c1:], what + " columns after the heads")
    p = pos.clamp(0, T - 1)
    seg = x[:, col0:c1].double().view(M, nheads, D)
    x1, x2 = seg[..., :half], seg[..., half:]
    c, s = tabs[0].double()[p][:, None], tabs[1].double()[p][:, None]
    ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).reshape(M, nheads * D)
    terms = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1).reshape(M, nheads * D)
    # two products and a difference in fp32, then one bf16 rounding (RNE: within one ulp)
    _expect_close(buf.view[:, col0:c1], ref, _ulp_bf16(ref) + 2 * U * terms, what)


def _greedy_logits(V, dev, g):
    """rows: max at 0 / at V - 1, ties across threads and warps, +0 / -0 ties both ways, all -inf, a finished row, an EOS
    row; every row has +inf in its pad columns >= V"""
    B = 8
    x = torch.randn(B, V, generator=g, device=dev) * 4
    x[0, 0] = 100
    x[1, V - 1] = 100
    for i in (260, 300, 40 + 256 * 5, 3 + 256 * 300):                  # threads 4 / 44 (warp 1) / 40 / 3: lowest is 260
        if i < V:
            x[2, i] = 50
    a, b = (7, 33) if V < 2000 else (300, 1256)                         # b in another warp than a
    if b < V:
        for row, (lo, hi) in ((3, (0.0, -0.0)), (4, (-0.0, 0.0))):
            x[row] = -1.0
            x[row, a], x[row, b] = lo, hi
    x[5] = float("-inf")
    x[7, V - 1] = 100                                                   # V - 1 is an EOS id
    buf = torch.full((B, V + 64), float("inf"), dtype=bf16, device=dev)
    buf[:, :V] = x.to(bf16)
    return buf


@pytest.mark.parametrize("V", [1, 40, 128256, 152064])
@pytest.mark.parametrize("device_cols", [False, True])
def test_greedy_step(ops, cuda_dev, V, device_cols):
    dev, B, T, pad_id = cuda_dev, 8, 16, 77
    g = torch.Generator(device=dev).manual_seed(V)
    buf = _greedy_logits(V, dev, g)
    logits = buf[:, :V]
    eos = torch.tensor([V - 1, 10 ** 9], dtype=torch.int64, device=dev)
    unfinished = torch.ones(B, dtype=torch.int32, device=dev)
    unfinished[6] = 0
    tokens = torch.full((B, T + 5), -7, dtype=torch.int64, device=dev)
    mask = torch.zeros(B, T + 3, dtype=torch.int64, device=dev)
    next_ids = torch.full((B,), -1, dtype=torch.int64, device=dev)
    pos = torch.arange(B, dtype=torch.int64, device=dev) * 3
    alive = torch.zeros(T, dtype=torch.int32, device=dev)
    cur = torch.tensor([8, 3, 0, 12, 8, T - 1, 5, 9], dtype=torch.int32, device=dev)   # row 5: past the end -> no-op
    state = [t.clone().cpu() for t in (unfinished, tokens, mask, next_ids, pos, alive, cur)]
    ops.greedy_step_(logits, V, eos, pad_id, unfinished, tokens[:, :T], mask[:, :T], cur if device_cols else 9, next_ids, pos,
                     alive)
    # model: argmax of the bf16 row (first index of the maximum; -0 == +0; an all -inf row gives 0), then HF's bookkeeping
    row = logits.double().cpu()
    cand = [int((row[b] == row[b].max()).nonzero()[0]) for b in range(B)]
    u, tk, mk, nx, ps, al, cr = state
    for b in range(B):
        col = int(cr[b]) + 1 if device_cols else 9
        if col >= T:
            continue
        tok = cand[b] if u[b] else pad_id
        tk[b, col], mk[b, col], nx[b] = tok, 1, tok
        ps[b] += 1
        if u[b] and tok in (V - 1, 10 ** 9):
            u[b] = 0
        if u[b]:
            al[col] += 1
        if device_cols:
            cr[b] = col
    what = f"greedy_step V {V} device {device_cols}"
    for name, got, want in (("unfinished", unfinished, u), ("tokens", tokens, tk), ("mask", mask, mk),
                            ("next_ids", next_ids, nx), ("pos", pos, ps), ("alive", alive, al), ("columns", cur, cr)):
        assert torch.equal(got.cpu(), want), f"{what}: {name} {got.cpu().tolist()} != {want.tolist()}"


# ----------------------------------------------------------------------------------------------------------------
# wrapper refusals: every call below would hand a kernel an operand it reads or writes past. The operands are views into
# larger allocations, so even an unchecked call stays inside memory it owns; the wrappers must refuse before any launch.
# ----------------------------------------------------------------------------------------------------------------
def _z(*shape, dtype=bf16, dev="cuda"):
    return torch.zeros(*shape, dtype=dtype, device=dev)


REFUSALS = {
    "skinny_gemm_w_rows": lambda o, d: o.skinny_gemm(_z(64, 128), _z(16, 128)[:8], _z(64, 16), K=128, R=16),
    "skinny_gemm_out_cols": lambda o, d: o.skinny_gemm(_z(64, 128), _z(16, 128), _z(64, 16)[:, :8], K=128, R=16),
    "skinny_gemm_x_dtype": lambda o, d: o.skinny_gemm(_z(64, 128, dtype=f32), _z(16, 128), _z(64, 16), K=128, R=16),
    "skinny_gemm_oob_cpu_x": lambda o, d: o.skinny_gemm(_z(64, 128, dev="cpu"), _z(16, 128), _z(64, 16), K=128, R=16),
    "lora_wgrad_g_cols": lambda o, d: o.lora_wgrad_(_z(64, 128), _z(64, 16)[:, :8], _z(8, 128, dtype=f32), 128, 1, 128, 16,
                                                    out1=_z(8, 128, dtype=f32)),
    "lora_wgrad_out_rows": lambda o, d: o.lora_wgrad_(_z(64, 128), _z(64, 8), _z(8, 128, dtype=f32)[:4], 128, 1, 128, 8),
    "lora_wgrad_out_transposed": lambda o, d: o.lora_wgrad_(_z(64, 128), _z(64, 8), _z(128 * 8, dtype=f32)[:128 * 8 - 8], 1, 8,
                                                            128, 8),
    "lora_dx_a_rows": lambda o, d: o.lora_dx_(_z(64, 128), _z(64, 16), _z(16, 128)[:8], K=128, R=16, drop=o.Drop(0.1, 1, 1)),
    "topk_ip_p_narrow": lambda o, d: o.topk_ip(_z(3, 128, dtype=f32), _z(100, 256, dtype=f32)[:, :124], 4),
    "inbatch_loss_cvec_short": lambda o, d: o.inbatch_loss(_z(8, 64, dtype=f32), _z(8, 64, dtype=f32), 1.0,
                                                           _z(16, dtype=f32)[:7], _z(1, dtype=f32)),
    "inbatch_loss_nsum_dtype": lambda o, d: o.inbatch_loss(_z(8, 64, dtype=f32), _z(8, 64, dtype=f32), 1.0, _z(8, dtype=f32),
                                                           _z(1, dtype=f64)),
    "ce_marginal_nsum_dtype": lambda o, d: o.ce_marginal(_z(2, 3, 64), _z(2, 3, dtype=torch.int64), _z(2, 3, dtype=torch.int64),
                                                         _z(1, dtype=f64)),
    "ce_marginal_rows_nsum_dtype": lambda o, d: o.ce_marginal_rows_(_z(6, 64), _z(2, 3, dtype=torch.int64),
                                                                    _z(2, 3, dtype=torch.int64), _z(1, dtype=f64),
                                                                    _z(2, 3, dtype=f32), 0, 64),
    "finalize_loss_tok_lp_strided": lambda o, d: o.finalize_loss(_z(2, 6, dtype=f32)[:, :3], _z(2, 3, dtype=torch.int64),
                                                                 _z(1, dtype=f32), None),
    "marginal_counts_qlen_short": lambda o, d: o.marginal_counts(_z(4, 5, dtype=torch.int64), _z(8, dtype=torch.int64)[:3]),
    "attention_decode_v_cols": lambda o, d: o.attention_decode(_z(2, 256)[:, :96], 0, 64, 96, _z(2, 16, 32), _z(2, 16, 32),
                                                               _z(2, 16, dtype=torch.int64), 3, 2, 1, 32),
    "attention_decode_out_cols": lambda o, d: o.attention_decode(_z(2, 128), 0, 64, 96, _z(2, 16, 32), _z(2, 16, 32),
                                                                 _z(2, 16, dtype=torch.int64), 3, 2, 1, 32,
                                                                 out=_z(2, 128)[:, :56]),
    "attention_decode_cache_width": lambda o, d: o.attention_decode(_z(2, 128), 0, 64, 96, _z(2, 16, 64)[:, :, :24],
                                                                    _z(2, 16, 64)[:, :, :24], _z(2, 16, dtype=torch.int64), 3,
                                                                    2, 1, 32),
    "rope_pos_cols": lambda o, d: o.rope_pos_(_z(4, 512)[:, :200], 16, 3, 64, _z(10, 32, dtype=f32), _z(10, 32, dtype=f32),
                                              _z(4, dtype=torch.int64)),
    "rope_pos_table_strided": lambda o, d: o.rope_pos_(_z(4, 256), 0, 2, 64, _z(10, 64, dtype=f32)[:, :32],
                                                       _z(10, 64, dtype=f32)[:, :32], _z(4, dtype=torch.int64)),
    "pool_norm_bwd_norm_short": lambda o, d: o.pool_norm_bwd(_z(4, 64, dtype=f32), _z(8, dtype=f32)[:3], _z(4, 64, dtype=f32),
                                                             _z(4, 5, dtype=torch.int64), 5),
    "pool_norm_bwd_emb_strided": lambda o, d: o.pool_norm_bwd(_z(4, 128, dtype=f32)[:, :64], _z(4, dtype=f32),
                                                              _z(4, 64, dtype=f32), _z(4, 5, dtype=torch.int64), 5),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusal(ops, cuda_dev, Err, case):
    with pytest.raises(Err):
        REFUSALS[case](ops, cuda_dev)
    torch.cuda.synchronize()
