"""Tensor-level wrappers over the C ABI (one function per kernel entry point).

PyTorch is used here only to own device memory and the current stream; all arithmetic happens in libdalm_b200.so.
Every wrapper validates device / dtype / contiguity and then passes raw pointers.
"""
from __future__ import annotations

import math
import os
from typing import Optional, Tuple

import torch

from . import _lib

bf16 = torch.bfloat16
f32 = torch.float32
i64 = torch.int64


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, dtype, name: str, inner_contig: bool = True) -> None:
    if not t.is_cuda:
        raise _lib.DalmB200Error(f"{name}: expected a CUDA tensor (dalm_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.DalmB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if inner_contig and t.dim() > 0 and t.stride(-1) != 1:
        raise _lib.DalmB200Error(f"{name}: innermost dimension must be contiguous")


def _rows32(t: Optional[torch.Tensor], name: str, H: int, M: Optional[int] = None) -> None:
    """fp32 [M (any when None), H] operand that the kernels index as dense rows (ptr + r * H): a row-strided view would be
    read at the wrong elements, so it is refused"""
    if t is None:
        return
    _chk(t, f32, name)
    if t.dim() != 2 or t.shape[1] != H or (M is not None and t.shape[0] != M) or not t.is_contiguous():
        want = f"[{M if M is not None else 'rows'}, {H}]"
        raise _lib.DalmB200Error(f"{name}: expected dense fp32 rows {want}, got shape {tuple(t.shape)} strides {t.stride()}")


def _vec(t: Optional[torch.Tensor], dtype, name: str, n: int) -> None:
    """a vector the kernels index as t[0 .. n): anything shorter (or strided) would be read past its end"""
    if t is None:
        return
    _chk(t, dtype, name)
    if t.numel() != n or not t.is_contiguous():
        raise _lib.DalmB200Error(f"{name}: expected {n} contiguous {dtype} values, got shape {tuple(t.shape)} strides {t.stride()}")


def _bf16_rows(t: torch.Tensor, name: str, rows: int, cols: int) -> None:
    """bf16 2-D view with contiguous rows and at least [rows, cols] elements (the kernels read rows x cols at its row stride)"""
    _chk(t, bf16, name)
    if t.dim() != 2 or t.shape[0] < rows or t.shape[1] < cols:
        raise _lib.DalmB200Error(f"{name}: expected a bf16 view of at least [{rows}, {cols}], got shape {tuple(t.shape)}")


def _out_rows(t: torch.Tensor, name: str, M: int, N: int, dev: torch.device, dtypes=(bf16, f32)) -> None:
    """an output or residual the GEMM epilogues index as t[m * ld + n], m < M, n < N: on the operands' device, with a
    contiguous inner dimension and at least [M, N] elements (a smaller view would be written or read past)"""
    if not t.is_cuda or t.device != dev:
        raise _lib.DalmB200Error(f"{name}: expected a tensor on {dev}, got one on {t.device}")
    if t.dtype not in dtypes:
        raise _lib.DalmB200Error(f"{name}: expected dtype {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
    if t.dim() != 2 or t.stride(-1) != 1 or t.shape[0] < M or t.shape[1] < N:
        raise _lib.DalmB200Error(f"{name}: expected a 2-D view of at least [{M}, {N}] with contiguous rows, got shape "
                                 f"{tuple(t.shape)} strides {t.stride()}")


def _operands(a: torch.Tensor, b: torch.Tensor, what: str, layout: int = 0, K: Optional[int] = None,
              N: Optional[int] = None) -> Tuple[int, int, int]:
    """2-D GEMM operands on one device in `layout` (see `gemm`) -> (M, K, N). Without a K override the contraction extents
    of a and b must agree; overrides must fit inside the operands (the kernels read K elements of both and N of b)"""
    if a.dim() != 2 or b.dim() != 2 or b.device != a.device:
        raise _lib.DalmB200Error(f"{what}: expected 2-D operands on one device, got {tuple(a.shape)} on {a.device} and "
                                 f"{tuple(b.shape)} on {b.device}")
    M, ka = (a.shape[1], a.shape[0]) if layout == 2 else (a.shape[0], a.shape[1])
    kb, nb = (b.shape[1], b.shape[0]) if layout == 0 else (b.shape[0], b.shape[1])
    if K is None and ka != kb:
        raise _lib.DalmB200Error(f"{what}: the operands disagree on K ({ka} vs {kb}): a {tuple(a.shape)}, b {tuple(b.shape)}")
    K = ka if K is None else K
    N = nb if N is None else N
    if K > min(ka, kb) or N > nb:
        raise _lib.DalmB200Error(f"{what}: K={K} / N={N} exceed the operands a {tuple(a.shape)}, b {tuple(b.shape)}")
    return M, K, N


def _reach(t: torch.Tensor) -> int:
    """largest element offset a (non-negatively strided) view covers"""
    return sum((s - 1) * st for s, st in zip(t.shape, t.stride()))


def _tables16(*named) -> None:
    """bf16 embedding tables, which the gathers index as dense rows (id * H)"""
    for name, t in named:
        _chk(t, bf16, name)
        if not t.is_contiguous():
            raise _lib.DalmB200Error(f"{name}: expected a dense bf16 table, got strides {t.stride()}")


class Drop:
    """dropout site descriptor: probability, seed, stream id (identifies layer / tensor / call) and an optional device
    uint64 counter added to the stream id (see include/dalm_b200.h)"""
    __slots__ = ("p", "seed", "stream", "offset")

    def __init__(self, p: float, seed: int, stream: int, offset: Optional[torch.Tensor] = None):
        self.p, self.seed, self.stream, self.offset = float(p), int(seed) & (2**64 - 1), int(stream) & (2**64 - 1), offset


def _d(drop: Optional["Drop"]):
    if drop is None or drop.p <= 0.0:
        return (0.0, 0, 0, None)
    return (drop.p, drop.seed, drop.stream, _p(drop.offset))


def _ld(t: torch.Tensor) -> int:
    """row stride (elements) of a 2-D row-major view"""
    return t.stride(0) if t.dim() == 2 else t.stride(-2)


# ----------------------------------------------------------------------------------------------------------------
# loss path
# ----------------------------------------------------------------------------------------------------------------
def marginal_counts(gen_mask: torch.Tensor, qlen: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    _chk(gen_mask, i64, "gen_mask"); _chk(qlen, i64, "qlen")
    gen_mask = gen_mask.contiguous(); qlen = qlen.contiguous()
    B, L = gen_mask.shape
    _vec(qlen, i64, "marginal_counts qlen", B)
    cvec = torch.empty(B, dtype=f32, device=gen_mask.device)
    nsum = torch.empty(1, dtype=f32, device=gen_mask.device)
    _lib.call("dalm_b200_marginal_counts", _p(gen_mask), _p(qlen), B, L, _p(cvec), _p(nsum), _stream())
    return cvec, nsum


def inbatch_loss(q: torch.Tensor, p: torch.Tensor, logit_scale: float, cvec: Optional[torch.Tensor] = None,
                 nsum: Optional[torch.Tensor] = None, need_grad: bool = True, grad_out: float = 1.0):
    """returns dict(S, dlp, losses[4]={Lc, doc, Lc+doc, N}, dQ, dP)"""
    _chk(q, f32, "q"); _chk(p, f32, "p")
    q = q.contiguous(); p = p.contiguous()
    B, D = q.shape
    if p.shape != q.shape:
        raise _lib.DalmB200Error(f"inbatch_loss: q {tuple(q.shape)} and p {tuple(p.shape)} must match (in-batch negatives)")
    if (cvec is None) != (nsum is None):
        raise _lib.DalmB200Error("inbatch_loss: cvec and nsum go together")
    _vec(cvec, f32, "inbatch_loss cvec", B); _vec(nsum, f32, "inbatch_loss nsum", 1)
    dev = q.device
    S = torch.empty(B, B, dtype=f32, device=dev)
    dlp = torch.empty(B, dtype=f32, device=dev)
    losses = torch.empty(4, dtype=f32, device=dev)
    dQ = torch.empty_like(q) if need_grad else None
    dP = torch.empty_like(p) if need_grad else None
    _lib.call("dalm_b200_inbatch_loss_fwd_bwd", _p(q), _p(p), B, D, float(logit_scale), _p(cvec), _p(nsum), _p(S),
              _p(dlp), _p(losses), _p(dQ), _p(dP), float(grad_out), _stream())
    return {"S": S, "dlp": dlp, "losses": losses, "dQ": dQ, "dP": dP}


def ce_marginal(logits: torch.Tensor, ids: torch.Tensor, mask: torch.Tensor, nsum: torch.Tensor,
                need_grad: bool = True, inplace: bool = False, grad_out: float = 1.0):
    """logits [B,L,V] bf16|fp32 -> (tok_lp [B,L] fp32, dlogits or None)"""
    if logits.dtype not in (bf16, f32):
        raise _lib.DalmB200Error(f"ce_marginal: logits dtype {logits.dtype} unsupported")
    _chk(logits, logits.dtype, "logits"); _chk(ids, i64, "ids"); _chk(mask, i64, "mask")
    B, L, V = logits.shape
    if ids.shape != (B, L) or mask.shape != (B, L):
        raise _lib.DalmB200Error(f"ce_marginal: ids {tuple(ids.shape)} / mask {tuple(mask.shape)} must be [{B}, {L}] like the logits")
    _vec(nsum, f32, "ce_marginal nsum", 1)
    # rows may be padded (row stride ld >= V, e.g. a vocabulary rounded up to the GEMM's N granularity)
    rows_ok = logits.stride(2) == 1 and logits.stride(0) == L * logits.stride(1) and logits.stride(1) >= V
    if not rows_ok:
        logits = logits.contiguous()
    ld = logits.stride(1)
    ids = ids.contiguous(); mask = mask.contiguous()
    tok_lp = torch.empty(B, L, dtype=f32, device=logits.device)
    dl = None
    if need_grad:
        if inplace:
            dl = logits
        else:
            # whole padded rows are allocated (a [B,L,V] view of them is returned): the head's dgrad reads all ld columns
            base = torch.empty(B * L, ld, dtype=logits.dtype, device=logits.device)
            if ld != V:
                base.zero_()
            dl = torch.as_strided(base, (B, L, V), (L * ld, ld, 1))
    _lib.call("dalm_b200_ce_marginal_fwd_bwd", _p(logits), _p(dl), 0 if logits.dtype == bf16 else 1, _p(ids), _p(mask),
              _p(nsum), _p(tok_lp), B, L, V, ld, float(grad_out), _stream())
    return tok_lp, dl


def ce_marginal_rows_(chunk: torch.Tensor, ids: torch.Tensor, mask: torch.Tensor, nsum: torch.Tensor, tok_lp: torch.Tensor,
                      row0: int, V: int, need_grad: bool = True, grad_out: float = 1.0) -> None:
    """chunk: bf16|fp32 [n, ld >= V] = the logits of token rows [row0, row0 + n) of the flattened [B*L] rows. Writes
    tok_lp[B,L] at those rows and (need_grad) overwrites `chunk` with d(logits) in place."""
    if chunk.dtype not in (bf16, f32):
        raise _lib.DalmB200Error(f"ce_marginal_rows: logits dtype {chunk.dtype} unsupported")
    _chk(chunk, chunk.dtype, "chunk"); _chk(ids, i64, "ids"); _chk(mask, i64, "mask"); _chk(tok_lp, f32, "tok_lp")
    if chunk.dim() != 2 or not ids.is_contiguous() or not mask.is_contiguous() or not tok_lp.is_contiguous():
        raise _lib.DalmB200Error("ce_marginal_rows: chunk must be 2-D, ids / mask / tok_lp contiguous")
    B, L = ids.shape
    if mask.shape != (B, L) or tok_lp.shape != (B, L):
        raise _lib.DalmB200Error(f"ce_marginal_rows: mask {tuple(mask.shape)} / tok_lp {tuple(tok_lp.shape)} must be [{B}, {L}] "
                                 "like ids")
    if chunk.shape[1] < V:
        raise _lib.DalmB200Error(f"ce_marginal_rows: chunk {tuple(chunk.shape)} narrower than the vocabulary ({V})")
    _vec(nsum, f32, "ce_marginal_rows nsum", 1)
    _lib.call("dalm_b200_ce_marginal_rows", _p(chunk), _p(chunk) if need_grad else None, 0 if chunk.dtype == bf16 else 1, _p(ids),
              _p(mask), _p(nsum), _p(tok_lp), B, L, int(V), chunk.stride(0), float(grad_out), int(row0), chunk.shape[0], _stream())


def num_sms() -> int:
    """SM count of the current CUDA device (what the persistent GEMM grids are sized to)"""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def head_chunk_rows(M: int, Vp: int, budget_bytes: int, tile_n: int = 256, sms: Optional[int] = None) -> int:
    """Row-chunk height of the chunked lm_head + CE pass: the largest split into equal, 128-row-aligned chunks whose bf16
    logits scratch [rows, Vp] stays within `budget_bytes`, choosing among the next few chunk counts the one whose GEMMs
    waste the fewest tile waves on `sms` persistent CTAs (a chunk of m x n tiles costs ceil(m n / sms) waves; default: the
    current device's SM count)."""
    if sms is None:
        sms = num_sms()
    m_tiles = (M + 127) // 128
    n_tiles = (Vp + tile_n - 1) // tile_n
    max_rows = max(128, budget_bytes // (2 * Vp) // 128 * 128)
    n_min = max(1, -(-M // max_rows))
    best = None
    for n in range(n_min, min(m_tiles, n_min + 4) + 1):
        per = -(-m_tiles // n)                                   # m-tiles per chunk (the last chunk may be shorter)
        if per * 128 > max_rows and n > n_min:
            continue
        waves, left = 0, m_tiles
        while left > 0:
            k = min(per, left)
            waves += -(-(k * n_tiles) // sms)
            left -= k
        if best is None or waves < best[0]:
            best = (waves, per * 128)
    return best[1]


def finalize_loss(tok_lp: torch.Tensor, mask: torch.Tensor, nsum: torch.Tensor,
                  inbatch_losses: Optional[torch.Tensor]) -> torch.Tensor:
    _chk(tok_lp, f32, "finalize_loss tok_lp"); _chk(mask, i64, "finalize_loss mask")
    B, L = tok_lp.shape
    if not tok_lp.is_contiguous() or mask.shape != (B, L):
        raise _lib.DalmB200Error(f"finalize_loss: need a dense fp32 tok_lp and a mask of its shape, got tok_lp "
                                 f"{tuple(tok_lp.shape)} strides {tok_lp.stride()}, mask {tuple(mask.shape)}")
    _vec(nsum, f32, "finalize_loss nsum", 1); _vec(inbatch_losses, f32, "finalize_loss inbatch_losses", 4)
    out = torch.empty(4, dtype=f32, device=tok_lp.device)
    _lib.call("dalm_b200_finalize_loss", _p(tok_lp), _p(mask.contiguous()), B, L, _p(nsum), _p(inbatch_losses), _p(out), _stream())
    return out


def small_matmul(a: torch.Tensor, b: torch.Tensor, trans_a: bool = False, trans_b: bool = False, alpha: float = 1.0) -> torch.Tensor:
    """fp32 C = alpha * op(a) @ op(b) for the small [B,D] matrices of the stand-alone similarity API"""
    _chk(a, f32, "a"); _chk(b, f32, "b")
    a = a.contiguous(); b = b.contiguous()
    M, K = (a.shape[1], a.shape[0]) if trans_a else a.shape
    N = b.shape[0] if trans_b else b.shape[1]
    c = torch.empty(M, N, dtype=f32, device=a.device)
    _lib.call("dalm_b200_small_matmul_f32", _p(a), _p(b), _p(c), M, N, K, 1 if trans_a else 0, 1 if trans_b else 0, float(alpha), _stream())
    return c


# ----------------------------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *, out_dtype=bf16, alpha: float = 1.0,
         bias: Optional[torch.Tensor] = None, act: int = 0, resid: Optional[torch.Tensor] = None, block_n: int = 0,
         max_ctas: int = 0, K: Optional[int] = None, N: Optional[int] = None, drop: Optional[Drop] = None,
         layout: int = 0) -> torch.Tensor:
    """out[M,N] = act(alpha * A @ B^T-or-B + bias) + resid.   a, b: bf16 2-D views with contiguous rows.
    layout 0 (TN): a[M,K], b[N,K]   1 (NN, dgrad against W[out,in]): a[M,K], b[K,N]   2 (wgrad): a[K,M], b[K,N]
    act 1: GELU(erf).  act 2: GELU backward - out = bf16(alpha * A @ B + bias) * gelu'(resid), resid = the bf16 pre-activation
    (multiplied, not added): d(pre) straight out of the output projection's dgrad GEMM."""
    _chk(a, bf16, "gemm a"); _chk(b, bf16, "gemm b")
    M, K, N = _operands(a, b, f"gemm layout {layout}", layout, K, N)
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype, device=a.device)
    _out_rows(out, "gemm out", M, N, a.device)
    _chk_bias(bias, N, "gemm bias")
    rf32 = 0
    if resid is not None:
        _out_rows(resid, "gemm resid", M, N, a.device)
        rf32 = 1 if resid.dtype == f32 else 0
    if max_ctas == 0 and GEMM_MAX_CTAS:
        max_ctas = GEMM_MAX_CTAS
    timer = GEMM_TIMER
    if timer is not None:
        timer.begin(2.0 * M * N * K, (M, N, K, int(layout), str(out.dtype)[6:], "resid" if resid is not None else "-",
                                      "bias" if bias is not None else "-"))
    _lib.call("dalm_b200_gemm_bf16", int(layout), _p(a), _ld(a), _p(b), _ld(b), _p(out), _ld(out), 1 if out.dtype == f32 else 0,
              M, N, K, float(alpha), _p(bias), int(act), _p(resid), _ld(resid) if resid is not None else 0, rf32,
              int(block_n), int(max_ctas), *_d(drop), _stream())
    if timer is not None:
        timer.end()
    return out


class GemmTimer:
    """CUDA-event bracket around every GEMM launch on the launching stream (bench.py's live roofline measurement)."""

    def __init__(self, capacity: int = 4096):
        self.ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(capacity)]
        self.flops = []
        self.tags = []
        self.n = 0

    def begin(self, flops: float, tag=None) -> None:
        if self.n < len(self.ev):
            self.ev[self.n][0].record()
            self.flops.append(flops)
            self.tags.append(tag)

    def end(self) -> None:
        if self.n < len(self.ev):
            self.ev[self.n][1].record()
            self.n += 1

    def reset(self) -> None:
        self.n = 0
        self.flops = []
        self.tags = []

    def by_shape(self):
        """[(tag, launches, total_ms, TFLOP/s)] sorted by time: which GEMM shapes the step spends its tensor time in"""
        torch.cuda.synchronize()
        agg = {}
        for i in range(self.n):
            ms = self.ev[i][0].elapsed_time(self.ev[i][1])
            a = agg.setdefault(self.tags[i], [0, 0.0, 0.0])
            a[0] += 1; a[1] += ms; a[2] += self.flops[i]
        return sorted(((t, a[0], a[1], a[2] / (a[1] * 1e-3) / 1e12) for t, a in agg.items()), key=lambda r: -r[2])

    def summary(self):
        torch.cuda.synchronize()
        ms = [self.ev[i][0].elapsed_time(self.ev[i][1]) for i in range(self.n)]
        return {"launches": self.n, "total_ms": sum(ms), "total_flops": sum(self.flops[: self.n])}


GEMM_TIMER = None
# Persistent-GEMM grid cap (0 = one CTA per SM). accel.GradientSync lowers it while collectives overlap the backward (full
# fine-tuning on > 1 rank): the GEMM walks its tiles with a static stride of gridDim, so a CTA that cannot be scheduled because
# NCCL's kernels hold its SM would run ALL of its tiles after the others finished, and the overlap would buy nothing. Leaving
# NCCL its SMs keeps the wave intact.
GEMM_MAX_CTAS = 0


# ----------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------
def _window_arg(causal, window, bidirectional) -> int:
    """a window without causal means a bidirectional window (|i - j| < window, ModernBERT's local layers); the caller has to ask
    for that meaning with bidirectional=True, so that dropping `causal` from a causal (Mistral) call is still refused"""
    if bidirectional and causal:
        raise _lib.DalmB200Error("attention: bidirectional=True and causal=True are exclusive")
    if window > 0 and not causal and not bidirectional:
        raise _lib.DalmB200Error(f"attention: window {window} without causal is a bidirectional window; pass bidirectional=True "
                                 "to ask for it")
    return int(window)


def _attention_fwd(sym, q, k, v, mask, B, L, Hq, Hkv, D, causal, out, scale, drop, window, bidirectional=False):
    window = _window_arg(causal, window, bidirectional)
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _chk(t, bf16, n)
    if out is None:
        out = torch.empty(B * L, Hq * D, dtype=bf16, device=q.device)
    lse = torch.empty(B, Hq, L, dtype=f32, device=q.device)
    if mask is not None and mask.dtype != i64:
        raise _lib.DalmB200Error("attention: mask must be int64")
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    _lib.call(sym, _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(mask), _p(out), _ld(out),
              _p(lse), B, L, Hq, Hkv, D, float(scale), 1 if causal else 0, int(window), *_d(drop), _stream())
    return out, lse


def _attention_bwd(sym, q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq, dk, dv, scale, drop, window,
                   bidirectional=False):
    window = _window_arg(causal, window, bidirectional)
    dev = q.device
    if dq is None: dq = torch.empty(B * L, Hq * D, dtype=bf16, device=dev)
    if dk is None: dk = torch.empty(B * L, Hkv * D, dtype=bf16, device=dev)
    if dv is None: dv = torch.empty(B * L, Hkv * D, dtype=bf16, device=dev)
    delta = torch.empty(B, Hq, L, dtype=f32, device=dev)
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    _lib.call(sym, _p(q), _ld(q), _p(k), _ld(k), _p(v), _ld(v), _p(mask), _p(out), _ld(out),
              _p(lse), _p(d_out), _ld(d_out), _p(delta), _p(dq), _ld(dq), _p(dk), _ld(dk), _p(dv), _ld(dv),
              B, L, Hq, Hkv, D, float(scale), 1 if causal else 0, int(window), *_d(drop), _stream())
    return dq, dk, dv


def attention_fwd(q, k, v, mask, B: int, L: int, Hq: int, Hkv: int, D: int, causal: bool, out=None,
                  scale: Optional[float] = None, drop: Optional[Drop] = None, window: int = 0, bidirectional: bool = False):
    """mma.sync attention forward (head_dim 32/64/128). q/k/v: bf16 token-major 2-D views [B*L, H*D] (may be column slices
    of one qkv buffer). window > 0 with causal: query i sees key j iff i - window < j <= i (Mistral's sliding window, counted
    in the padded row); with bidirectional=True (causal False): iff |i - j| < window (ModernBERT's local layers); 0 = no
    window. -> (out, lse)"""
    return _attention_fwd("dalm_b200_attention_fwd", q, k, v, mask, B, L, Hq, Hkv, D, causal, out, scale, drop, window,
                          bidirectional)


def attention_bwd(q, k, v, mask, out, lse, d_out, B: int, L: int, Hq: int, Hkv: int, D: int, causal: bool,
                  dq=None, dk=None, dv=None, scale: Optional[float] = None, drop: Optional[Drop] = None, window: int = 0,
                  bidirectional: bool = False):
    """mma.sync attention backward (the window must be the forward's). -> (dq, dk, dv)"""
    return _attention_bwd("dalm_b200_attention_bwd", q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq, dk, dv, scale, drop,
                          window, bidirectional)


def attention_tc_fwd(q, k, v, mask, B: int, L: int, Hq: int, Hkv: int, D: int, causal: bool, out=None,
                     scale: Optional[float] = None, drop: Optional[Drop] = None, window: int = 0, bidirectional: bool = False):
    """wgmma/TMA attention forward (head_dim 128 or 64; probability dropout at 64). Same contract as attention_fwd."""
    return _attention_fwd("dalm_b200_attention_tc_fwd", q, k, v, mask, B, L, Hq, Hkv, D, causal, out, scale, drop, window,
                          bidirectional)


def attention_tc_bwd(q, k, v, mask, out, lse, d_out, B: int, L: int, Hq: int, Hkv: int, D: int, causal: bool,
                     dq=None, dk=None, dv=None, scale: Optional[float] = None, drop: Optional[Drop] = None, window: int = 0,
                     bidirectional: bool = False):
    """wgmma/TMA attention backward (head_dim 128 or 64). Same contract as attention_bwd."""
    return _attention_bwd("dalm_b200_attention_tc_bwd", q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq, dk, dv, scale, drop,
                          window, bidirectional)


def attention_auto_fwd(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=None, scale=None, drop=None, window: int = 0,
                       bidirectional: bool = False):
    """head_dim 64 / 128 -> wgmma kernels; head_dim 32 (bge-small) -> mma.sync kernels."""
    f = attention_tc_fwd if D in (64, 128) else attention_fwd
    return f(q, k, v, mask, B, L, Hq, Hkv, D, causal, out=out, scale=scale, drop=drop, window=window, bidirectional=bidirectional)


def attention_auto_bwd(q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq=None, dk=None, dv=None, scale=None, drop=None,
                       window: int = 0, bidirectional: bool = False):
    f = attention_tc_bwd if D in (64, 128) else attention_bwd
    return f(q, k, v, mask, out, lse, d_out, B, L, Hq, Hkv, D, causal, dq=dq, dk=dk, dv=dv, scale=scale, drop=drop, window=window,
             bidirectional=bidirectional)


# ----------------------------------------------------------------------------------------------------------------
# row-wise
# ----------------------------------------------------------------------------------------------------------------
def layernorm_fwd(z, gamma, beta, eps: float, y16=None, want_f32: bool = True, drop: Optional[Drop] = None):
    _chk(z, f32, "z")
    M, H = z.shape
    _rows32(z, "layernorm_fwd z", H)
    y32 = torch.empty_like(z) if want_f32 else None
    if y16 is None:
        y16 = torch.empty(M, H, dtype=bf16, device=z.device)
    mean = torch.empty(M, dtype=f32, device=z.device); rstd = torch.empty_like(mean)
    _lib.call("dalm_b200_layernorm_fwd", _p(z), _p(gamma), _p(beta), _p(y32), _p(y16), _ld(y16), _p(mean), _p(rstd), M, H,
              float(eps), *_d(drop), _stream())
    return y32, y16, mean, rstd


def layernorm_bwd(z, gamma, mean, rstd, dy_f32=None, dy_bf16=None, want_f32: bool = True, dz16=None, want_bf16: bool = True,
                  drop16: Optional[Drop] = None):
    M, H = z.shape
    _rows32(z, "layernorm_bwd z", H); _rows32(dy_f32, "layernorm_bwd dy_f32", H, M)
    if dy_bf16 is not None:
        _chk(dy_bf16, bf16, "layernorm_bwd dy_bf16")
    dz32 = torch.empty_like(z) if want_f32 else None
    if want_bf16 and dz16 is None:
        dz16 = torch.empty(M, H, dtype=bf16, device=z.device)
    _lib.call("dalm_b200_layernorm_bwd", _p(z), _p(gamma), _p(mean), _p(rstd), _p(dy_f32), _p(dy_bf16),
              _ld(dy_bf16) if dy_bf16 is not None else 0, _p(dz32), _p(dz16), _ld(dz16) if dz16 is not None else 0, M, H,
              *_d(drop16), _stream())
    return dz32, dz16


def layernorm_bwd_res(z, gamma, mean, rstd, dy_bf16, dres, dz32=None, dz16=None):
    """pre-LN residual block: dz = LayerNorm-backward(dy) + dres  -> (dz32, dz16); dz32 may be `dres` itself (in place)"""
    M, H = z.shape
    _rows32(z, "layernorm_bwd_res z", H); _rows32(dres, "layernorm_bwd_res dres", H, M); _rows32(dz32, "layernorm_bwd_res dz32", H, M)
    _chk(dy_bf16, bf16, "layernorm_bwd_res dy_bf16")
    if dz32 is None:
        dz32 = torch.empty_like(z)
    if dz16 is None:
        dz16 = torch.empty(M, H, dtype=bf16, device=z.device)
    _lib.call("dalm_b200_layernorm_bwd_res", _p(z), _p(gamma), _p(mean), _p(rstd), None, _p(dy_bf16), _ld(dy_bf16), _p(dres),
              _p(dz32), _p(dz16), _ld(dz16), M, H, _stream())
    return dz32, dz16


def rmsnorm_fwd(x, g, eps: float, h=None):
    _chk(x, f32, "x")
    M, H = x.shape
    _rows32(x, "rmsnorm_fwd x", H)
    if h is None:
        h = torch.empty(M, H, dtype=bf16, device=x.device)
    rstd = torch.empty(M, dtype=f32, device=x.device)
    _lib.call("dalm_b200_rmsnorm_fwd", _p(x), _p(g), _p(h), _ld(h), _p(rstd), M, H, float(eps), _stream())
    return h, rstd


def rmsnorm_bwd(x, g, rstd, dh, dres_in=None, dres_out=None, dres16=None, want_bf16: bool = True):
    M, H = x.shape
    _rows32(x, "rmsnorm_bwd x", H); _rows32(dres_in, "rmsnorm_bwd dres_in", H, M); _rows32(dres_out, "rmsnorm_bwd dres_out", H, M)
    _chk(dh, bf16, "rmsnorm_bwd dh")
    if dres_out is None:
        dres_out = torch.empty_like(x)
    if want_bf16 and dres16 is None:
        dres16 = torch.empty(M, H, dtype=bf16, device=x.device)
    _lib.call("dalm_b200_rmsnorm_bwd", _p(x), _p(g), _p(rstd), _p(dh), _ld(dh), _p(dres_in), _p(dres_out), _p(dres16),
              _ld(dres16) if dres16 is not None else 0, M, H, _stream())
    return dres_out, dres16


def bert_embed(ids, word, pos, type_emb, out=None):
    B, L = ids.shape
    V, H = word.shape
    _rows32(out, "bert_embed out", H, B * L)
    _tables16(("bert_embed word", word), ("bert_embed pos", pos), ("bert_embed type", type_emb))
    z = torch.empty(B * L, H, dtype=f32, device=ids.device) if out is None else out
    _lib.call("dalm_b200_bert_embed", _p(ids.contiguous()), _p(word), _p(pos), _p(type_emb), _p(z), B * L, L, H, V, _stream())
    return z


def roberta_embed(ids, word, pos, type_emb, pad_id: int, out=None, pos_ids=None):
    """RoBERTa / XLM-RoBERTa embeddings: positions from the ids (HF create_position_ids_from_input_ids with padding_idx =
    pad_id), computed on the device. Returns (z fp32 [B*L, H], position ids int64 [B*L]). Positions past the table are clamped
    by the kernel; callers check L against the table first."""
    B, L = ids.shape
    V, H = word.shape
    _rows32(out, "roberta_embed out", H, B * L)
    _tables16(("roberta_embed word", word), ("roberta_embed pos", pos), ("roberta_embed type", type_emb))
    if pos.shape[1] != H or type_emb.numel() != H:
        raise _lib.DalmB200Error(f"roberta_embed: tables must be {H} wide (pos {tuple(pos.shape)}, type {tuple(type_emb.shape)})")
    z = torch.empty(B * L, H, dtype=f32, device=ids.device) if out is None else out
    if pos_ids is None:
        pos_ids = torch.empty(B * L, dtype=i64, device=ids.device)
    _chk(pos_ids, i64, "roberta_embed pos_ids")
    if pos_ids.numel() != B * L or not pos_ids.is_contiguous():
        raise _lib.DalmB200Error(f"roberta_embed: pos_ids must be a dense int64 [{B * L}]")
    _lib.call("dalm_b200_roberta_embed", _p(ids.contiguous()), _p(word), _p(pos), _p(type_emb), int(pad_id), _p(z), _p(pos_ids),
              B, L, H, V, pos.shape[0], _stream())
    return z, pos_ids


def embed_gather(ids, table, out=None):
    M = ids.numel()
    V, H = table.shape
    _tables16(("embed_gather table", table))
    _rows32(out, "embed_gather out", H, M)
    x = torch.empty(M, H, dtype=f32, device=ids.device) if out is None else out
    _lib.call("dalm_b200_embed_gather", _p(ids.contiguous()), _p(table), _p(x), M, H, V, _stream())
    return x


def rope_(buf, col0: int, nheads: int, D: int, cos_t, sin_t, L: int, backward: bool = False):
    M = buf.shape[0]
    _lib.call("dalm_b200_rope", _p(buf), _ld(buf), col0, nheads, D, _p(cos_t), _p(sin_t), M, L, 1 if backward else 0, _stream())
    return buf


def swiglu_fwd(gu, F: int, act=None, interleave: int = 0):
    M = gu.shape[0]
    if act is None:
        act = torch.empty(M, F, dtype=bf16, device=gu.device)
    _lib.call("dalm_b200_swiglu_fwd", _p(gu), _ld(gu), _p(act), _ld(act), M, F, int(interleave), _stream())
    return act


def swiglu_bwd_(gu, dact, F: int, interleave: int = 0):
    _lib.call("dalm_b200_swiglu_bwd", _p(gu), _ld(gu), _p(dact), _ld(dact), gu.shape[0], F, int(interleave), _stream())
    return gu


def geglu_fwd(x, F: int, act=None):
    """ModernBertMLP: x = [input | gate] (bf16 [M, 2F]) -> gelu_erf(input) * gate (bf16 [M, F])"""
    M = x.shape[0]
    if act is None:
        act = torch.empty(M, F, dtype=bf16, device=x.device)
    _lib.call("dalm_b200_geglu_fwd", _p(x), _ld(x), _p(act), _ld(act), M, F, _stream())
    return act


def geglu_bwd_(x, dact, F: int):
    """in place: x <- [d_input | d_gate]"""
    _lib.call("dalm_b200_geglu_bwd", _p(x), _ld(x), _p(dact), _ld(dact), x.shape[0], F, _stream())
    return x


def gemm_swiglu(a: torch.Tensor, w_il: torch.Tensor, gu: Optional[torch.Tensor] = None, act: Optional[torch.Tensor] = None):
    """LlamaMLP's gate|up projection with SiLU(gate) * up in the GEMM epilogue. w_il: [2F, K] bf16, gate / up rows interleaved in
    blocks of 128 features (see `interleave_gate_up`). -> (gu [M,2F] interleaved bf16, act [M,F] bf16)"""
    _chk(a, bf16, "gemm_swiglu a"); _chk(w_il, bf16, "gemm_swiglu w")
    M, K, N = _operands(a, w_il, "gemm_swiglu")
    if gu is None:
        gu = torch.empty(M, N, dtype=bf16, device=a.device)
    if act is None:
        act = torch.empty(M, N // 2, dtype=bf16, device=a.device)
    _out_rows(gu, "gemm_swiglu gu", M, N, a.device, (bf16,))
    _out_rows(act, "gemm_swiglu act", M, N // 2, a.device, (bf16,))
    timer = GEMM_TIMER
    if timer is not None:
        timer.begin(2.0 * M * N * K, (M, N, K, 0, "bfloat16", "swiglu", "-"))
    _lib.call("dalm_b200_gemm_bf16_swiglu", _p(a), _ld(a), _p(w_il), _ld(w_il), _p(gu), _ld(gu), _p(act), _ld(act), M, N, K, _stream())
    if timer is not None:
        timer.end()
    return gu, act


# GELU in the GEMM epilogues pays only when the tile's mainloop is long enough to hide the erf / exp work of the 256 epilogue
# threads, so the fusion is taken from K >= 2048 (Falcon's 4544-wide MLP) and BERT (K = 1024: 16 k-blocks per tile) keeps the
# separate kernels. The threshold was chosen on the previous (Blackwell) kernels and has not been re-measured on H100.
def fuse_gelu(K: int) -> bool:
    return K >= 2048


def gemm_gelu(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, pre: Optional[torch.Tensor] = None,
              act: Optional[torch.Tensor] = None):
    """intermediate projection of a GELU MLP with the activation in the GEMM epilogue: -> (pre = a w^T + bias, gelu(pre)), both
    bf16 [M,N], one launch. Bit-identical to gemm(...) followed by gelu_fwd (the activation is taken of the rounded bf16 pre)."""
    _chk(a, bf16, "gemm_gelu a"); _chk(w, bf16, "gemm_gelu w")
    M, K, N = _operands(a, w, "gemm_gelu")
    _chk_bias(bias, N, "gemm_gelu bias")
    if pre is None:
        pre = torch.empty(M, N, dtype=bf16, device=a.device)
    if act is None:
        act = torch.empty(M, N, dtype=bf16, device=a.device)
    _out_rows(pre, "gemm_gelu pre", M, N, a.device, (bf16,))
    _out_rows(act, "gemm_gelu act", M, N, a.device, (bf16,))
    timer = GEMM_TIMER
    if timer is not None:
        timer.begin(2.0 * M * N * K, (M, N, K, 0, "bfloat16", "gelu2", "bias" if bias is not None else "-"))
    _lib.call("dalm_b200_gemm_bf16_gelu", _p(a), _ld(a), _p(w), _ld(w), _p(pre), _ld(pre), _p(act), _ld(act), M, N, K, _p(bias), _stream())
    if timer is not None:
        timer.end()
    return pre, act


def _chk_bias(bias: Optional[torch.Tensor], N: int, what: str) -> None:
    if bias is not None:
        _chk(bias, f32, what)
        if bias.dim() != 1 or bias.shape[0] < N or not bias.is_contiguous():
            raise _lib.DalmB200Error(f"{what}: need a contiguous fp32 vector of at least {N} elements, got {tuple(bias.shape)}")


def gemm_rope(a: torch.Tensor, w: torch.Tensor, cos_t: torch.Tensor, sin_t: torch.Tensor, L: int, rope_cols: int,
              out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None, *, q_norm: Optional[torch.Tensor] = None,
              k_norm: Optional[torch.Tensor] = None, nq_heads: int = 0, eps: float = 1e-6, pre_out: Optional[torch.Tensor] = None,
              rstd_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q|k|v projection with RoPE (head_dim 128) on the first `rope_cols` output columns fused into the GEMM epilogue.
    a [M,K], w [N,K] bf16; cos_t / sin_t fp32 [L, 64]; rows are token-major (position = row % L). bias: fp32 [N], added in fp32
    before the rotation (Qwen2's q/k/v biases).
    q_norm / k_norm (fp32 [128], Qwen3): each head of the rope columns is RMS-normalised (eps) before the rotation, heads
    [0, nq_heads) with q_norm, the rest with k_norm. pre_out (bf16 [M, rope_cols]) / rstd_out (fp32 [M, rope_cols // 128])
    receive the pre-norm columns and the heads' rstd, which `qk_norm_rope_bwd_` reads."""
    _chk(a, bf16, "gemm_rope a"); _chk(w, bf16, "gemm_rope w"); _chk(cos_t, f32, "gemm_rope cos"); _chk(sin_t, f32, "gemm_rope sin")
    M, K, N = _operands(a, w, "gemm_rope")
    _chk_bias(bias, N, "gemm_rope bias")
    if cos_t.shape != (L, 64) or sin_t.shape != (L, 64) or not cos_t.is_contiguous() or not sin_t.is_contiguous():
        raise _lib.DalmB200Error("gemm_rope: cos / sin must be contiguous fp32 [L, 64] (head_dim 128)")
    if (q_norm is None) != (k_norm is None) or (q_norm is None and (pre_out is not None or rstd_out is not None)):
        raise _lib.DalmB200Error("gemm_rope: q_norm and k_norm go together; pre_out / rstd_out need them")
    if q_norm is not None:
        _chk_norm_w(q_norm, "gemm_rope q_norm"); _chk_norm_w(k_norm, "gemm_rope k_norm")
        _chk_norm_saves(pre_out, rstd_out, M, rope_cols, "gemm_rope")
    if out is None:
        out = torch.empty(M, N, dtype=bf16, device=a.device)
    _out_rows(out, "gemm_rope out", M, N, a.device, (bf16,))
    timer = GEMM_TIMER
    if timer is not None:
        timer.begin(2.0 * M * N * K, (M, N, K, 0, "bfloat16", "rope" if q_norm is None else "norm_rope",
                                      "bias" if bias is not None else "-"))
    _lib.call("dalm_b200_gemm_bf16_rope", _p(a), _ld(a), _p(w), _ld(w), _p(out), _ld(out), M, N, K, _p(bias), _p(cos_t), _p(sin_t),
              int(L), int(rope_cols), _p(q_norm), _p(k_norm), int(nq_heads), float(eps), _p(pre_out),
              _ld(pre_out) if pre_out is not None else 0, _p(rstd_out), _ld(rstd_out) if rstd_out is not None else 0, _stream())
    if timer is not None:
        timer.end()
    return out


def _chk_norm_w(w: torch.Tensor, what: str) -> None:
    _chk(w, f32, what)
    if w.shape != (128,) or not w.is_contiguous():
        raise _lib.DalmB200Error(f"{what}: need a contiguous fp32 [128] weight, got {tuple(w.shape)}")


def _chk_norm_saves(pre: Optional[torch.Tensor], rstd: Optional[torch.Tensor], M: int, cols: int, what: str) -> None:
    if pre is not None:
        _chk(pre, bf16, what + " pre")
        if pre.dim() != 2 or pre.shape[0] != M or pre.shape[1] < cols:
            raise _lib.DalmB200Error(f"{what}: pre must be bf16 [{M}, >= {cols}], got {tuple(pre.shape)}")
    if rstd is not None:
        _chk(rstd, f32, what + " rstd")
        if rstd.dim() != 2 or rstd.shape[0] != M or rstd.shape[1] < cols // 128:
            raise _lib.DalmB200Error(f"{what}: rstd must be fp32 [{M}, >= {cols // 128}], got {tuple(rstd.shape)}")


def qk_norm_rope_(buf: torch.Tensor, nheads: int, nq_heads: int, q_norm: torch.Tensor, k_norm: torch.Tensor, eps: float,
                  cos_t: torch.Tensor, sin_t: torch.Tensor, L: int = 0, pos: Optional[torch.Tensor] = None,
                  pre: Optional[torch.Tensor] = None, rstd: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Qwen3's per-head q/k RMSNorm, then RoPE (head_dim 128), in place on the first `nheads` heads of buf [M, >= 128 nheads]
    (bf16, token-major): heads [0, nq_heads) take q_norm, the rest k_norm. Positions: pos[M] (int64) when given, else row % L;
    cos_t / sin_t fp32 [T, 64]. pre (bf16 [M, 128 nheads]) / rstd (fp32 [M, nheads]) optionally receive the pre-norm values and
    the heads' rstd. Allocates nothing (safe under CUDA-graph capture)."""
    _chk(buf, bf16, "qk_norm_rope buf"); _chk(cos_t, f32, "qk_norm_rope cos"); _chk(sin_t, f32, "qk_norm_rope sin")
    _chk_norm_w(q_norm, "qk_norm_rope q_norm"); _chk_norm_w(k_norm, "qk_norm_rope k_norm")
    M = buf.shape[0]
    if cos_t.dim() != 2 or cos_t.shape[1] != 64 or sin_t.shape != cos_t.shape or not cos_t.is_contiguous() or not sin_t.is_contiguous():
        raise _lib.DalmB200Error("qk_norm_rope: cos / sin must be contiguous fp32 [T, 64] (head_dim 128)")
    if pos is not None:
        _chk(pos, i64, "qk_norm_rope pos")
        if pos.numel() != M or not pos.is_contiguous():
            raise _lib.DalmB200Error(f"qk_norm_rope: need one contiguous position id per row ({pos.numel()} for {M} rows)")
    _chk_norm_saves(pre, rstd, M, 128 * nheads, "qk_norm_rope")
    _lib.call("dalm_b200_qk_norm_rope", _p(buf), _ld(buf), int(nheads), int(nq_heads), _p(q_norm), _p(k_norm), float(eps), _p(cos_t),
              _p(sin_t), cos_t.shape[0], int(L), _p(pos), M, _p(pre), _ld(pre) if pre is not None else 0, _p(rstd),
              _ld(rstd) if rstd is not None else 0, _stream())
    return buf


def qk_norm_rope_bwd_(dbuf: torch.Tensor, nheads: int, nq_heads: int, q_norm: torch.Tensor, k_norm: torch.Tensor,
                      cos_t: torch.Tensor, sin_t: torch.Tensor, L: int, pre: torch.Tensor, rstd: torch.Tensor,
                      dw_q: Optional[torch.Tensor] = None, dw_k: Optional[torch.Tensor] = None) -> torch.Tensor:
    """backward of `qk_norm_rope_` / the NormRoPE epilogue (positions row % L), in place on d(out)'s first `nheads` heads: they
    become d(pre-norm q|k). dw_q / dw_k (fp32 [128], both or neither) accumulate the norm weights' gradients (+=)."""
    _chk(dbuf, bf16, "qk_norm_rope_bwd dbuf"); _chk(cos_t, f32, "qk_norm_rope_bwd cos"); _chk(sin_t, f32, "qk_norm_rope_bwd sin")
    _chk_norm_w(q_norm, "qk_norm_rope_bwd q_norm"); _chk_norm_w(k_norm, "qk_norm_rope_bwd k_norm")
    M = dbuf.shape[0]
    if cos_t.shape != (L, 64) or sin_t.shape != (L, 64) or not cos_t.is_contiguous() or not sin_t.is_contiguous():
        raise _lib.DalmB200Error("qk_norm_rope_bwd: cos / sin must be contiguous fp32 [L, 64] (head_dim 128)")
    _chk_norm_saves(pre, rstd, M, 128 * nheads, "qk_norm_rope_bwd")
    if (dw_q is None) != (dw_k is None):
        raise _lib.DalmB200Error("qk_norm_rope_bwd: dw_q and dw_k go together")
    if dw_q is not None:
        _chk_norm_w(dw_q, "qk_norm_rope_bwd dw_q"); _chk_norm_w(dw_k, "qk_norm_rope_bwd dw_k")
    _lib.call("dalm_b200_qk_norm_rope_bwd", _p(dbuf), _ld(dbuf), int(nheads), int(nq_heads), _p(q_norm), _p(k_norm), _p(cos_t),
              _p(sin_t), int(L), _p(pre), _ld(pre), _p(rstd), _ld(rstd), M, _p(dw_q), _p(dw_k), _stream())
    return dbuf


def _chk_rope_tables(cos_t: torch.Tensor, sin_t: torch.Tensor, hd: int, what: str, T: Optional[int] = None) -> None:
    _chk(cos_t, f32, what + " cos"); _chk(sin_t, f32, what + " sin")
    if (cos_t.dim() != 2 or cos_t.shape[1] != hd // 2 or sin_t.shape != cos_t.shape or (T is not None and cos_t.shape[0] != T)
            or not cos_t.is_contiguous() or not sin_t.is_contiguous()):
        raise _lib.DalmB200Error(f"{what}: cos / sin must be contiguous fp32 [{T if T is not None else 'T'}, {hd // 2}]")


def qk_fullnorm_rope_(buf: torch.Tensor, nq_heads: int, nk_heads: int, hd: int, q_norm: torch.Tensor, k_norm: torch.Tensor,
                      eps: float, cos_t: torch.Tensor, sin_t: torch.Tensor, L: int = 0, pos: Optional[torch.Tensor] = None,
                      pre: Optional[torch.Tensor] = None, rstd: Optional[torch.Tensor] = None,
                      round_first: bool = False) -> torch.Tensor:
    """OLMo 2 / 3 / OLMoE q/k RMSNorm over the whole q (nq_heads * hd) and k (nk_heads * hd) widths, then RoPE, in place on
    the first (nq_heads + nk_heads) * hd columns of buf (bf16, token-major). round_first: OlmoeRMSNorm's rounding (bf16 before
    the weight multiply) instead of Olmo2RMSNorm's. Positions: pos[M] (int64) when given, else row % L. pre (bf16
    [M, >= width]) / rstd (fp32 [M, 2]) optionally receive the pre-norm columns and the q / k rstd. Allocates nothing."""
    _chk(buf, bf16, "qk_fullnorm_rope buf")
    _chk_rope_tables(cos_t, sin_t, hd, "qk_fullnorm_rope")
    Nq, Nk = nq_heads * hd, nk_heads * hd
    _vec(q_norm, f32, "qk_fullnorm_rope q_norm", Nq); _vec(k_norm, f32, "qk_fullnorm_rope k_norm", Nk)
    M = buf.shape[0]
    if buf.dim() != 2 or buf.shape[1] < Nq + Nk:
        raise _lib.DalmB200Error(f"qk_fullnorm_rope: buf must be bf16 [M, >= {Nq + Nk}], got {tuple(buf.shape)}")
    if pos is not None:
        _vec(pos, i64, "qk_fullnorm_rope pos", M)
    _chk_fullnorm_saves(pre, rstd, M, Nq + Nk, "qk_fullnorm_rope")
    _lib.call("dalm_b200_qk_fullnorm_rope", _p(buf), _ld(buf), int(nq_heads), int(nq_heads + nk_heads), int(hd), _p(q_norm),
              _p(k_norm), float(eps), int(bool(round_first)), _p(cos_t), _p(sin_t), cos_t.shape[0], int(L), _p(pos), M, _p(pre),
              _ld(pre) if pre is not None else 0, _p(rstd), _ld(rstd) if rstd is not None else 0, _stream())
    return buf


def _chk_fullnorm_saves(pre: Optional[torch.Tensor], rstd: Optional[torch.Tensor], M: int, cols: int, what: str) -> None:
    if pre is not None:
        _chk(pre, bf16, what + " pre")
        if pre.dim() != 2 or pre.shape[0] != M or pre.shape[1] < cols:
            raise _lib.DalmB200Error(f"{what}: pre must be bf16 [{M}, >= {cols}], got {tuple(pre.shape)}")
    if rstd is not None:
        _chk(rstd, f32, what + " rstd")
        if rstd.dim() != 2 or rstd.shape[0] != M or rstd.shape[1] < 2:
            raise _lib.DalmB200Error(f"{what}: rstd must be fp32 [{M}, 2], got {tuple(rstd.shape)}")


def qk_fullnorm_rope_bwd_(dbuf: torch.Tensor, nq_heads: int, nk_heads: int, hd: int, q_norm: torch.Tensor, k_norm: torch.Tensor,
                          cos_t: torch.Tensor, sin_t: torch.Tensor, L: int, pre: torch.Tensor, rstd: torch.Tensor,
                          dw_q: Optional[torch.Tensor] = None, dw_k: Optional[torch.Tensor] = None) -> torch.Tensor:
    """backward of `qk_fullnorm_rope_` (positions row % L), in place on d(out)'s q|k columns: they become d(pre-norm q|k).
    dw_q / dw_k (fp32 [Nq] / [Nkv], both or neither) accumulate the norm weights' gradients (+=), deterministically
    (`norm_wgrad_`, run first: it reads the rotated gradient)."""
    _chk(dbuf, bf16, "qk_fullnorm_rope_bwd dbuf")
    _chk_rope_tables(cos_t, sin_t, hd, "qk_fullnorm_rope_bwd", T=L)
    Nq, Nk = nq_heads * hd, nk_heads * hd
    _vec(q_norm, f32, "qk_fullnorm_rope_bwd q_norm", Nq); _vec(k_norm, f32, "qk_fullnorm_rope_bwd k_norm", Nk)
    M = dbuf.shape[0]
    if dbuf.dim() != 2 or dbuf.shape[1] < Nq + Nk:
        raise _lib.DalmB200Error(f"qk_fullnorm_rope_bwd: dbuf must be bf16 [M, >= {Nq + Nk}], got {tuple(dbuf.shape)}")
    if pre is None or rstd is None:
        raise _lib.DalmB200Error("qk_fullnorm_rope_bwd: needs the saved pre-norm columns and rstd")
    _chk_fullnorm_saves(pre, rstd, M, Nq + Nk, "qk_fullnorm_rope_bwd")
    if (dw_q is None) != (dw_k is None):
        raise _lib.DalmB200Error("qk_fullnorm_rope_bwd: dw_q and dw_k go together")
    if dw_q is not None:
        norm_wgrad_(dbuf[:, :Nq + Nk], pre, rstd, dw_q, dw_k, hd=hd, cos_t=cos_t, sin_t=sin_t, L=L)
    _lib.call("dalm_b200_qk_fullnorm_rope_bwd", _p(dbuf), _ld(dbuf), int(nq_heads), int(nq_heads + nk_heads), int(hd), _p(q_norm),
              _p(k_norm), _p(cos_t), _p(sin_t), int(L), _p(pre), _ld(pre), _p(rstd), _ld(rstd), M, _stream())
    return dbuf


NORM_WGRAD_MAX_SPLITS = 64


def norm_wgrad_(dy: torch.Tensor, x: torch.Tensor, rstd: torch.Tensor, dw0: torch.Tensor, dw1: Optional[torch.Tensor] = None,
                hd: int = 8, cos_t: Optional[torch.Tensor] = None, sin_t: Optional[torch.Tensor] = None, L: int = 0) -> None:
    """RMSNorm weight gradient over bf16 inputs x [M, N] (normalised by rstd), without atomics (the same bits on every run):
    dw0[c] += sum_m g[m,c] x[m,c] rstd[m,0] over the first len(dw0) columns, dw1 (+=) over the rest with rstd[m,1]. g = dy
    (fp32 or bf16 [M, N]), un-rotated within heads of width hd at positions m % L when cos_t / sin_t are given. rstd: fp32 [M]
    (one segment) or [M, 2]."""
    M, N = x.shape[0], dy.shape[1]
    _chk(x, bf16, "norm_wgrad x")
    if dy.dtype not in (bf16, f32):
        raise _lib.DalmB200Error("norm_wgrad: dy must be bf16 or fp32")
    _chk(dy, dy.dtype, "norm_wgrad dy"); _chk(rstd, f32, "norm_wgrad rstd")
    N0 = dw0.numel()
    _vec(dw0, f32, "norm_wgrad dw0", N0)
    if dw1 is not None:
        _vec(dw1, f32, "norm_wgrad dw1", N - N0)
    if dy.shape[0] != M or x.shape[1] < N or N0 + (dw1.numel() if dw1 is not None else 0) != N:
        raise _lib.DalmB200Error(f"norm_wgrad: dy {tuple(dy.shape)}, x {tuple(x.shape)}, dw widths {N0} + "
                                 f"{dw1.numel() if dw1 is not None else 0} disagree")
    segs = 2 if dw1 is not None else 1
    if rstd.shape[0] != M or (rstd.dim() == 2 and rstd.shape[1] < segs) or (rstd.dim() == 1 and segs == 2):
        raise _lib.DalmB200Error(f"norm_wgrad: rstd must be fp32 [{M}] or [{M}, {segs}], got {tuple(rstd.shape)}")
    if cos_t is not None:
        _chk_rope_tables(cos_t, sin_t, hd, "norm_wgrad", T=L)
    splits = max(1, min(NORM_WGRAD_MAX_SPLITS, (M + 63) // 64))
    part = torch.empty(splits, N, dtype=f32, device=x.device)
    _lib.call("dalm_b200_norm_wgrad", _p(dy), 1 if dy.dtype == f32 else 0, _ld(dy), _p(x), _ld(x), _p(rstd),
              rstd.stride(0), int(N0), int(N), int(hd), _p(cos_t), _p(sin_t), int(L), M, _p(part), splits, _p(dw0), _p(dw1),
              _stream())


def postnorm_fwd(y: torch.Tensor, w: torch.Tensor, resid: torch.Tensor, eps: float, out16: Optional[torch.Tensor] = None):
    """OLMo 2 / 3 post-sublayer norm and residual add: (out fp32 [M,H] = resid + bf16(w * y rstd), rstd fp32 [M]); y is the
    bf16 sublayer output. out16 (bf16 [M,H] view) optionally receives bf16(out), the next GEMM's operand."""
    _chk(y, bf16, "postnorm_fwd y")
    M, H = y.shape
    _rows32(resid, "postnorm_fwd resid", H, M); _vec(w, f32, "postnorm_fwd w", H)
    if out16 is not None:
        _bf16_rows(out16, "postnorm_fwd out16", M, H)
    out = torch.empty(M, H, dtype=f32, device=y.device)
    rstd = torch.empty(M, dtype=f32, device=y.device)
    _lib.call("dalm_b200_postnorm_fwd", _p(y), _ld(y), _p(w), _p(resid), _p(out), _p(out16), _ld(out16) if out16 is not None else 0,
              _p(rstd), M, H, float(eps), _stream())
    return out, rstd


def postnorm_bwd(y: torch.Tensor, w: torch.Tensor, rstd: torch.Tensor, dres: torch.Tensor, dh: Optional[torch.Tensor] = None):
    """backward of `postnorm_fwd`: d = dres (fp32 [M,H]) + dh (bf16, the branch gradient joining the residual here; optional)
    -> (d fp32, the residual gradient passed on; dy bf16 [M,H], the gradient of the sublayer output y)"""
    _chk(y, bf16, "postnorm_bwd y")
    M, H = y.shape
    _rows32(dres, "postnorm_bwd dres", H, M); _vec(w, f32, "postnorm_bwd w", H); _vec(rstd, f32, "postnorm_bwd rstd", M)
    if dh is not None:
        _bf16_rows(dh, "postnorm_bwd dh", M, H)
    d = torch.empty(M, H, dtype=f32, device=y.device)
    dy = torch.empty(M, H, dtype=bf16, device=y.device)
    _lib.call("dalm_b200_postnorm_bwd", _p(y), _ld(y), _p(w), _p(rstd), _p(dres), _p(dh), _ld(dh) if dh is not None else 0, _p(d),
              _p(dy), _ld(dy), M, H, _stream())
    return d, dy


def interleave_gate_up(gate_w: torch.Tensor, up_w: torch.Tensor, block: int = 128) -> torch.Tensor:
    """[F,K] gate and up weights -> [2F,K] with rows [gate blk0 | up blk0 | gate blk1 | ...] (blocks of `block` features)"""
    F, K = gate_w.shape
    if F % block:
        raise _lib.DalmB200Error(f"interleave_gate_up: F={F} is not a multiple of {block}")
    return torch.stack([gate_w.view(F // block, block, K), up_w.view(F // block, block, K)], dim=1).reshape(2 * F, K).contiguous()


def gelu_fwd(pre, act=None):
    M, F = pre.shape
    if act is None:
        act = torch.empty(M, F, dtype=bf16, device=pre.device)
    _lib.call("dalm_b200_gelu_fwd", _p(pre), _ld(pre), _p(act), _ld(act), M, F, _stream())
    return act


def gelu_bwd_(pre, dact):
    M, F = pre.shape
    _lib.call("dalm_b200_gelu_bwd", _p(pre), _ld(pre), _p(dact), _ld(dact), M, F, _stream())
    return dact


def pool_norm_fwd(hidden, mask, normalize: bool = True):
    B, L, H = hidden.shape
    _chk(hidden, f32, "hidden"); _chk(mask, i64, "mask")
    if mask.shape != (B, L):
        raise _lib.DalmB200Error(f"pool_norm_fwd: mask {tuple(mask.shape)} must be [{B}, {L}] like hidden")
    pooled = torch.empty(B, H, dtype=f32, device=hidden.device)
    emb = torch.empty_like(pooled)
    norm = torch.empty(B, dtype=f32, device=hidden.device)
    _lib.call("dalm_b200_pool_norm_fwd", _p(hidden.contiguous()), _p(mask.contiguous()), _p(pooled), _p(emb), _p(norm), B, L, H,
              1 if normalize else 0, _stream())
    return emb, norm


def pool_norm_bwd(emb, norm, d_emb, mask, L: int, normalize: bool = True):
    B, H = emb.shape
    _rows32(emb, "pool_norm_bwd emb", H, B); _vec(norm, f32, "pool_norm_bwd norm", B)
    _chk(d_emb, f32, "pool_norm_bwd d_emb", inner_contig=False); _chk(mask, i64, "pool_norm_bwd mask", inner_contig=False)
    if d_emb.shape != (B, H) or mask.shape != (B, L):
        raise _lib.DalmB200Error(f"pool_norm_bwd: d_emb {tuple(d_emb.shape)} / mask {tuple(mask.shape)} must be [{B}, {H}] / "
                                 f"[{B}, {L}]")
    d_hidden = torch.empty(B, L, H, dtype=f32, device=emb.device)
    _lib.call("dalm_b200_pool_norm_bwd", _p(emb), _p(norm), _p(d_emb.contiguous()), _p(mask.contiguous()), _p(d_hidden), B, L, H,
              1 if normalize else 0, _stream())
    return d_hidden


def lora_wgrad_(x, g, out, so_r: int, so_k: int, K: int, R: int, scale: float = 1.0, out1=None, dropx: Optional[Drop] = None):
    """out[r*so_r + k*so_k] += scale * sum_m g[m,r] x[m,k]; with R == 16 rows 8..15 accumulate into out1 (same strides)"""
    M = x.shape[0]
    _bf16_rows(x, "lora_wgrad x", M, K); _bf16_rows(g, "lora_wgrad g", M, R)
    need = (min(R, 8) - 1) * so_r + (K - 1) * so_k                      # farthest element written in each output
    for t, n in ((out, "out"), (out1, "out1")):
        if t is None:
            continue
        _chk(t, f32, f"lora_wgrad {n}", inner_contig=False)
        if so_r < 0 or so_k < 0 or min(t.stride()) < 0 or _reach(t) < need:
            raise _lib.DalmB200Error(f"lora_wgrad: {n} {tuple(t.shape)} strides {t.stride()} does not cover "
                                     f"[{min(R, 8)}, {K}] at strides ({so_r}, {so_k})")
    _lib.call("dalm_b200_lora_wgrad", _p(x), _ld(x), _p(g), _ld(g), _p(out), _p(out1), so_r, so_k, M, K, R, float(scale),
              *_d(dropx), _stream())
    return out


def skinny_gemm(x, w, out, K: int, R: int, dropx: Optional[Drop] = None):
    """out[M,R] (bf16 view) = x[M,K] @ w[R,K]^T   (R in {8,16,24,32})"""
    M = x.shape[0]
    _bf16_rows(x, "skinny_gemm x", M, K); _bf16_rows(w, "skinny_gemm w", R, K); _bf16_rows(out, "skinny_gemm out", M, R)
    if out.shape[0] != M:
        raise _lib.DalmB200Error(f"skinny_gemm: out {tuple(out.shape)} must have one row per row of x ({M})")
    _lib.call("dalm_b200_skinny_gemm", _p(x), _ld(x), _p(w), _ld(w), _p(out), _ld(out), x.shape[0], K, R, *_d(dropx), _stream())
    return out


def lora_dx_(dh, g, a_stack, K: int, R: int, drop: Drop):
    """dh[m,k] += mask(m,k)/(1-p) * sum_r g[m,r] a_stack[r,k]"""
    M = dh.shape[0]
    _bf16_rows(dh, "lora_dx dh", M, K); _bf16_rows(g, "lora_dx g", M, R); _bf16_rows(a_stack, "lora_dx a_stack", R, K)
    p, seed, stream, off = _d(drop)
    _lib.call("dalm_b200_lora_dx", _p(dh), _ld(dh), _p(g), _ld(g), _p(a_stack), _ld(a_stack), dh.shape[0], K, R, p, seed, stream, off, _stream())
    return dh


def bump_counter_(counter: torch.Tensor) -> None:
    _lib.call("dalm_b200_bump_counter", _p(counter), _stream())


def dropout_scale(n: int, drop: Drop, device) -> torch.Tensor:
    """the scale (0 or 1/(1-p)) dropout applies to each of n elements under `drop` — lets tests apply identical masks"""
    out = torch.empty(n, dtype=f32, device=device)
    p, seed, stream, off = _d(drop) if drop.p > 0 else (0.0, 0, 0, None)
    _lib.call("dalm_b200_dropout_scale", _p(out), n, p, seed, stream, off, _stream())
    return out


def pack_scaled_bf16_(src, si_r: int, si_c: int, dst, rows: int, cols: int, scale: float):
    _lib.call("dalm_b200_pack_scaled_bf16", _p(src), si_r, si_c, _p(dst), _ld(dst), rows, cols, float(scale), _stream())
    return dst


def build_pack_table(entries, device) -> torch.Tensor:
    """entries: iterable of (src_f32, si_r, si_c, dst_bf16_view, rows, cols, scale) -> device table for pack_table_()"""
    import numpy as np
    dt = np.dtype([("in", "<u8"), ("si_r", "<i8"), ("si_c", "<i8"), ("out", "<u8"), ("ldo", "<i8"), ("rows", "<i4"),
                   ("cols", "<i4"), ("scale", "<f4"), ("pad", "<i4")])
    assert dt.itemsize == 56
    rows = [(s.data_ptr(), si_r, si_c, d.data_ptr(), _ld(d), r, c, sc, 0) for (s, si_r, si_c, d, r, c, sc) in entries]
    arr = np.array(rows, dtype=dt)
    t = torch.from_numpy(arr.view(np.uint8).reshape(-1).copy()).to(device)
    t._n_entries = len(rows)
    return t


def pack_table_(table: torch.Tensor) -> None:
    _lib.call("dalm_b200_pack_table", _p(table), int(table._n_entries), _stream())


def cast_f32_bf16(src, dst=None):
    """dst bf16 [M,N] = src fp32 [M,N] (both with contiguous rows; a transposed source is refused, not misread)"""
    _chk(src, f32, "cast_f32_bf16 src")
    if dst is not None:
        _chk(dst, bf16, "cast_f32_bf16 dst")
    M, N = src.shape
    if dst is None:
        dst = torch.empty(M, N, dtype=bf16, device=src.device)
    _lib.call("dalm_b200_cast_f32_bf16", _p(src), _ld(src), _p(dst), _ld(dst), M, N, _stream())
    return dst


def wgrad_(dy, x, gw, accumulate: bool, K: Optional[int] = None) -> None:
    """gw[out,in] (fp32) = (or +=) dy[T,out]^T @ x[T,in]: the weight gradient of y = x W^T as one wgmma GEMM contracting
    over the token rows (both operands read MN-major from their row-major buffers)"""
    gemm(dy, x, out=gw, layout=2, resid=gw if accumulate else None, K=K)


def col_reduce_(dy_f32=None, dy_bf16=None, z=None, mean=None, rstd=None, out_sum=None, out_prod=None) -> None:
    """out_sum[h] += sum_m dy[m,h]; out_prod[h] += sum_m dy[m,h] * (z[m,h]-mean[m]) * rstd[m]   (dy = dy_f32 + dy_bf16)"""
    ref = dy_f32 if dy_f32 is not None else dy_bf16
    M, H = ref.shape
    _rows32(dy_f32, "col_reduce dy_f32", H, M); _rows32(z, "col_reduce z", H, M)
    if dy_bf16 is not None:
        _chk(dy_bf16, bf16, "col_reduce dy_bf16")
    _lib.call("dalm_b200_col_reduce", _p(dy_f32), _p(dy_bf16), _ld(dy_bf16) if dy_bf16 is not None else 0, _p(z), _p(mean),
              _p(rstd), _p(out_sum), _p(out_prod), M, H, _stream())


def embed_scatter_add_(d, ids, dword, dpos=None, L: int = 1, *, pos_ids=None, pad_id: int = -1) -> None:
    """pos_ids: int64 [M] positions to scatter into dpos (roberta_embed's output; None: m % L). pad_id >= 0: that word row and
    that position row receive no gradient (nn.Embedding padding_idx); -1: none"""
    M, H = d.shape
    _rows32(d, "embed_scatter_add d", H); _rows32(dword, "embed_scatter_add dword", H); _rows32(dpos, "embed_scatter_add dpos", H)
    _chk(ids, i64, "embed_scatter_add ids")
    if ids.numel() != M or not ids.is_contiguous():
        raise _lib.DalmB200Error(f"embed_scatter_add: need one contiguous id per row ({ids.numel()} for {M} rows)")
    if pos_ids is not None:
        _chk(pos_ids, i64, "embed_scatter_add pos_ids")
        if pos_ids.numel() != M or not pos_ids.is_contiguous():
            raise _lib.DalmB200Error(f"embed_scatter_add: need one contiguous position per row ({pos_ids.numel()} for {M} rows)")
    _lib.call("dalm_b200_embed_scatter_add", _p(d), _p(ids), _p(pos_ids), _p(dword), _p(dpos), M, H, int(L), dword.shape[0],
              int(pad_id), _stream())


def masked_add(a=None, b=None, drop: Optional[Drop] = None, out=None):
    ref = a if a is not None else b
    M, H = ref.shape
    _rows32(a, "masked_add a", H, M); _rows32(out, "masked_add out", H, M)
    if b is not None:
        _chk(b, bf16, "masked_add b")
    if out is None:
        out = torch.empty(M, H, dtype=f32, device=ref.device)
    _lib.call("dalm_b200_masked_add", _p(a), _p(b), _ld(b) if b is not None else 0, _p(out), M, H, *_d(drop), _stream())
    return out


def adam_step_shadow_(p, g, m, v, shadow, lr: float, beta1: float, beta2: float, eps: float, step: int, grad_scale: float = 1.0):
    _lib.call("dalm_b200_adam_step_shadow", _p(p), _p(g), _p(m), _p(v), _p(shadow), p.numel(), float(lr), float(beta1),
              float(beta2), float(eps), int(step), float(grad_scale), _stream())
    return p


def adam_step_(p, g, m, v, lr: float, beta1: float, beta2: float, eps: float, step: int, grad_scale: float = 1.0):
    _lib.call("dalm_b200_adam_step", _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2), float(eps),
              int(step), float(grad_scale), _stream())
    return p


# ----------------------------------------------------------------------------------------------------------------
# evaluation: exact inner-product top-k
# ----------------------------------------------------------------------------------------------------------------
def topk_ip(q: torch.Tensor, p: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """q fp32 [nq,D], p fp32 [N,D] (row-strided) -> (scores fp32 [nq,k] descending, idx int32 [nq,k]; -1 past N)"""
    _chk(q, f32, "topk q"); _chk(p, f32, "topk p")
    if not q.is_contiguous():
        q = q.contiguous()
    nq, D = q.shape
    N = p.shape[0]
    if p.dim() != 2 or p.shape[1] != D:
        raise _lib.DalmB200Error(f"topk_ip: passages {tuple(p.shape)} must be [N, {D}] like the queries")
    scores =torch.empty(nq, k, dtype=f32, device=q.device)
    idx = torch.empty(nq, k, dtype=torch.int32, device=q.device)
    ws = torch.empty(int(_lib.load().dalm_b200_topk_ip_workspace(nq, k)), dtype=torch.uint8, device=q.device)
    _lib.call("dalm_b200_topk_ip", _p(q), _p(p), _ld(p), nq, N, D, int(k), _p(scores), _p(idx), _p(ws), _stream())
    return scores, idx


# ----------------------------------------------------------------------------------------------------------------
# use_bnb with 4-bit storage: packed NF4 codes + absmax, expanded to bf16 right before the GEMM
def nf4_quantize(w: torch.Tensor):
    """w fp32 contiguous [rows, cols] -> (packed uint8 [rows*cols/2], absmax fp32 [rows*cols/64]); blocks of 64 over the
    flattened row-major weight (bitsandbytes quantize_4bit, nf4, blocksize 64)"""
    _chk(w, f32, "nf4_quantize w")
    if not w.is_contiguous():
        raise _lib.DalmB200Error("nf4_quantize: tensor must be contiguous")
    n = w.numel()
    packed = torch.empty((n + 1) // 2, dtype=torch.uint8, device=w.device)
    absmax = torch.empty((n + 63) // 64, dtype=f32, device=w.device)
    _lib.call("dalm_b200_nf4_quantize", _p(w), n, _p(packed), _p(absmax), _stream())
    return packed, absmax


def nf4_dequant_(packed: torch.Tensor, absmax: torch.Tensor, rows: int, cols: int, out: torch.Tensor,
                 tail: Optional[torch.Tensor] = None) -> torch.Tensor:
    """packed / absmax of a [rows, cols] weight -> out[:, :cols] (bf16, row stride out.stride(0)); `tail` (bf16 [rows, t]) is
    copied into out[:, cols:cols+t]"""
    _chk(out, bf16, "nf4_dequant out")
    t = 0 if tail is None else tail.shape[1]
    if out.shape[0] != rows or out.shape[1] < cols + t:
        raise _lib.DalmB200Error(f"nf4_dequant: out {tuple(out.shape)} too small for [{rows}, {cols}+{t}]")
    _lib.call("dalm_b200_nf4_dequant_bf16", _p(packed), _p(absmax), rows, cols, _p(out), out.stride(0), _p(tail),
              tail.stride(0) if tail is not None else 0, t, _stream())
    return out


# use_bnb: NF4 round trip of a weight at load time
# ----------------------------------------------------------------------------------------------------------------
def nf4_roundtrip_(w: torch.Tensor, want_codes: bool = False):
    """w fp32 contiguous (any shape) -> overwritten with dequant(quant_nf4(fp16(w))); optionally (codes uint8 [n], absmax [n/64])"""
    _chk(w, f32, "nf4 w")
    if not w.is_contiguous():
        raise _lib.DalmB200Error("nf4_roundtrip_: tensor must be contiguous (blocks are taken over the flattened row-major weight)")
    n = w.numel()
    codes = torch.empty(n, dtype=torch.uint8, device=w.device) if want_codes else None
    absmax = torch.empty((n + 63) // 64, dtype=f32, device=w.device) if want_codes else None
    _lib.call("dalm_b200_nf4_roundtrip", _p(w), n, _p(codes), _p(absmax), _stream())
    return (w, codes, absmax) if want_codes else w


# ----------------------------------------------------------------------------------------------------------------
# greedy decoding (evaluation: reference dalm/eval/eval_rag.py:126-140)
# ----------------------------------------------------------------------------------------------------------------
def decode_gemm(a: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, *, out_dtype=bf16, act: int = 0,
                resid: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M,N] = act(a[M,K] @ w[N,K]^T + bias) + resid for the M <= 16 token rows of a decode step: weight-streaming kernel,
    every weight read once. a, w bf16 with contiguous rows (row strides multiples of 8); bias fp32 [N]; resid / out bf16 or fp32."""
    _chk(a, bf16, "decode_gemm a"); _chk(w, bf16, "decode_gemm w")
    M, K, N = _operands(a, w, "decode_gemm")
    _chk_bias(bias, N, "decode_gemm bias")
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype, device=a.device)
    _out_rows(out, "decode_gemm out", M, N, a.device)
    if resid is not None:
        _out_rows(resid, "decode_gemm resid", M, N, a.device)
    _lib.call("dalm_b200_decode_gemm", _p(a), _ld(a), _p(w), _ld(w), _p(out), _ld(out), 1 if out.dtype == f32 else 0, _p(bias), _p(resid),
              _ld(resid) if resid is not None else 0, 1 if (resid is not None and resid.dtype == f32) else 0, int(act), M, N, K,
              _stream())
    return out


def gemm_rows(a: torch.Tensor, w: torch.Tensor, *, out_dtype=bf16, act: int = 0, resid: Optional[torch.Tensor] = None,
              bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act(a[M,K] @ w[N,K]^T + bias) + resid for a decode step: up to 16 rows go through the weight-streaming `decode_gemm` (the
    128-row wgmma tile would be 7/8 empty), larger batches through the training GEMM. DALM_B200_DECODE_GEMM=0 forces the latter."""
    if a.shape[0] <= 16 and os.environ.get("DALM_B200_DECODE_GEMM", "1") != "0":
        return decode_gemm(a, w, out_dtype=out_dtype, act=act, resid=resid, bias=bias)
    return gemm(a, w, out_dtype=out_dtype, act=act, resid=resid, bias=bias)


def rope_pos_(buf, col0: int, nheads: int, D: int, cos_t, sin_t, pos):
    """in-place RoPE of `nheads` heads at explicit position ids pos[M] (int64); cos_t / sin_t fp32 [T, D/2]"""
    _chk(buf, bf16, "rope_pos buf"); _chk(pos, i64, "rope_pos pos"); _chk(cos_t, f32, "rope_pos cos"); _chk(sin_t, f32, "rope_pos sin")
    M = buf.shape[0]
    if pos.numel() != M or not pos.is_contiguous():
        raise _lib.DalmB200Error(f"rope_pos: need one contiguous position id per row ({pos.numel()} for {M} rows)")
    if buf.dim() != 2 or col0 < 0 or col0 + nheads * D > buf.shape[1]:
        raise _lib.DalmB200Error(f"rope_pos: heads [{col0}, {col0} + {nheads} x {D}) outside buf {tuple(buf.shape)}")
    if cos_t.dim() != 2 or cos_t.shape[1] != D // 2 or sin_t.shape != cos_t.shape or not cos_t.is_contiguous() \
            or not sin_t.is_contiguous():
        raise _lib.DalmB200Error(f"rope_pos: cos / sin must be dense fp32 [T, {D // 2}], got {tuple(cos_t.shape)} strides "
                                 f"{cos_t.stride()} / {tuple(sin_t.shape)} strides {sin_t.stride()}")
    _lib.call("dalm_b200_rope_pos", _p(buf), _ld(buf), col0, nheads, D, _p(cos_t), _p(sin_t), _p(pos), M, cos_t.shape[0], _stream())
    return buf


def _cur_arg(cur, B: int, what: str):
    """host column (int) or per-row device columns (int32 [B] tensor: CUDA-graph mode) -> (host int, device pointer)"""
    if torch.is_tensor(cur):
        if cur.dtype != torch.int32 or not cur.is_cuda or cur.numel() != B or not cur.is_contiguous():
            raise _lib.DalmB200Error(f"{what}: device columns must be a contiguous int32 CUDA tensor with one entry per row")
        return 0, _p(cur)
    return int(cur), None


def attention_decode(qkv, q_col: int, k_col: int, v_col: int, cache_k, cache_v, mask, cur, Hq: int, Hkv: int, D: int,
                     out=None, scale: Optional[float] = None, window: int = 0):
    """qkv bf16 [B, >=v_col+Hkv*D] (current token of every sequence); cache_k / cache_v bf16 [B, T, Hkv*D]; mask int64 [B, T].
    Appends the token's K / V at column `cur` (int, or int32 [B] device tensor) and returns the attention output bf16 [B, Hq*D].
    window > 0: only columns t > cur - window are visible (0 = no window)."""
    _chk(qkv, bf16, "attention_decode qkv"); _chk(cache_k, bf16, "cache_k"); _chk(cache_v, bf16, "cache_v"); _chk(mask, i64, "mask")
    B, T = cache_k.shape[0], cache_k.shape[1]
    if cache_k.shape != cache_v.shape or cache_k.stride() != cache_v.stride() or cache_k.dim() != 3 or mask.shape[0] != B or mask.shape[1] < T:
        raise _lib.DalmB200Error("attention_decode: cache_k / cache_v / mask shapes disagree")
    if qkv.shape[0] != B:
        raise _lib.DalmB200Error("attention_decode: one qkv row per cached sequence")
    for c, n, what in ((q_col, Hq, "q"), (k_col, Hkv, "k"), (v_col, Hkv, "v")):
        if c < 0 or c + n * D > qkv.shape[1]:
            raise _lib.DalmB200Error(f"attention_decode: {what} columns [{c}, {c} + {n} x {D}) outside qkv {tuple(qkv.shape)}")
    if cache_k.shape[2] < Hkv * D:
        raise _lib.DalmB200Error(f"attention_decode: cache rows {tuple(cache_k.shape)} narrower than {Hkv} x {D}")
    if out is None:
        out = torch.empty(B, Hq * D, dtype=bf16, device=qkv.device)
    _chk(out, bf16, "attention_decode out")
    if out.dim() != 2 or out.shape[0] != B or out.shape[1] < Hq * D:
        raise _lib.DalmB200Error(f"attention_decode: out {tuple(out.shape)} must be bf16 [{B}, >= {Hq * D}]")
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    cur_host, cur_dev = _cur_arg(cur, B, "attention_decode")
    _lib.call("dalm_b200_attention_decode", _p(qkv), _ld(qkv), q_col, k_col, v_col, _p(cache_k), _p(cache_v),
              cache_k.stride(0), cache_k.stride(1), _p(mask), mask.stride(0), _p(out), _ld(out), B, Hq, Hkv, D, cur_host, cur_dev,
              T, float(scale), int(window), _stream())
    return out


def greedy_step_(logits, V: int, eos_ids, pad_id: int, unfinished, tokens, mask, col, next_ids, pos, alive) -> None:
    """one greedy-search step on device state (see include/dalm_b200.h): logits bf16 [B, >=V]; eos_ids int64 [n] or None;
    unfinished int32 [B]; tokens / mask int64 [B, T]; next_ids / pos int64 [B]; alive int32 [T] (zeroed by the caller).
    col: the column to write (int), or the int32 [B] device tensor holding each row's CURRENT column (the kernel writes
    column + 1 and advances it: CUDA-graph mode)."""
    _lib.call("dalm_b200_greedy_step", *_step_args("greedy_step", logits, V, eos_ids, pad_id, unfinished, tokens, mask, col,
                                                   next_ids, pos, alive), _stream())


def _step_args(what: str, logits, V: int, eos_ids, pad_id: int, unfinished, tokens, mask, col, next_ids, pos, alive) -> tuple:
    """checks and C arguments shared by greedy_step_ and sample_step_ (everything up to `alive`)"""
    _chk(logits, bf16, f"{what} logits"); _chk(tokens, i64, "tokens"); _chk(mask, i64, "mask")
    _chk(next_ids, i64, "next_ids"); _chk(pos, i64, "pos")
    T = tokens.shape[1]
    if unfinished.dtype != torch.int32 or alive.dtype != torch.int32 or alive.numel() < T or mask.shape[1] < T:
        raise _lib.DalmB200Error(f"{what}: unfinished / alive must be int32, alive and mask as long as the token buffer")
    if eos_ids is not None:
        _chk(eos_ids, i64, "eos_ids")
    B = logits.shape[0]
    col_host, cur_dev = _cur_arg(col, B, what)
    return (_p(logits), _ld(logits), B, int(V), _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(), int(pad_id),
            _p(unfinished), _p(tokens), tokens.stride(0), _p(mask), mask.stride(0), col_host, cur_dev, T, _p(next_ids), _p(pos),
            _p(alive))


def sample_step_(logits, V: int, eos_ids, pad_id: int, unfinished, tokens, mask, col, next_ids, pos, alive, *,
                 temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
                 u: Optional[torch.Tensor] = None, scores_out: Optional[torch.Tensor] = None) -> None:
    """one sampling step on device state: greedy_step_'s arguments and bookkeeping, the token drawn from HF's warper stack
    temperature -> top-k (0 = off) -> top-p (1 = off) with a Philox draw keyed by `seed` and (column, row); see
    include/dalm_b200.h. Test hooks: u fp64 [B] replaces the draw; scores_out fp32 [B, >=V] with the logits' row stride
    receives the warped scores (-inf where removed)."""
    args = _step_args("sample_step", logits, V, eos_ids, pad_id, unfinished, tokens, mask, col, next_ids, pos, alive)
    B = logits.shape[0]
    if u is not None:
        _chk(u, torch.float64, "sample_step u")
        if u.numel() != B or not u.is_contiguous():
            raise _lib.DalmB200Error(f"sample_step: u needs one contiguous fp64 value per row ({u.numel()} for {B} rows)")
    if scores_out is not None:
        _chk(scores_out, f32, "sample_step scores_out")
        if scores_out.shape[0] != B or scores_out.shape[1] < V or _ld(scores_out) != _ld(logits):
            raise _lib.DalmB200Error("sample_step: scores_out must be fp32 [B, >=V] with the logits' row stride")
    _lib.call("dalm_b200_sample_step", *args, float(temperature), int(top_k), float(top_p), int(seed) & (2**64 - 1), _p(u),
              _p(scores_out), _stream())


# ----------------------------------------------------------------------------------------------------------------
# routed mixture-of-experts MLP (Qwen3-MoE)
# ----------------------------------------------------------------------------------------------------------------
i32 = torch.int32


def moe_tiles(pairs: int, E: int) -> int:
    """static bound of 128-row M tiles over `pairs` (token, slot) pairs whose E expert segments are each padded to the tile"""
    return (pairs + 127 * E + 127) // 128


def _dense_experts(w: torch.Tensor, name: str) -> None:
    _chk(w, bf16, name)
    if w.dim() != 3 or not w.is_contiguous():
        raise _lib.DalmB200Error(f"{name}: expected a dense bf16 [E, rows, cols] stack, got shape {tuple(w.shape)} strides {w.stride()}")


def gemm_grouped(a: torch.Tensor, w: torch.Tensor, tile_expert: torch.Tensor, live: torch.Tensor, out: Optional[torch.Tensor] = None,
                 *, layout: int = 0, swiglu: bool = False, act: Optional[torch.Tensor] = None, max_ctas: int = 0):
    """grouped GEMM over experts: row block m // 128 of `a` (bf16 [rows, K], rows = 128 n_tiles) is multiplied by expert
    e = tile_expert[m // 128]: layout 0 out = a @ w[e]^T (w [E, N, K]), layout 1 out = a @ w[e] (w [E, K, N]). Only the first
    live[0] tiles are computed; the rest of `out` is left as it was. swiglu: w[e] holds interleaved gate / up rows
    (`interleave_gate_up`) -> (gu [rows, N], act [rows, N / 2] = silu(gate) * up)."""
    _chk(a, bf16, "gemm_grouped a")
    _dense_experts(w, "gemm_grouped w")
    _vec(live, i32, "gemm_grouped live", 1)
    M, K = a.shape
    E = w.shape[0]
    N = w.shape[1] if layout == 0 else w.shape[2]
    if (w.shape[2] if layout == 0 else w.shape[1]) != K:
        raise _lib.DalmB200Error(f"gemm_grouped: a is [{M}, {K}] but w is {tuple(w.shape)} (layout {layout})")
    _vec(tile_expert, i32, "gemm_grouped tile_expert", (M + 127) // 128)
    if out is None:
        out = torch.empty(M, N, dtype=bf16, device=a.device)
    _bf16_rows(out, "gemm_grouped out", M, N)
    if swiglu and act is None:
        act = torch.empty(M, N // 2, dtype=bf16, device=a.device)
    if act is not None:
        _bf16_rows(act, "gemm_grouped act", M, N // 2)
    if max_ctas == 0 and GEMM_MAX_CTAS:
        max_ctas = GEMM_MAX_CTAS
    _lib.call("dalm_b200_gemm_bf16_grouped", int(layout), 1 if swiglu else 0, _p(a), _ld(a), _p(w), E, _p(out), _ld(out),
              _p(act), _ld(act) if act is not None else 0, M, N, K, _p(tile_expert), _p(live), int(max_ctas), _stream())
    return (out, act) if swiglu else out


class MoeRouting:
    """where each (token, slot) pair of a routed batch sits in the expert-sorted, tile-padded rows (see moe_permute)"""
    __slots__ = ("M", "k", "E", "n_tiles", "counts", "seg_off", "tile_expert", "live", "pair_row", "row_pair", "chunk_counts")

    def __init__(self, M: int, k: int, E: int, device, n_tiles: Optional[int] = None):
        P = M * k
        self.M, self.k, self.E = M, k, E
        self.n_tiles = moe_tiles(P, E) if n_tiles is None else n_tiles
        z = lambda n: torch.empty(n, dtype=i32, device=device)
        self.counts, self.seg_off, self.tile_expert, self.live = z(E), z(E + 1), z(self.n_tiles), z(1)
        self.pair_row, self.row_pair = z(P), z(128 * self.n_tiles)
        self.chunk_counts = z(-(-P // 1024) * E)

    @property
    def rows(self) -> int:
        return 128 * self.n_tiles


def moe_router(logits: torch.Tensor, k: int, norm_topk: bool, ids: Optional[torch.Tensor] = None, w: Optional[torch.Tensor] = None):
    """fp32 router logits [M, E] -> (ids int32 [M, k], weights fp32 [M, k]): softmax, top-k, renormalised when norm_topk"""
    _chk(logits, f32, "moe_router logits")
    M, E = logits.shape
    ids = torch.empty(M, k, dtype=i32, device=logits.device) if ids is None else ids
    w = torch.empty(M, k, dtype=f32, device=logits.device) if w is None else w
    _vec(ids, i32, "moe_router ids", M * k); _vec(w, f32, "moe_router w", M * k)
    _lib.call("dalm_b200_moe_router", _p(logits), _ld(logits), M, E, int(k), int(bool(norm_topk)), _p(ids), _p(w), _stream())
    return ids, w


def moe_router_bwd(logits: torch.Tensor, ids: torch.Tensor, w: torch.Tensor, dw: torch.Tensor, norm_topk: bool,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d(router logits) as bf16 [M, E] (the operand of dh += dlogits @ W_gate) from d(routing weights) fp32 [M, k]"""
    _chk(logits, f32, "moe_router_bwd logits")
    M, E = logits.shape
    k = ids.shape[-1]
    for t, dt, nm in ((ids, i32, "ids"), (w, f32, "w"), (dw, f32, "dw")):
        _vec(t, dt, f"moe_router_bwd {nm}", M * k)
    out = torch.empty(M, E, dtype=bf16, device=logits.device) if out is None else out
    _bf16_rows(out, "moe_router_bwd out", M, E)
    _lib.call("dalm_b200_moe_router_bwd", _p(logits), _ld(logits), _p(ids), _p(w), _p(dw), M, E, int(k), int(bool(norm_topk)),
              _p(out), _ld(out), _stream())
    return out


def moe_permute(ids: torch.Tensor, E: int, routing: Optional[MoeRouting] = None) -> MoeRouting:
    """expert-sorted, tile-padded placement of the pairs of ids (int32 [M, k]); `routing` is reused when given (a captured
    step keeps its buffers)"""
    M, k = ids.shape
    r = MoeRouting(M, k, E, ids.device) if routing is None else routing
    if (r.M, r.k, r.E) != (M, k, E):
        raise _lib.DalmB200Error(f"moe_permute: routing buffers are for M={r.M} k={r.k} E={r.E}, not M={M} k={k} E={E}")
    _vec(ids, i32, "moe_permute ids", M * k)
    _lib.call("dalm_b200_moe_permute", _p(ids), M * k, E, r.n_tiles, _p(r.chunk_counts), _p(r.counts), _p(r.seg_off),
              _p(r.tile_expert), _p(r.live), _p(r.pair_row), _p(r.row_pair), _stream())
    return r


def moe_gather(x: torch.Tensor, r: MoeRouting, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """rows [r.rows, H] (bf16): each live row holds its token's row of x (bf16 or fp32), padding rows 0"""
    if x.dtype not in (bf16, f32):
        raise _lib.DalmB200Error("moe_gather: x must be bf16 or fp32")
    _chk(x, x.dtype, "moe_gather x")
    H = x.shape[1]
    out = torch.empty(r.rows, H, dtype=bf16, device=x.device) if out is None else out
    _bf16_rows(out, "moe_gather out", r.rows, H)
    _lib.call("dalm_b200_moe_gather", _p(x), _ld(x), 1 if x.dtype == f32 else 0, H, _p(r.row_pair), r.k, _p(r.live), r.rows,
              _p(out), _ld(out), _stream())
    return out


def moe_combine(y: torch.Tensor, r: MoeRouting, w: Optional[torch.Tensor], resid: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, out_dtype=f32) -> torch.Tensor:
    """out[t] = resid[t] + sum_s w[t, s] y[row(t, s)] (fp32 sums, slots in order); w None = weights of 1. resid / out: fp32
    or bf16 [M, H] of one dtype; resid may be out itself."""
    _chk(y, bf16, "moe_combine y")
    H = y.shape[1]
    if out is None:
        out = torch.empty(r.M, H, dtype=resid.dtype if resid is not None else out_dtype, device=y.device)
    if out.dtype not in (bf16, f32) or (resid is not None and resid.dtype != out.dtype):
        raise _lib.DalmB200Error("moe_combine: out and resid must both be bf16 or both fp32")
    _chk(out, out.dtype, "moe_combine out")
    if resid is not None:
        _chk(resid, resid.dtype, "moe_combine resid")
    if w is not None:
        _vec(w, f32, "moe_combine w", r.M * r.k)
    _lib.call("dalm_b200_moe_combine", _p(y), _ld(y), _p(r.pair_row), _p(w), r.M, r.k, H, _p(resid),
              _ld(resid) if resid is not None else 0, _p(out), _ld(out), 1 if out.dtype == f32 else 0, _stream())
    return out


def moe_down_bwd(da: torch.Tensor, act: torch.Tensor, r: MoeRouting, w: torch.Tensor, d_act: Optional[torch.Tensor] = None):
    """-> (dw fp32 [M, k] = <da[row], act[row]>, d_act bf16 [rows, I] = w da[row] on the live rows)"""
    _chk(da, bf16, "moe_down_bwd da"); _chk(act, bf16, "moe_down_bwd act")
    _vec(w, f32, "moe_down_bwd w", r.M * r.k)
    I = act.shape[1]
    d_act = torch.empty(r.rows, I, dtype=bf16, device=da.device) if d_act is None else d_act
    _bf16_rows(d_act, "moe_down_bwd d_act", r.rows, I)
    dw = torch.empty(r.M, r.k, dtype=f32, device=da.device)
    _lib.call("dalm_b200_moe_down_bwd", _p(da), _ld(da), _p(act), _ld(act), _p(r.pair_row), _p(w), r.M * r.k, I, _p(dw),
              _p(d_act), _ld(d_act), _stream())
    return dw, d_act
