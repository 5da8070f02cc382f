"""The dense GEMMs at the shapes the engines issue, element by element, and the wrapper checks in front of them.

The element-wise GEMM tests elsewhere stay near the tile edges (K of a few hundred). Here every forward, dgrad and wgrad
GEMM of the bench configs runs at its full K: the Llama-family decoders of cfg-3 (M = 18 x 256 = 4608 token rows), the
bge-large encoder of cfg-3 (18 x 128 = 2304 passages, 18 x 50 = 900 queries) and cfg-2 (150 x 128 = 19200) and the
Falcon-7B of cfg-5 (18 x 2048 = 36864). Each shape also runs at a ragged M (a partial last m-tile at full K).

Operands are integers in [-2, 2], so every partial sum is an integer of magnitude at most 4K; the largest contraction, the
Falcon wgrad over 36864 token rows, stays at 147456 < 2^24. Every fp32 sum is therefore exact in any order: fp32 outputs
must equal the reference bit for bit and bf16 outputs its round-to-nearest-even. The reference is a torch fp32 matmul
with TF32 off (exact for the same reason), computed and compared in row chunks; one chunk per shape is re-checked against
fp64, so the reference itself is tested. The fused epilogues (RoPE, q/k norm, SwiGLU, GELU, dropout) are held to the
bounds the tile-edge tests state. Every operand is a NaN-padded view and every output a guarded one (exact_helpers).

The decode GEMM runs at every M from 1 to 16 at each family's decode projections, across the per-warp ring's wrap, and
on both sides of `gemm_rows`' 16-row switch.
"""
import zlib
from collections import namedtuple

import pytest
import torch

from exact_helpers import (EPS, PAD_C, PAD_R, Guarded, _expect_close, _expect_equal, _gelu64, _gelu_grad64, _norm_w,
                           _pick_block_n, _ref_norm_rope, _tables, _ulp_bf16, _ulp_f32, dev, ops)  # noqa: F401

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
H100_SMS = 132                                   # H100 SXM: the SM count the chunked head's row split is derived for
HEAD_BUDGET, FULL_HEAD_BUDGET = 24 << 20, 512 << 20     # engine/head.py: L2_BUDGET (frozen head), FULL_BUDGET (trained head)
CHUNK_ELEMS = 64 << 20                           # reference / comparison chunk: rows x N at most this many elements
DG_STAGES = 6                                    # decode.cu: k-chunks in flight per lane of the decode GEMM


@pytest.fixture(scope="module")
def exact_fp32():
    """fp32 matmuls without TF32 (the integer reference is exact only in full fp32); the previous setting comes back"""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.get_float32_matmul_precision()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev[0]
    torch.set_float32_matmul_precision(prev[1])


# ----------------------------------------------------------------------------------------------------------------
# 1. the shape table, from the engines and the public config fields
# ----------------------------------------------------------------------------------------------------------------
# (model, projection, entry point, layout, M, N, K, epilogue). Entry points: gemm, wgrad (ops.wgrad_: layout 2, M and N the
# weight's [out, in], K the token rows), swiglu, gelu (gemm_gelu), rope (gemm_rope). Epilogues: bf16 / f32 plain output,
# +bias, +resid (fp32), +drop (dropout 0.1 before the residual), act1 (GELU), act2 (times gelu'(bf16 pre)), inplace (bf16
# out is resid), acc (wgrad accumulate: fp32 out is resid), rope C (RoPE on the first C columns), norm C/Q (Qwen3 q/k RMSNorm
# then RoPE on C columns, Q query heads, with pre_out / rstd_out).
Row = namedtuple("Row", "model proj entry layout M N K epi")

# public config.json fields of the checkpoints
LLAMA2_7B = dict(hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_key_value_heads=32, vocab_size=32000)
LLAMA3_8B = dict(hidden_size=4096, intermediate_size=14336, num_attention_heads=32, num_key_value_heads=8, vocab_size=128256)
QWEN25_7B = dict(hidden_size=3584, intermediate_size=18944, num_attention_heads=28, num_key_value_heads=4, vocab_size=152064)
QWEN3_8B = dict(hidden_size=4096, intermediate_size=12288, num_attention_heads=32, num_key_value_heads=8, vocab_size=151936)
OLMO2_7B = dict(hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_key_value_heads=32, vocab_size=100352)
FALCON_7B = dict(hidden_size=4544, num_attention_heads=71, vocab_size=65024)          # multi_query, ffn 4 x hidden
BGE_LARGE = dict(hidden_size=1024, intermediate_size=4096, num_attention_heads=16)
R = 8                                            # LoRA rank: K-augmented QKV operands, 2r in llama.py, 3r in bert.py


def _head_rows(M, V, budget):
    """rows of one chunk of the chunked lm_head (head.py:51) on an H100, and of the last one"""
    rows = ops_mod().head_chunk_rows(M, (V + 7) // 8 * 8, budget, sms=H100_SMS)
    return rows, M - (M - 1) // rows * rows


def ops_mod():
    from dalm_b200 import ops as o
    return o


def _decoder(model, c, M, qkv, peft=True, full=False, post_norm=False):
    """the GEMMs of engine/llama.py at M token rows, head_dim 128. qkv: "rope", "rope+bias" (Qwen2), "norm" (Qwen3) or
    "plain" (OLMo 2: full-width q/k norm after the GEMM)"""
    H, F, nh, nkv, V = (c[k] for k in ("hidden_size", "intermediate_size", "num_attention_heads", "num_key_value_heads",
                                       "vocab_size"))
    Nqkv, rope_cols, Vp = (nh + 2 * nkv) * 128, (nh + nkv) * 128, (V + 7) // 8 * 8
    Ka = H + 2 * R if peft else H                                # llama.py:118 Ra = 2r; _aug_buf appends it to h1
    rows = []
    q = {"rope": ("rope", f"rope {rope_cols}"), "rope+bias": ("rope", f"rope {rope_cols}+bias"),
         "norm": ("rope", f"norm {rope_cols}/{nh}"), "plain": ("gemm", "bf16")}[qkv]
    rows.append(Row(model, "qkv", q[0], 0, M, Nqkv, Ka, q[1]))  # llama.py:527 gemm_rope(h1_aug, Wqkv_aug) / :521 fullnorm
    if post_norm:
        rows.append(Row(model, "o", "gemm", 0, M, H, H, "bf16"))                      # llama.py:544 yo = gemm(att, Wo)
    else:
        rows.append(Row(model, "o", "gemm", 0, M, H, H, "f32+resid"))                 # llama.py:548 x + o_proj(att)
    if peft:
        rows.append(Row(model, "gate|up", "swiglu", 0, M, 2 * F, H, "-"))             # llama.py:556 gemm_swiglu(h2, Wgu)
    else:
        rows.append(Row(model, "gate|up", "gemm", 0, M, 2 * F, H, "bf16"))            # llama.py:558 (full: HF order)
    rows.append(Row(model, "down", "gemm", 0, M, H, F, "bf16" if post_norm else "f32+resid"))   # llama.py:561 / :565
    if peft:
        hr, _ = _head_rows(M, V, HEAD_BUDGET)
        rows.append(Row(model, "lm_head", "gemm", 0, hr, Vp, H, "bf16"))             # head.py:58 gemm(hf[r0:r0+n], w_head)
        rows.append(Row(model, "lm_head dgrad", "gemm", 0, hr, H, Vp, "bf16"))       # head.py:65 gemm(lg, w_headT)
        # dgrads against the resident transposes (llama.py:296 _dgrad): d act, d h2, d att, d h1 (base path, :748)
        rows.append(Row(model, "down dgrad", "gemm", 0, M, F, H, "bf16"))             # llama.py:685
        rows.append(Row(model, "gate|up dgrad", "gemm", 0, M, H, 2 * F, "bf16"))     # llama.py:689
        rows.append(Row(model, "o dgrad", "gemm", 0, M, nh * 128, H, "bf16"))        # llama.py:702
        rows.append(Row(model, "qkv dgrad", "gemm", 0, M, H, Nqkv, "bf16"))          # llama.py:748 dqkv[:, :Nqkv] @ WqkvT
        rows.append(Row(model, "qkv dgrad+A", "gemm", 0, M, H, Nqkv + 2 * R, "bf16"))   # llama.py:746 LoRA A folded into K
    if full:
        # full fine-tuning (llama.py:295: layout 1 against W[out,in]); weight gradients contract over the M token rows
        rows.append(Row(model, "down dgrad", "gemm", 1, M, F, H, "bf16"))             # llama.py:685
        rows.append(Row(model, "gate|up dgrad", "gemm", 1, M, H, 2 * F, "bf16"))     # llama.py:689
        rows.append(Row(model, "o dgrad", "gemm", 1, M, nh * 128, H, "bf16"))        # llama.py:702
        rows.append(Row(model, "qkv dgrad", "gemm", 1, M, H, Nqkv, "bf16"))          # llama.py:721
        rows.append(Row(model, "lm_head dgrad", "gemm", 1, M, H, Vp, "bf16"))        # llama.py:660
        rows.append(Row(model, "down wgrad", "wgrad", 2, H, F, M, "acc"))             # llama.py:684 wgrad_(dx16, act)
        rows.append(Row(model, "gate|up wgrad", "wgrad", 2, 2 * F, H, M, "f32"))     # llama.py:688 wgrad_(gu, h2)
        rows.append(Row(model, "o wgrad", "wgrad", 2, H, nh * 128, M, "acc"))        # llama.py:699 wgrad_(dmid16, att)
        rows.append(Row(model, "qkv wgrad", "wgrad", 2, Nqkv, H, M, "f32"))          # llama.py:718 wgrad_(dqkv, h1[:, :H])
        rows.append(Row(model, "lm_head wgrad", "wgrad", 2, Vp, H, M, "acc"))        # llama.py:658 wgrad_(dl2, hf)
    return rows


def _falcon(model, c, M):
    """engine/falcon.py, cfg-5: Falcon-7B fully fine-tuned, multi-query attention (one k and one v head of 64)"""
    H, nh, V = c["hidden_size"], c["num_attention_heads"], c["vocab_size"]
    F, hd, Vp = 4 * H, H // nh, (V + 7) // 8 * 8
    Nqkv = nh * hd + 2 * hd
    hr, _ = _head_rows(M, V, FULL_HEAD_BUDGET)
    return [
        Row(model, "qkv", "gemm", 0, M, Nqkv, H, "bf16"),                 # falcon.py:172 gemm(h, Wqkv)
        Row(model, "dense", "gemm", 0, M, H, H, "f32+resid"),             # falcon.py:181 gemm(att, Wd, f32, resid=x)
        Row(model, "W1", "gelu", 0, M, F, H, "-"),                        # falcon.py:184 gemm_gelu(h, W1) (recompute)
        Row(model, "W1 eval", "gemm", 0, M, F, H, "act1"),                # falcon.py:189 gemm(h, W1, act=1)
        Row(model, "W2", "gemm", 0, M, H, F, "f32+resid"),                # falcon.py:190 gemm(h4, W2, f32, resid=t)
        Row(model, "lm_head", "gemm", 0, hr, Vp, H, "bf16"),              # head.py:58
        Row(model, "lm_head dgrad", "gemm", 1, hr, H, Vp, "bf16"),        # head.py:67 gemm(lg, w_head, layout=1)
        Row(model, "lm_head wgrad", "wgrad", 2, Vp, H, hr, "acc"),        # falcon.py:271 (head.py:63) wgrad_(lg, hf rows)
        Row(model, "W2 wgrad", "wgrad", 2, H, F, M, "acc"),               # falcon.py:203 wgrad_(dx16, h4)
        Row(model, "W2 dgrad", "gemm", 1, M, F, H, "act2"),               # falcon.py:205 act=2, resid=pre
        Row(model, "W1 wgrad", "wgrad", 2, F, H, M, "f32"),               # falcon.py:209 wgrad_(dpre, h)
        Row(model, "W1 dgrad", "gemm", 1, M, H, F, "bf16"),               # falcon.py:210
        Row(model, "dense wgrad", "wgrad", 2, H, H, M, "acc"),            # falcon.py:212
        Row(model, "dense dgrad", "gemm", 1, M, H, H, "bf16"),            # falcon.py:213
        Row(model, "qkv wgrad", "wgrad", 2, Nqkv, H, M, "f32"),           # falcon.py:219
        Row(model, "qkv dgrad", "gemm", 1, M, H, Nqkv, "inplace"),        # falcon.py:220 out=dh, resid=dh
    ]


def _bert(model, c, M):
    """engine/bert.py with LoRA on q|k|v (Ra = 3r, bert.py:95), frozen base: dgrads against the transposes (bert.py:255).
    BERT keeps GELU out of the GEMM (fuse_gelu(1024) is False)"""
    H, F = c["hidden_size"], c["intermediate_size"]
    return [
        Row(model, "qkv", "gemm", 0, M, 3 * H, H + 3 * R, "bf16+bias"),   # bert.py:397 gemm(x_aug, Wqkv_aug, bias)
        Row(model, "Wo", "gemm", 0, M, H, H, "f32+bias+resid+drop"),      # bert.py:406
        Row(model, "Wi", "gemm", 0, M, F, H, "bf16+bias"),                # bert.py:413
        Row(model, "Wo2", "gemm", 0, M, H, F, "f32+bias+resid+drop"),     # bert.py:415
        Row(model, "Wo2 dgrad", "gemm", 0, M, F, H, "bf16"),              # bert.py:468
        Row(model, "Wi dgrad", "gemm", 0, M, H, F, "bf16"),               # bert.py:473
        Row(model, "Wo dgrad", "gemm", 0, M, H, H, "bf16"),               # bert.py:482
        Row(model, "qkv dgrad", "gemm", 0, M, H, 3 * H, "bf16"),          # bert.py:515 base path
        Row(model, "qkv dgrad+A", "gemm", 0, M, H, 3 * H + 3 * R, "bf16"),   # bert.py:513 LoRA A folded into K
    ]


def _with_ragged(rows, ragged):
    """each row, then the same row at the ragged token count (M, or K for a wgrad) given for its token count"""
    out = []
    for r in rows:
        out.append(r)
        t = r.K if r.entry == "wgrad" else r.M
        if t in ragged:
            out.append(r._replace(K=ragged[t]) if r.entry == "wgrad" else r._replace(M=ragged[t]))
    return out


def _ragged_head(M, V, budget):
    rows, last = _head_rows(M, V, budget)
    return {rows: last if last != rows else rows - 18}


def _table():
    t = []
    t += _with_ragged(_decoder("llama2-7b", LLAMA2_7B, 4608, "rope"), {4608: 4590, **_ragged_head(4608, 32000, HEAD_BUDGET)})
    t += _with_ragged(_decoder("llama2-7b-full", LLAMA2_7B, 4608, "rope", peft=False, full=True), {4608: 4590})
    t += _with_ragged(_decoder("llama3-8b", LLAMA3_8B, 4608, "rope"), {4608: 4590, 128: 110})
    t += _with_ragged(_decoder("qwen2.5-7b", QWEN25_7B, 4608, "rope+bias"), {4608: 4590, 128: 110})
    t += _with_ragged(_decoder("qwen3-8b", QWEN3_8B, 4608, "norm"), {4608: 4590, 128: 110})
    t += _with_ragged(_decoder("olmo2-7b", OLMO2_7B, 4608, "plain", post_norm=True), {4608: 4590, 128: 110})
    t += _with_ragged(_falcon("falcon-7b", FALCON_7B, 36864), {36864: 36850, **_ragged_head(36864, 65024, FULL_HEAD_BUDGET)})
    t += _with_ragged(_bert("bge-large", BGE_LARGE, 2304), {2304: 900})
    t += [r._replace(M=19200) for r in _bert("bge-large", BGE_LARGE, 2304)[:4]]      # cfg-2: 150 x 128 passage rows
    return t


TABLE = _table()


def _widths(r):
    """the dispatcher's choice, then (plain kernels, first token count of the row) every other tile width N allows"""
    if r.entry not in ("gemm", "wgrad"):
        return (0,)
    ws = [bn for bn in (64, 128, 256) if r.N >= bn]
    if r.layout == 0:
        ws += [bn for bn in (2128, 2256) if r.N >= bn % 1000]
    return (0, *ws)


def _first_of_shape(table):
    seen, first = set(), []
    for r in table:
        key = (r.model, r.proj, r.layout, r.N)
        first.append(key not in seen)
        seen.add(key)
    return first


def _params():
    out = []
    for r, first in zip(TABLE, _first_of_shape(TABLE)):
        ws = _widths(r) if first else (0,)
        out.append(pytest.param(r, ws, id=f"{r.model}-{r.proj}-L{r.layout}-M{r.M}-N{r.N}-K{r.K}".replace(" ", "_").replace("|", "")))
    return out


def test_table_rederives():
    """CPU: the table covers every family, the token counts follow the bench configs, and every shape meets the kernels'
    alignment rules"""
    models = {r.model for r in TABLE}
    assert {"llama2-7b", "llama3-8b", "qwen2.5-7b", "qwen3-8b", "olmo2-7b", "falcon-7b", "bge-large"} <= models
    assert _head_rows(4608, 32000, HEAD_BUDGET) == (384, 384)
    assert _head_rows(36864, 65024, FULL_HEAD_BUDGET) == (3456, 2304)
    for r in TABLE:
        assert r.N % 8 == 0 and (r.K % 8 == 0 or r.entry == "wgrad") and (r.M % 8 == 0 or r.entry != "wgrad"), r
        assert 4 * r.K < 2 ** 24, r                               # |partial sums| <= 4K: exact in fp32
    ks = {(r.model, r.proj): r.K for r in TABLE if r.layout == 0}
    assert ks[("llama2-7b", "qkv")] == 4112 and ks[("qwen2.5-7b", "qkv")] == 3600 and ks[("bge-large", "qkv")] == 1048
    assert max(r.K for r in TABLE if r.entry == "wgrad") == 36864


# ----------------------------------------------------------------------------------------------------------------
# 2. the wgmma GEMMs at those shapes
# ----------------------------------------------------------------------------------------------------------------
def _dev_ints(rows, cols, g, dev, dtype=bf16, hi=2, pad_c=PAD_C):
    """integers in [-hi, hi] drawn on the device into a view of a NaN buffer (NaN columns right, NaN rows below)"""
    buf = torch.full((rows + PAD_R, cols + pad_c), float("nan"), dtype=dtype, device=dev)
    v = buf[:rows, :cols]
    v.copy_(torch.randint(-hi, hi + 1, (rows, cols), generator=g, device=dev, dtype=torch.int8 if hi < 128 else torch.int16))
    return v


def _dev_vec(n, g, dev, hi=4096):
    buf = torch.full((n + 256,), float("nan"), dtype=f32, device=dev)
    buf[:n].copy_(torch.randint(-hi, hi + 1, (n,), generator=g, device=dev, dtype=torch.int16))
    return buf[:n]


class _Case:
    """the operands, extra inputs and output views of one table row at one token count (drawn once, reused per width)"""

    def __init__(self, r, dev, seed):
        self.r, self.dev = r, dev
        g = torch.Generator(device=dev).manual_seed(seed)
        M, N, K = r.M, r.N, r.K
        ash, bsh = {0: ((M, K), (N, K)), 1: ((M, K), (K, N)), 2: ((K, M), (K, N))}[r.layout]
        self.a, self.b = _dev_ints(*ash, g, dev), _dev_ints(*bsh, g, dev)
        e = r.epi
        self.bias = _dev_vec(N, g, dev) if "bias" in e else None
        self.resid = None
        if "resid" in e or e == "acc":
            self.resid = _dev_ints(M, N, g, dev, f32, 2048)
        elif e == "inplace":
            self.resid = _dev_ints(M, N, g, dev, bf16, 256)
        elif e == "act2":
            pre = torch.full((M + PAD_R, N + PAD_C), float("nan"), dtype=bf16, device=dev)
            pre[:M, :N].copy_(torch.randn(M, N, generator=g, device=dev) * 2)
            self.resid = pre[:M, :N]
        self.drop = ops_mod().Drop(0.1, seed=0xD20 + seed, stream=7) if "drop" in e else None
        if r.entry == "rope":
            cols = int(e.split()[1].split("/")[0].split("+")[0])
            self.rope_cols, self.L = cols, 256                       # cfg-3 generator rows: position = row % 256
            self.cos, self.sin = _tables(dev, self.L)
            if e.startswith("norm"):
                gh = torch.Generator().manual_seed(seed)
                self.nq = int(e.split("/")[1])
                self.wq, self.wk = _norm_w(gh, dev), _norm_w(gh, dev)
            else:
                self.nq = None
        self.odt = f32 if (e.startswith("f32") or r.entry == "wgrad") else bf16

    def run(self, bn):
        """one launch at tile width bn (0: the dispatcher's choice) into fresh guarded outputs -> dict of them"""
        r, o, dev, M, N = self.r, ops_mod(), self.dev, self.r.M, self.r.N
        outs = {}
        if r.entry == "wgrad":
            gw = outs["out"] = Guarded(M, N, f32, dev, init=self.resid if r.epi == "acc" else None)
            if bn == 0:                                              # the engines' entry point
                o.wgrad_(self.a, self.b, gw.view, accumulate=r.epi == "acc")
            else:                                                    # the launch wgrad_ makes, at a forced tile width
                o.gemm(self.a, self.b, out=gw.view, layout=2, resid=gw.view if r.epi == "acc" else None, block_n=bn)
        elif r.entry == "gemm":
            inplace = r.epi == "inplace"
            outs["out"] = Guarded(M, N, self.odt, dev, init=self.resid if inplace else None)
            act = 1 if r.epi == "act1" else (2 if r.epi == "act2" else 0)
            o.gemm(self.a, self.b, out=outs["out"].view, out_dtype=self.odt, bias=self.bias, act=act,
                   resid=outs["out"].view if inplace else self.resid, block_n=bn, drop=self.drop, layout=r.layout)
        elif r.entry == "swiglu":
            outs["out"], outs["act"] = Guarded(M, N, bf16, dev), Guarded(M, N // 2, bf16, dev)
            o.gemm_swiglu(self.a, self.b, gu=outs["out"].view, act=outs["act"].view)
        elif r.entry == "gelu":
            outs["out"], outs["act"] = Guarded(M, N, bf16, dev), Guarded(M, N, bf16, dev)
            o.gemm_gelu(self.a, self.b, bias=self.bias, pre=outs["out"].view, act=outs["act"].view)
        else:
            outs["out"] = Guarded(M, N, bf16, dev)
            kw = {}
            if self.nq is not None:
                nheads = self.rope_cols // 128
                outs["pre"], outs["rstd"] = Guarded(M, self.rope_cols, bf16, dev), Guarded(M, nheads, f32, dev)
                kw = dict(q_norm=self.wq, k_norm=self.wk, nq_heads=self.nq, eps=EPS, pre_out=outs["pre"].view,
                          rstd_out=outs["rstd"].view)
            o.gemm_rope(self.a, self.b, self.cos, self.sin, self.L, self.rope_cols, out=outs["out"].view, bias=self.bias, **kw)
        return outs

    def chunks(self):
        """(r0, r1, exact accumulator rows [r0, r1) in fp64): torch fp32 on the GPU, one fp64 cross-check on the last chunk"""
        r = self.r
        bt = self.b.float()
        bt = bt.t() if r.layout == 0 else bt
        rows = max(128, CHUNK_ELEMS // r.N // 128 * 128)
        for r0 in range(0, r.M, rows):
            r1 = min(r.M, r0 + rows)
            ar = self.a[:, r0:r1].t() if r.layout == 2 else self.a[r0:r1]
            acc = (ar.float() @ bt).double()
            if r1 == r.M:                                            # the reference itself, against fp64 (ragged tile, 2048 cols)
                t0, c1 = max(r0, r1 - 128), min(r.N, 2048)
                a64 = ar[t0 - r0:].double()
                b64 = (self.b[:c1].double().t() if r.layout == 0 else self.b[:, :c1].double())
                assert torch.equal(a64 @ b64, acc[t0 - r0:, :c1]), f"{r}: the fp32 reference is not exact"
            yield r0, r1, acc

    def check(self, outs, bn):
        r, e = self.r, self.r.epi
        tn = bn % 1000 if bn else _tile_n(r)
        what = f"{r.model} {r.proj} ({r.entry} layout {r.layout}, {e}) M {r.M} N {r.N} K {r.K} block_n {bn}"
        for r0, r1, acc in self.chunks():
            got = outs["out"].view[r0:r1]
            x = acc + (self.bias.double() if self.bias is not None else 0)
            if r.entry == "rope":
                self._check_rope(outs, x, r0, r1, what)
                continue
            if r.entry == "swiglu":
                _expect_equal(got, x.to(bf16), what + " gu", 128, 256, row0=r0)
                blk = acc.view(r1 - r0, r.N // 256, 2, 128)
                gate, up = blk[:, :, 0].reshape(r1 - r0, r.N // 2), blk[:, :, 1].reshape(r1 - r0, r.N // 2)
                ref = gate * torch.sigmoid(gate) * up                  # tolerance as in test_gemm_swiglu_exact
                _expect_close(outs["act"].view[r0:r1], ref, _ulp_bf16(ref) + 2.0 ** -20 * ref.abs() + 2.0 ** -100,
                              what + " act", 128, 128, row0=r0)
                continue
            if r.entry == "gelu":
                _expect_equal(got, x.to(bf16), what + " pre", 128, tn, row0=r0)
                p = x.to(bf16).double()                                  # as in test_gemm_gelu_exact
                ref = _gelu64(p)
                _expect_close(outs["act"].view[r0:r1], ref, _ulp_bf16(ref) + 2.0 ** -21 * (ref.abs() + p.abs()),
                              what + " act", 128, tn, row0=r0)
                continue
            res = self.resid[r0:r1].double() if self.resid is not None and e not in ("act2",) else 0
            if e == "act1":                                              # tolerances as in test_exact_tiles_gpu._run_gemm
                ref = _gelu64(x)
                _expect_close(got, ref, _ulp_bf16(ref) + 2.0 ** -21 * (ref.abs() + x.abs()), what, 128, tn, row0=r0)
            elif e == "act2":
                d = x.to(bf16).double()
                gg = _gelu_grad64(self.resid[r0:r1].double())
                ref = d * gg
                _expect_close(got, ref, _ulp_bf16(ref) + 2.0 ** -20 * d.abs() * (gg.abs() + 1), what, 128, tn, row0=r0)
            elif self.drop is not None:
                sc = ops_mod().dropout_scale(r1 * r.N, self.drop, self.dev)[r0 * r.N:].view(r1 - r0, r.N).double()
                xs = x * sc
                ref = xs + res
                _expect_close(got, ref, _ulp_f32(torch.maximum(ref.abs(), xs.abs())), what, 128, tn, row0=r0)
            else:
                _expect_equal(got, (x + res).to(self.odt), what, 128, tn, row0=r0)
        for name, gd in outs.items():
            gd.check(f"{what} {name}")

    def _check_rope(self, outs, y, r0, r1, what):
        """bounds as in test_gemm_rope_exact (RoPE) and test_gemm_rope_qk_norm_exact (q/k norm + RoPE)"""
        C, n = self.rope_cols, r1 - r0
        pos = torch.arange(r0, r1, device=self.dev) % self.L
        got = outs["out"].view[r0:r1]
        if self.nq is not None:
            rot, r64, terms = _ref_norm_rope(y, C // 128, self.nq, self.wq, self.wk, self.cos, self.sin, pos)
            _expect_equal(outs["pre"].view[r0:r1], y[:, :C].to(bf16), what + " pre", 128, 256, row0=r0)
            _expect_close(outs["rstd"].view[r0:r1], r64, 4 * _ulp_f32(r64), what + " rstd", 128, 2, row0=r0)
            _expect_close(got[:, :C], rot, _ulp_bf16(rot) + 2.0 ** -20 * terms, what + " rotated", 128, 256, row0=r0)
        else:
            c, s = self.cos.double()[pos][:, None], self.sin.double()[pos][:, None]
            h = y[:, :C].reshape(n, C // 128, 2, 64)
            x1, x2 = h[:, :, 0], h[:, :, 1]
            rot = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).view(n, C)
            terms = torch.stack([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], 2).view(n, C)
            _expect_close(got[:, :C], rot, _ulp_bf16(rot) + 2.0 ** -22 * terms, what + " rotated", 128, 256, row0=r0)
        _expect_equal(got[:, C:], y[:, C:].to(bf16), what + " plain", 128, 256, row0=r0)


def _tile_n(r):
    """the tile width the launch used (for failure messages): the fused epilogues run 256-wide tiles"""
    return 256 if r.entry in ("swiglu", "rope") else _pick_block_n(r.M, r.N, ops_mod().num_sms())


@pytest.mark.gpu
@pytest.mark.parametrize("row,widths", _params())
def test_gemm_production_exact(dev, exact_fp32, row, widths):
    """one table row: every output element against the exact reference, at the dispatcher's tile width and (plain kernels)
    every other width"""
    case = _Case(row, dev, seed=zlib.crc32(f"{row}".encode()) & 0xFFFF)
    for bn in widths:
        case.check(case.run(bn), bn)


# random-valued operands (bf16 from randn) per family: layout 0, fp32 output, the family's longest forward contraction.
# Three m-tiles (first, middle, ragged last) against fp64 within the fp32 dot-product bound gamma_K sum |a| |b|: products of
# bf16 values are exact in fp32 and the output is the fp32 accumulator itself (no further rounding).
RANDOM = [("llama2-7b down", 4590, 4096, 11008), ("llama3-8b down", 4590, 4096, 14336), ("qwen2.5-7b down", 4590, 3584, 18944),
          ("qwen3-8b down", 4590, 4096, 12288), ("olmo2-7b down", 4590, 4096, 11008), ("falcon-7b W2", 36850, 4544, 18176),
          ("bge-large Wo2", 900, 1024, 4096)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,M,N,K", RANDOM, ids=[r[0].replace(" ", "-") for r in RANDOM])
def test_gemm_production_random(dev, name, M, N, K):
    g = torch.Generator(device=dev).manual_seed(K)
    a = torch.full((M + PAD_R, K + PAD_C), float("nan"), dtype=bf16, device=dev)
    a[:M, :K].copy_(torch.randn(M, K, generator=g, device=dev))
    b = torch.full((N + PAD_R, K + PAD_C), float("nan"), dtype=bf16, device=dev)
    b[:N, :K].copy_(torch.randn(N, K, generator=g, device=dev))
    a, b = a[:M, :K], b[:N, :K]
    out = Guarded(M, N, f32, dev)
    ops_mod().gemm(a, b, out=out.view, out_dtype=f32)
    U = 2.0 ** -24
    gamma = K * U / (1 - K * U)
    b64 = b.double()
    last = (M - 1) // 128
    worst = 0.0
    for t in (0, last // 2, last):
        rows = slice(128 * t, min(M, 128 * t + 128))
        a64 = a[rows].double()
        ref = a64 @ b64.t()
        bound = gamma * (a64.abs() @ b64.abs().t())
        err = (out.view[rows].double() - ref).abs()
        worst = max(worst, (err / bound).max().item())
        _expect_close(out.view[rows], ref, bound, f"{name} random M {M} N {N} K {K} m-tile {t}", 128, 256, row0=128 * t)
    print(f"[random] {name} M {M} N {N} K {K}: worst |err| / (gamma_K sum|a||b|) = {worst:.3e}")
    out.check(f"{name} random")


# ----------------------------------------------------------------------------------------------------------------
# 3. the decode GEMM: every M <= 16, the ring's wrap, the gemm_rows switch
# ----------------------------------------------------------------------------------------------------------------
def _decode_rows():
    """(model, projection, N, K, out dtype, act, bias, resid) of llama.py _decode_step (:592 qkv on the K-augmented
    h1 with bias, :606 o + resid, :611 gate|up, :617 down + resid, :619 lm_head; post-norm :604 / :614 bf16) and
    falcon.py _decode_step (:301 qkv, :305 dense + resid, :306 W1 act=1 and W2 + resid, :308 lm_head)"""
    out = []
    for model, c, bias, post in (("llama2-7b", LLAMA2_7B, False, False), ("llama3-8b", LLAMA3_8B, False, False),
                                 ("qwen2.5-7b", QWEN25_7B, True, False), ("qwen3-8b", QWEN3_8B, False, False),
                                 ("olmo2-7b", OLMO2_7B, False, True)):
        H, F, nh, nkv, V = (c[k] for k in ("hidden_size", "intermediate_size", "num_attention_heads", "num_key_value_heads",
                                           "vocab_size"))
        out += [(model, "qkv", (nh + 2 * nkv) * 128, H + 2 * R, bf16, 0, bias, False),
                (model, "o", H, nh * 128, bf16 if post else f32, 0, False, not post),
                (model, "gate|up", 2 * F, H, bf16, 0, False, False),
                (model, "down", H, F, bf16 if post else f32, 0, False, not post),
                (model, "lm_head", (V + 7) // 8 * 8, H, bf16, 0, False, False)]
    H, nh = FALCON_7B["hidden_size"], FALCON_7B["num_attention_heads"]
    hd = H // nh
    out += [("falcon-7b", "qkv", nh * hd + 2 * hd, H, bf16, 0, False, False), ("falcon-7b", "dense", H, H, f32, 0, False, True),
            ("falcon-7b", "W1", 4 * H, H, bf16, 1, False, False), ("falcon-7b", "W2", H, 4 * H, f32, 0, False, True),
            ("falcon-7b", "lm_head", (FALCON_7B["vocab_size"] + 7) // 8 * 8, H, bf16, 0, False, False)]
    return out


DECODE = _decode_rows()


def _decode_case(dev, M, N, K, odt, act, bias, resid, g, a16=None, w=None, acc16=None, shift=0):
    """decode_gemm on the first M rows of a16 (re-poisoned) and w into a guarded output -> (output, exact pre-activation
    fp64, residual). acc16: a16 @ w^T, when the caller has it"""
    if w is None:
        w = _dev_ints(N, K, g, dev, pad_c=48)
    if a16 is None:
        a16 = _dev_ints(16, K, g, dev)
    a = torch.full((M + PAD_R, K + 48), float("nan"), dtype=bf16, device=dev)   # row stride K + 48: the aug buffer's H + 64
    a[:M, :K] = a16[:M]
    a = a[:M, :K]
    bv = _dev_vec(N, g, dev) if bias else None
    rv = _dev_ints(M, N, g, dev, odt, 2048 if odt == f32 else 256) if resid else None
    out = Guarded(M, N, odt, dev, shift=shift)
    ops_mod().decode_gemm(a, w, out=out.view, out_dtype=odt, act=act, resid=rv, bias=bv)
    acc = acc16[:M] if acc16 is not None else (a.float() @ w.float().t()).double()
    return out, acc + (bv.double() if bias else 0), rv


def _decode_check(out, x, rv, odt, act, what):
    if act == 1:
        ref = _gelu64(x) + (rv.double() if rv is not None else 0)
        _expect_close(out.view, ref, (_ulp_bf16(ref) if odt == bf16 else 0) + 2.0 ** -21 * (ref.abs() + x.abs()), what, 128, 16)
    else:
        _expect_equal(out.view, (x + (rv.double() if rv is not None else 0)).to(odt), what, 128, 16)
    out.check(what)


@pytest.mark.gpu
@pytest.mark.parametrize("model,proj,N,K,odt,act,bias,resid", DECODE,
                         ids=[f"{d[0]}-{d[1]}".replace("|", "") for d in DECODE])
def test_decode_gemm_every_m(dev, exact_fp32, model, proj, N, K, odt, act, bias, resid):
    """M = 1 .. 16 at one decode projection: integer operands, exact (GELU: the tile tests' bound); odd M write through a
    view that starts one element past a 16-byte boundary (the kernel stores scalars)"""
    g = torch.Generator(device=dev).manual_seed(N + K)
    w = _dev_ints(N, K, g, dev, pad_c=48)
    a16 = _dev_ints(16, K, g, dev)
    acc16 = (a16.float() @ w.float().t()).double()
    for M in range(1, 17):
        out, x, rv = _decode_case(dev, M, N, K, odt, act, bias, resid, g, a16=a16, w=w, acc16=acc16, shift=M % 2)
        _decode_check(out, x, rv, odt, act, f"decode_gemm {model} {proj} M {M} N {N} K {K} {odt} act {act} bias {bias}")


def _ring_ks():
    """K whose per-warp chunk counts ceil((ceil(K/32) - w) / 8) run over DG_STAGES - 1, DG_STAGES, DG_STAGES + 1 (all warps
    equal at 8 (S-1), 8 S, 8 (S+1) chunks; mixed between), each at every K % 32"""
    out = []
    for nch in (8 * (DG_STAGES - 1), 8 * (DG_STAGES - 1) + 1, 8 * DG_STAGES - 1, 8 * DG_STAGES, 8 * DG_STAGES + 1,
                8 * DG_STAGES + 4, 8 * (DG_STAGES + 1)):
        for tail in (32, 8, 16, 24):                          # K % 32 = 0, 8, 16, 24
            out.append(32 * (nch - 1) + tail)
    return out


def test_ring_ks_cover_the_wrap():
    """CPU: the ring sweep reaches chunk counts S - 1, S and S + 1 for every warp, and every K % 32"""
    ks = _ring_ks()
    for w in range(8):
        counts = {-(-(-(-K // 32) - w) // 8) for K in ks}
        assert {DG_STAGES - 1, DG_STAGES, DG_STAGES + 1} <= counts, (w, counts)
    assert {K % 32 for K in ks} == {0, 8, 16, 24}


@pytest.mark.gpu
@pytest.mark.parametrize("N", [8, 32, 40])
def test_decode_gemm_ring_sweep(dev, exact_fp32, N):
    """every K of the ring sweep at N % 16 in {0, 8} (N = 8: a CTA with one live n-tile), M cycling 1 / 8 / 9 / 16"""
    g = torch.Generator(device=dev).manual_seed(N)
    for i, K in enumerate(_ring_ks()):
        M = (1, 8, 9, 16)[i % 4]
        odt = (bf16, f32)[i % 2]
        out, x, rv = _decode_case(dev, M, N, K, odt, 0, i % 3 == 0, i % 5 == 0, g)
        _decode_check(out, x, rv, odt, 0, f"decode_gemm ring sweep M {M} N {N} K {K} ({-(-K // 32)} chunks) {odt}")


GEMM_ROWS = [(d[0], d[1], d[2], d[3], d[6]) for d in DECODE if d[1] in ("qkv", "lm_head")]


@pytest.mark.gpu
@pytest.mark.parametrize("model,proj,N,K,bias", GEMM_ROWS, ids=[f"{d[0]}-{d[1]}" for d in GEMM_ROWS])
def test_gemm_rows_switch(dev, exact_fp32, monkeypatch, model, proj, N, K, bias):
    """gemm_rows at M = 16 (decode kernel), 17 (wgmma) and, with DALM_B200_DECODE_GEMM=0, 16 on the wgmma GEMM: all exact"""
    g = torch.Generator(device=dev).manual_seed(N * 3 + K)
    w = _dev_ints(N, K, g, dev, pad_c=48)
    a17 = _dev_ints(17, K, g, dev, pad_c=48)
    bv = _dev_vec(N, g, dev) if bias else None
    ref = (a17.float() @ w.float().t()).double() + (bv.double() if bias else 0)
    for M, env in ((16, None), (17, None), (16, "0")):
        if env is not None:
            monkeypatch.setenv("DALM_B200_DECODE_GEMM", env)
        a = torch.full((M + PAD_R, K + 48), float("nan"), dtype=bf16, device=dev)
        a[:M, :K] = a17[:M]
        got = ops_mod().gemm_rows(a[:M, :K], w, bias=bv)
        _expect_equal(got, ref[:M].to(bf16), f"gemm_rows {model} {proj} M {M} N {N} K {K} DALM_B200_DECODE_GEMM={env}", 128, 16)


# ----------------------------------------------------------------------------------------------------------------
# 4. wrapper contracts: every call below hands a kernel an operand it would read or write past, or misread. With
# `_lib.call` replaced by a recorder, no case may reach it: the wrapper must raise DalmB200Error first.
# ----------------------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


@pytest.fixture
def recorder(dev, monkeypatch):
    from dalm_b200 import _lib
    calls = []

    def rec(name, *args):
        calls.append(name)
        raise _Reached(name)
    monkeypatch.setattr(_lib, "call", rec)
    return calls


def _z(*shape, dtype=bf16, dev="cuda"):
    return torch.zeros(*shape, dtype=dtype, device=dev)


def _tab(L=4):
    return _z(L, 64, dtype=f32), _z(L, 64, dtype=f32)


_A, _B = (lambda: _z(256, 64)), (lambda: _z(128, 64))         # gemm layout 0: M 256, N 128, K 64
_DA, _DW = (lambda: _z(4, 64)), (lambda: _z(32, 64))          # decode: M 4, N 32, K 64

REFUSALS = {
    # gemm: out
    "gemm_out_rows": lambda o: o.gemm(_A(), _B(), out=_z(256, 128)[:200]),
    "gemm_out_cols": lambda o: o.gemm(_A(), _B(), out=_z(256, 256)[:, :120]),
    "gemm_out_transposed": lambda o: o.gemm(_A(), _B(), out=_z(128, 256).t()),
    "gemm_out_cpu": lambda o: o.gemm(_A(), _B(), out=_z(256, 128, dev="cpu")),
    "gemm_out_dtype": lambda o: o.gemm(_A(), _B(), out=_z(256, 128, dtype=torch.float16)),
    # gemm: bias
    "gemm_bias_short": lambda o: o.gemm(_A(), _B(), bias=_z(256, dtype=f32)[:100]),
    "gemm_bias_strided": lambda o: o.gemm(_A(), _B(), bias=_z(256, dtype=f32)[::2]),
    "gemm_bias_cpu": lambda o: o.gemm(_A(), _B(), bias=_z(128, dtype=f32, dev="cpu")),
    "gemm_bias_dtype": lambda o: o.gemm(_A(), _B(), bias=_z(128)),
    # gemm: resid
    "gemm_resid_rows": lambda o: o.gemm(_A(), _B(), out_dtype=f32, resid=_z(256, 128, dtype=f32)[:100]),
    "gemm_resid_cols": lambda o: o.gemm(_A(), _B(), out_dtype=f32, resid=_z(256, 256, dtype=f32)[:, :64]),
    "gemm_resid_transposed": lambda o: o.gemm(_A(), _B(), out_dtype=f32, resid=_z(128, 256, dtype=f32).t()),
    "gemm_resid_cpu": lambda o: o.gemm(_A(), _B(), out_dtype=f32, resid=_z(256, 128, dtype=f32, dev="cpu")),
    "gemm_resid_dtype": lambda o: o.gemm(_A(), _B(), resid=_z(256, 128, dtype=torch.float16)),
    # gemm: operands, K, overrides
    "gemm_a_cpu": lambda o: o.gemm(_z(256, 64, dev="cpu"), _B()),
    "gemm_a_dtype": lambda o: o.gemm(_z(256, 64, dtype=f32), _B()),
    "gemm_b_cpu": lambda o: o.gemm(_A(), _z(128, 64, dev="cpu")),
    "gemm_b_dtype": lambda o: o.gemm(_A(), _z(128, 64, dtype=torch.float16)),
    "gemm_k_mismatch_layout0": lambda o: o.gemm(_A(), _z(128, 72)),
    "gemm_k_mismatch_layout1": lambda o: o.gemm(_A(), _z(72, 128), layout=1),
    "gemm_k_override_past_a": lambda o: o.gemm(_A(), _z(128, 256)[:, :64], K=128),
    "gemm_n_override_past_b": lambda o: o.gemm(_A(), _B(), N=256),
    "gemm_1d_operand": lambda o: o.gemm(_z(64), _B()),
    # wgrad_ (layout 2): a [T, M], b [T, N], gw [M, N]
    "wgrad_k_mismatch": lambda o: o.wgrad_(_z(64, 128), _z(72, 256), _z(128, 256, dtype=f32), False),
    "wgrad_k_override_past": lambda o: o.wgrad_(_z(64, 128), _z(64, 256), _z(128, 256, dtype=f32), False, K=80),
    "wgrad_out_rows": lambda o: o.wgrad_(_z(64, 128), _z(64, 256), _z(128, 256, dtype=f32)[:64], False),
    "wgrad_acc_transposed": lambda o: o.wgrad_(_z(64, 128), _z(64, 256), _z(256, 128, dtype=f32).t(), True),
    "wgrad_out_cpu": lambda o: o.wgrad_(_z(64, 128), _z(64, 256), _z(128, 256, dtype=f32, dev="cpu"), False),
    # gemm_swiglu: a [256, 64], w [512, 64] -> gu [256, 512], act [256, 256]
    "swiglu_gu_rows": lambda o: o.gemm_swiglu(_A(), _z(512, 64), gu=_z(256, 512)[:128], act=_z(256, 256)),
    "swiglu_gu_dtype": lambda o: o.gemm_swiglu(_A(), _z(512, 64), gu=_z(256, 512, dtype=f32), act=_z(256, 256)),
    "swiglu_act_cols": lambda o: o.gemm_swiglu(_A(), _z(512, 64), gu=_z(256, 512), act=_z(256, 256)[:, :248]),
    "swiglu_act_cpu": lambda o: o.gemm_swiglu(_A(), _z(512, 64), gu=_z(256, 512), act=_z(256, 256, dev="cpu")),
    "swiglu_k_mismatch": lambda o: o.gemm_swiglu(_A(), _z(512, 72)),
    "swiglu_w_cpu": lambda o: o.gemm_swiglu(_A(), _z(512, 64, dev="cpu")),
    "swiglu_a_cpu": lambda o: o.gemm_swiglu(_z(256, 64, dev="cpu"), _z(512, 64)),
    "swiglu_a_dtype": lambda o: o.gemm_swiglu(_z(256, 64, dtype=f32), _z(512, 64)),
    # gemm_gelu: a [256, 64], w [128, 64]
    "gelu_bias_short": lambda o: o.gemm_gelu(_A(), _B(), bias=_z(128, dtype=f32)[:64]),
    "gelu_bias_cpu": lambda o: o.gemm_gelu(_A(), _B(), bias=_z(128, dtype=f32, dev="cpu")),
    "gelu_pre_rows": lambda o: o.gemm_gelu(_A(), _B(), pre=_z(256, 128)[:255], act=_z(256, 128)),
    "gelu_act_cols": lambda o: o.gemm_gelu(_A(), _B(), pre=_z(256, 128), act=_z(256, 128)[:, :64]),
    "gelu_pre_dtype": lambda o: o.gemm_gelu(_A(), _B(), pre=_z(256, 128, dtype=f32)),
    "gelu_k_mismatch": lambda o: o.gemm_gelu(_A(), _z(128, 72)),
    "gelu_a_dtype": lambda o: o.gemm_gelu(_z(256, 64, dtype=f32), _B()),
    "gelu_w_cpu": lambda o: o.gemm_gelu(_A(), _z(128, 64, dev="cpu")),
    "gelu_act_cpu": lambda o: o.gemm_gelu(_A(), _B(), pre=_z(256, 128), act=_z(256, 128, dev="cpu")),
    "gelu_bias_dtype": lambda o: o.gemm_gelu(_A(), _B(), bias=_z(128)),
    # gemm_rope: a [256, 64], w [256, 64], rope_cols 256
    "rope_out_rows": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, out=_z(256, 256)[:128]),
    "rope_out_cols": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, out=_z(256, 512)[:, :248]),
    "rope_out_dtype": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, out=_z(256, 256, dtype=f32)),
    "rope_out_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, out=_z(256, 256, dev="cpu")),
    "rope_k_mismatch": lambda o: o.gemm_rope(_A(), _z(256, 72), *_tab(), 4, 256),
    "rope_bias_short": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, bias=_z(200, dtype=f32)),
    "rope_cos_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64), _z(4, 64, dtype=f32, dev="cpu"), _z(4, 64, dtype=f32), 4, 256),
    "rope_sin_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64), _z(4, 64, dtype=f32), _z(4, 64, dtype=f32, dev="cpu"), 4, 256),
    "rope_a_dtype": lambda o: o.gemm_rope(_z(256, 64, dtype=f32), _z(256, 64), *_tab(), 4, 256),
    "rope_w_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64, dev="cpu"), *_tab(), 4, 256),
    "rope_bias_dtype": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, bias=_z(256)),
    "rope_q_norm_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, q_norm=_z(128, dtype=f32, dev="cpu"),
                                             k_norm=_z(128, dtype=f32), nq_heads=1),
    "rope_pre_out_cpu": lambda o: o.gemm_rope(_A(), _z(256, 64), *_tab(), 4, 256, q_norm=_z(128, dtype=f32),
                                              k_norm=_z(128, dtype=f32), nq_heads=1, pre_out=_z(256, 256, dev="cpu")),
    # decode_gemm: a [4, 64], w [32, 64]
    "decode_out_rows": lambda o: o.decode_gemm(_DA(), _DW(), out=_z(3, 32)),
    "decode_out_cols": lambda o: o.decode_gemm(_DA(), _DW(), out=_z(4, 64)[:, :24]),
    "decode_out_transposed": lambda o: o.decode_gemm(_DA(), _DW(), out=_z(32, 4).t()),
    "decode_out_cpu": lambda o: o.decode_gemm(_DA(), _DW(), out=_z(4, 32, dev="cpu")),
    "decode_out_dtype": lambda o: o.decode_gemm(_DA(), _DW(), out=_z(4, 32, dtype=torch.float16)),
    "decode_resid_rows": lambda o: o.decode_gemm(_DA(), _DW(), out_dtype=f32, resid=_z(2, 32, dtype=f32)),
    "decode_resid_transposed": lambda o: o.decode_gemm(_DA(), _DW(), out_dtype=f32, resid=_z(32, 4, dtype=f32).t()),
    "decode_resid_cpu": lambda o: o.decode_gemm(_DA(), _DW(), out_dtype=f32, resid=_z(4, 32, dtype=f32, dev="cpu")),
    "decode_resid_dtype": lambda o: o.decode_gemm(_DA(), _DW(), resid=_z(4, 32, dtype=torch.float16)),
    "decode_bias_short": lambda o: o.decode_gemm(_DA(), _DW(), bias=_z(16, dtype=f32)),
    "decode_k_mismatch": lambda o: o.decode_gemm(_DA(), _z(32, 72)),
    "decode_a_cpu": lambda o: o.decode_gemm(_z(4, 64, dev="cpu"), _DW()),
    "decode_w_dtype": lambda o: o.decode_gemm(_DA(), _z(32, 64, dtype=f32)),
    "decode_bias_dtype": lambda o: o.decode_gemm(_DA(), _DW(), bias=_z(32)),
    "decode_bias_cpu": lambda o: o.decode_gemm(_DA(), _DW(), bias=_z(32, dtype=f32, dev="cpu")),
    # gemm_rows: both sides of the 16-row switch
    "gemm_rows_decode_resid_rows": lambda o: o.gemm_rows(_DA(), _DW(), out_dtype=f32, resid=_z(3, 32, dtype=f32)),
    "gemm_rows_wgmma_resid_rows": lambda o: o.gemm_rows(_z(32, 64), _DW(), out_dtype=f32, resid=_z(20, 32, dtype=f32)),
    "gemm_rows_wgmma_bias_short": lambda o: o.gemm_rows(_z(32, 64), _DW(), bias=_z(16, dtype=f32)),
    "gemm_rows_decode_k_mismatch": lambda o: o.gemm_rows(_DA(), _z(32, 72)),
}


def _aug(rows, cols, ra):
    """engine _aug_buf: [rows, cols + ra] with the row stride padded to cols + 64"""
    return _z(rows, cols + 64)[:, :cols + ra]


def _inplace(o):
    buf = _z(256, 128, dtype=f32)
    o.gemm(_A(), _B(), out=buf, resid=buf)


def _inplace16(o):
    dh = _z(256, 128)
    o.gemm(_z(256, 72), _z(72, 128), out=dh, resid=dh, layout=1)


# legitimate calls the checks must let through: each must reach the (recorded) kernel launch
ACCEPTS = {
    "gemm": lambda o: o.gemm(_A(), _B()),
    "gemm_col_slice_out": lambda o: o.gemm(_A(), _B(), out=_z(256, 512)[:, 128:256]),
    "gemm_out_is_resid": _inplace,
    "gemm_out_is_resid_bf16_layout1": _inplace16,
    "gemm_head_chunk": lambda o: o.gemm(_z(200, 64), _B(), out=_z(384, 128)[:200]),
    "gemm_dgrad_row_slice_out": lambda o: o.gemm(_z(200, 128), _z(64, 128), out=_z(384, 64)[184:384]),
    "gemm_kaug_folded": lambda o: o.gemm(_aug(256, 384, 24), _aug(128, 384, 24)),
    "gemm_kaug_base": lambda o: o.gemm(_aug(256, 384, 24)[:, :384], _aug(128, 384, 24)[:, :384]),
    "gemm_kaug_base_layout1": lambda o: o.gemm(_aug(256, 384, 24)[:, :384], _aug(384, 128, 24)[:, :128], layout=1),
    "gemm_bias_longer": lambda o: o.gemm(_A(), _B(), bias=_z(256, dtype=f32)),
    "wgrad": lambda o: o.wgrad_(_z(64, 128), _aug(64, 256, 16)[:, :256], _z(128, 256, dtype=f32), True),
    "swiglu": lambda o: o.gemm_swiglu(_A(), _z(512, 64)),
    "gelu": lambda o: o.gemm_gelu(_A(), _B(), bias=_z(128, dtype=f32)),
    "rope": lambda o: o.gemm_rope(_aug(256, 64, 16), _aug(256, 64, 16), *_tab(), 4, 256, bias=_z(256, dtype=f32)),
    "decode_gemm": lambda o: o.decode_gemm(_aug(4, 64, 16), _aug(32, 64, 16), out_dtype=f32, resid=_z(4, 32, dtype=f32)),
    "gemm_rows_decode": lambda o: o.gemm_rows(_DA(), _DW(), bias=_z(32, dtype=f32)),
    "gemm_rows_wgmma": lambda o: o.gemm_rows(_z(32, 64), _DW(), out_dtype=f32, resid=_z(32, 32, dtype=f32)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusal(ops, recorder, case):
    from dalm_b200._lib import DalmB200Error
    try:
        REFUSALS[case](ops)
    except _Reached as e:
        pytest.fail(f"{case}: reached the kernel with {e}")
    except DalmB200Error:
        pass
    else:
        pytest.fail(f"{case}: accepted")
    assert recorder == []


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(ACCEPTS))
def test_accepted_reaches_kernel(ops, recorder, case):
    """positive control: the recorder is wired up, and the checks pass the shapes the engines use"""
    with pytest.raises(_Reached):
        ACCEPTS[case](ops)
    assert len(recorder) == 1
