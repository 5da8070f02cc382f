"""-m gpu: Qwen3 generators and retrievers (Llama + a per-head RMSNorm of q and k before RoPE).

Kernels, under the rules of test_exact_tiles_gpu.py (integer operands, NaN-poisoned padding, guard bands):
  * the NormRoPE epilogue of gemm_bf16_rope: the pre-norm columns bit for bit, rstd within 4 fp32 ulps of fp64 (the integer
    sums of squares are exact in fp32: only the eps addition and rsqrtf's <= 2 ulp error remain), the rotated q|k columns
    within one bf16 ulp plus 2^-20 of the magnitudes summed by the rotation (a few fp32 roundings), v columns bit-exact;
  * the row kernel in both position modes against the same reference, and bit-equal to the epilogue on bf16-exact input;
  * the backward kernel's dx, dw_q, dw_k against fp64 autograd, including an all-zero head (rstd = 1/sqrt(eps)).
Models: forward / backward against transformers' Qwen3ForCausalLM on bf16-rounded weights with q / k norm weights 1 + N(0, 0.5)
(a dropped, swapped or misplaced norm moves the logits far beyond bf16 noise), full fine-tuning including the norm weights,
the fused RAG step, an autoregressive Qwen3 retriever, `generate` on both decode-GEMM paths, and the trainer + eval-rag.
Tolerances are those of test_qwen2_gpu.py.
"""
import os

import pytest
import torch

from exact_helpers import Guarded, _expect_close, _expect_equal, _poisoned, _ulp_bf16, _ulp_f32
from test_exact_tiles_gpu import M_EDGE, _ints

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
NORM_STD = 0.5
EPS = 1e-6


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


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


# ----------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------
def test_gemm_rope_qk_norm_exact(cuda_dev):
    """the NormRoPE epilogue: pre-norm columns, rstd, rotated q|k and plain v columns, each against fp64; the launch without
    pre / rstd outputs writes the same rotated columns"""
    from dalm_b200 import ops
    dev = cuda_dev
    Lr = 37
    cos_t, sin_t = _tables(dev, Lr)
    i = 0
    for M in M_EDGE:
        for N, rope_cols in ((264, 256), (512, 512), (520, 512), (1792 + 256, 1792)):
            for K in (8, 72):
                g = torch.Generator().manual_seed(1700 + i)
                a = _poisoned(_ints((M, K), g).to(dev, bf16))
                w = _poisoned(_ints((N, K), g).to(dev, bf16))
                bias = _poisoned(_ints((N,), g, hi=64).to(dev)) if i % 2 else None
                wq, wk = _norm_w(g, dev), _norm_w(g, dev)
                nheads = rope_cols // 128
                nq = (nheads * 3) // 4                                               # q heads first, then k heads
                out, pre = Guarded(M, N, bf16, dev), Guarded(M, rope_cols, bf16, dev)
                rstd = Guarded(M, nheads, f32, dev)
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=out.view, bias=bias, q_norm=wq, k_norm=wk, nq_heads=nq,
                              eps=EPS, pre_out=pre.view, rstd_out=rstd.view)
                what = f"gemm_rope+norm M {M} N {N} K {K} rope_cols {rope_cols} bias {bias is not None}"
                y = a.double() @ w.double().t()
                if bias is not None:
                    y = y + bias.double()[None]                                      # exact in fp32 too
                pos = torch.arange(M, device=dev) % Lr
                rot, r64, terms = _ref_norm_rope(y, nheads, nq, wq, wk, cos_t, sin_t, pos)
                _expect_equal(pre.view, y[:, :rope_cols].to(bf16), what + " pre", 128, 256)
                _expect_close(rstd.view, r64, 4 * _ulp_f32(r64), what + " rstd", 128, 2)
                _expect_close(out.view[:, :rope_cols], rot, _ulp_bf16(rot) + 2.0 ** -20 * terms, what + " rotated", 128, 256)
                _expect_equal(out.view[:, rope_cols:], y[:, rope_cols:].to(bf16), what + " plain", 128, 256)
                out.check(what); pre.check(what + " pre"); rstd.check(what + " rstd")
                bare = Guarded(M, N, bf16, dev)
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=bare.view, bias=bias, q_norm=wq, k_norm=wk, nq_heads=nq, eps=EPS)
                _expect_equal(bare.view, out.view, what + " without pre / rstd", 128, 256)
                bare.check(what + " without pre / rstd")
                i += 1


@pytest.mark.parametrize("mode", ["row % L", "pos"])
def test_qk_norm_rope_row_kernel(cuda_dev, mode):
    """the row kernel (decode, prefill, unfused training) in both position modes, in place: q|k heads against fp64, pre equal to
    the input, rstd within 4 fp32 ulps, columns after the q|k heads untouched"""
    from dalm_b200 import ops
    dev = cuda_dev
    T = 50
    cos_t, sin_t = _tables(dev, T)
    for j, (M, nheads, nq, extra) in enumerate(((1, 2, 1, 0), (7, 5, 4, 256), (300, 9, 8, 384), (16, 40, 32, 1024))):
        g = torch.Generator().manual_seed(2100 + j)
        x = _ints((M, 128 * nheads + extra), g, hi=40)
        x[0, :128] = 0                                                               # an all-zero head: rstd = 1/sqrt(eps)
        buf = _poisoned(x.to(dev, bf16))
        x0 = buf.clone()
        wq, wk = _norm_w(g, dev), _norm_w(g, dev)
        pre, rstd = Guarded(M, 128 * nheads, bf16, dev), Guarded(M, nheads, f32, dev)
        if mode == "pos":
            p = torch.randint(-2, T + 2, (M,), generator=g).to(dev)                 # out-of-range ids are clamped
            ops.qk_norm_rope_(buf, nheads, nq, wq, wk, EPS, cos_t, sin_t, pos=p, pre=pre.view, rstd=rstd.view)
            pos = p.clamp(0, T - 1)
        else:
            L = 13
            ops.qk_norm_rope_(buf, nheads, nq, wq, wk, EPS, cos_t[:L], sin_t[:L], L=L, pre=pre.view, rstd=rstd.view)
            pos = torch.arange(M, device=dev) % L
        what = f"qk_norm_rope ({mode}) M {M} heads {nheads}"
        rot, r64, terms = _ref_norm_rope(x0.double(), nheads, nq, wq, wk, cos_t, sin_t, pos)
        _expect_close(buf[:, :128 * nheads], rot, _ulp_bf16(rot) + 2.0 ** -20 * terms, what + " rotated", 16, 128)
        _expect_equal(buf[:, 128 * nheads:], x0[:, 128 * nheads:], what + " other columns", 16, 128)
        _expect_equal(pre.view, x0[:, :128 * nheads], what + " pre", 16, 128)
        _expect_close(rstd.view, r64, 4 * _ulp_f32(r64), what + " rstd", 16, 1)
        assert rstd.view[0, 0].item() == pytest.approx(EPS ** -0.5, rel=1e-6)
        pre.check(what + " pre"); rstd.check(what + " rstd")


def test_row_kernel_matches_epilogue(cuda_dev):
    """on pre-norm values that bf16 holds exactly, the row kernel and the fused epilogue compute the same bits"""
    from dalm_b200 import ops
    dev = cuda_dev
    L = 29
    cos_t, sin_t = _tables(dev, L, poison=False)
    for j, (M, N, rope_cols, nq) in enumerate(((257, 1280, 1024, 6), (128, 512, 512, 3))):
        g = torch.Generator().manual_seed(2300 + j)
        a = _ints((M, 8), g).to(dev, bf16)                                           # |y| <= 32: exact in bf16
        w = _ints((N, 8), g).to(dev, bf16)
        wq, wk = _norm_w(g, dev), _norm_w(g, dev)
        fused = ops.gemm_rope(a, w, cos_t, sin_t, L, rope_cols, q_norm=wq, k_norm=wk, nq_heads=nq, eps=EPS)
        rows = ops.gemm(a, w)
        ops.qk_norm_rope_(rows, rope_cols // 128, nq, wq, wk, EPS, cos_t, sin_t, L=L)
        _expect_equal(rows, fused, f"row kernel vs epilogue M {M} N {N}", 128, 256)


def test_qk_norm_rope_bwd(cuda_dev):
    """dx, dw_q, dw_k of norm -> RoPE against fp64 autograd from the same bf16 pre-norm values; dw accumulates (+=); columns
    after the q|k heads untouched"""
    from dalm_b200 import ops
    dev = cuda_dev
    L = 21
    cos_t, sin_t = _tables(dev, L)
    for j, (M, nheads, nq, extra) in enumerate(((5, 2, 1, 128), (300, 5, 4, 128), (2048, 10, 8, 256))):
        g = torch.Generator().manual_seed(2500 + j)
        x = (torch.randn(M, 128 * nheads, generator=g) * 3).to(bf16)
        x[0, :128] = 0                                                               # all-zero head
        x[min(3, M - 1), 128:256] = 0
        pre = _poisoned(x.to(dev))
        scratch = pre.clone()
        rstd = torch.empty(M, nheads, dtype=f32, device=dev)
        wq, wk = _norm_w(g, dev), _norm_w(g, dev)
        ops.qk_norm_rope_(scratch, nheads, nq, wq, wk, EPS, cos_t, sin_t, L=L, rstd=rstd)
        dy = torch.randn(M, 128 * nheads + extra, generator=g).to(bf16)
        dbuf = _poisoned(dy.to(dev))
        dwq0 = torch.randn(128, generator=g).to(dev)
        dwk0 = torch.randn(128, generator=g).to(dev)
        dwq, dwk = _poisoned(dwq0.clone()), _poisoned(dwk0.clone())
        ops.qk_norm_rope_bwd_(dbuf, nheads, nq, wq, wk, cos_t, sin_t, L, pre, rstd, dw_q=dwq, dw_k=dwk)
        # fp64 autograd
        xx = x.double().requires_grad_(True)
        wq64 = wq.double().cpu().requires_grad_(True)
        wk64 = wk.double().cpu().requires_grad_(True)
        h = xx.view(M, nheads, 128)
        r = 1.0 / torch.sqrt((h * h).mean(-1, keepdim=True) + EPS)
        wst = torch.stack([wq64 if i < nq else wk64 for i in range(nheads)])[None]
        xn = h * r * wst
        pos = torch.arange(M) % L
        c, s = cos_t.double().cpu()[pos][:, None], sin_t.double().cpu()[pos][:, None]
        out = torch.cat([xn[..., :64] * c - xn[..., 64:] * s, xn[..., 64:] * c + xn[..., :64] * s], -1)
        dy64 = dy[:, :128 * nheads].double().view(M, nheads, 128)
        out.backward(dy64)
        what = f"qk_norm_rope_bwd M {M} heads {nheads}"
        dx = xx.grad.view(M, nheads, 128)
        # fp32 error scale of dx = rstd (w g - x_hat m): the magnitudes of its two terms, per head
        with torch.no_grad():
            gg = torch.cat([dy64[..., :64] * c + dy64[..., 64:] * s, dy64[..., 64:] * c - dy64[..., :64] * s], -1)
            xh = h * r
            wg = (wst * gg).abs()
            scale = r * (wg.amax(-1, keepdim=True) + xh.abs().amax(-1, keepdim=True) * (wg * xh.abs()).mean(-1, keepdim=True))
            tol = _ulp_bf16(dx) + 2.0 ** -18 * scale.expand_as(dx)
        _expect_close(dbuf[:, :128 * nheads].cpu(), dx.reshape(M, -1).detach(), tol.reshape(M, -1), what + " dx", 16, 128)
        _expect_equal(dbuf[:, 128 * nheads:], dy[:, 128 * nheads:].to(dev), what + " other columns", 16, 128)
        assert torch.isfinite(dbuf[0, :128].float()).all() and dbuf[0, :128].float().abs().max() > 100   # rstd = 1000 there
        with torch.no_grad():
            mag = lambda hs: (gg[:, hs] * xh[:, hs]).abs().sum((0, 1))
            for got, base, ref, hs, nm in ((dwq, dwq0, wq64.grad, slice(0, nq), "dw_q"), (dwk, dwk0, wk64.grad, slice(nq, nheads), "dw_k")):
                err = (got.double().cpu() - base.double().cpu() - ref).abs()
                assert (err <= 1e-5 * mag(hs) + 1e-6).all(), (what, nm, err.max().item())


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
def build_qwen3(cfg, sd):
    """transformers' Qwen3ForCausalLM, fp32, on the given HF-named weights (tied configs store no lm_head)"""
    from transformers import Qwen3Config, Qwen3ForCausalLM
    m = Qwen3ForCausalLM(Qwen3Config(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}))
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected and set(missing) <= ({"lm_head.weight"} if cfg.get("tie_word_embeddings") else set()), (missing, unexpected)
    return m.float().eval()


def _qwen3(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.qwen3_config(name, vocab_size=V)
    sd = params.random_state_dict("qwen3", cfg, seed=seed, qk_norm_std=NORM_STD)
    return cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def _mask(B, L, pad):
    mask = torch.ones(B, L, dtype=torch.int64)
    if pad == "right":
        mask[0, L - 5:] = 0
    else:
        mask[0, :5] = 0; mask[1, :2] = 0
    return mask


def _lora_init(dec, ref, seed):
    from oracle import models as om
    g = torch.Generator().manual_seed(seed)
    for n, _, _ in dec.lora.specs:
        dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(dec.dev))
    dec.repack_lora()
    om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})


@pytest.mark.parametrize("name,B,L,pad", [("qwen3-tiny", 3, 40, "right"), ("qwen3-tiny", 2, 33, "left"),
                                           ("qwen3-hd128", 2, 72, "left"), ("qwen3-hd128", 2, 130, "right")])
def test_qwen3_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF Qwen3ForCausalLM (qwen3-tiny: 5 q|k heads, the row kernel,
    tied head; qwen3-hd128: 8 q|k heads, q/k norm + RoPE in the QKV epilogue, untied)"""
    from dalm_b200 import ops
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import losses, models as om
    V = 504
    cfg, sd = _qwen3(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    assert dec.qk_norm and dec.fuse_rope and (((dec.nh + dec.nkv) * 128) % 256 == 0) == (name == "qwen3-hd128")
    ref = build_qwen3(cfg, sd)
    _lora_init(dec, ref, 9)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(3, V, (B, L), generator=g)
    mask = _mask(B, L, pad)
    qlen = torch.tensor([3, L // 2, L + 2][:B])
    S = torch.randn(B, B, generator=g) * 3
    logits, ctx = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev))
    ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert _rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2
    ref_loss = losses.marginalized_loss_loopform(ref_logits, ids, mask, S, qlen)
    ref_loss.backward()
    cvec, nsum = ops.marginal_counts(mask.to(cuda_dev), qlen.to(cuda_dev))
    tok_lp, dl = ops.ce_marginal(logits, ids.to(cuda_dev), mask.to(cuda_dev), nsum)
    mine = losses.marginalized_loss_loopform(logits.float().cpu(), ids, mask, S, qlen)
    assert abs(mine.item() - ref_loss.item()) / abs(ref_loss.item()) < 1e-3
    dec.lora.zero_grad()
    dec.backward_logits(ctx, dl)
    worst = 0.0
    for n, _, _ in dec.lora.specs:
        mod = om._get_module(ref, n)
        worst = max(worst, _rel(dec.lora.gA[n], mod.lora_A.grad), _rel(dec.lora.gB[n], mod.lora_B.grad))
    assert worst < 5e-2, worst


def _rag_models(dev, gcfg, gsd, lora):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from oracle import models as om
    bcfg = synthetic.bert_config("bge-tiny", 600)
    r16 = lambda sd: {k: v.to(bf16).float() for k, v in sd.items()}
    bsd = r16(params.random_state_dict("bert", bcfg, seed=11))
    enc = BertEncoder(bcfg, bsd, device=dev, lora=lora, full=not lora)
    dec = LlamaDecoder(gcfg, gsd, device=dev, lora=lora, full=not lora)
    bert, ref = om.build_bert(bcfg, bsd), build_qwen3(gcfg, gsd)
    if lora:
        g = torch.Generator().manual_seed(13)
        for bank in (enc.lora, dec.lora):
            for n, _, _ in bank.specs:
                bank.B[n].copy_((torch.randn(bank.B[n].shape, generator=g) * 0.02).to(dev))
        enc.repack_lora(); dec.repack_lora()
        om.attach_lora(bert, {n: {"A": enc.lora.A[n].cpu(), "B": enc.lora.B[n].cpu()} for n, _, _ in enc.lora.specs})
        om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH if lora else None, _retriever=enc, _generator=dec, _load_tokenizers=False)
    return model, enc, dec, bert, ref


@pytest.mark.parametrize("name,pad", [("qwen3-tiny", "left"), ("qwen3-hd128", "right")])
def test_fused_rag_step_qwen3_lora(cuda_dev, name, pad):
    """bge + Qwen3 generator, LoRA on both: the fused training step against the reference loop body"""
    from test_step_gpu import _batch, _check_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _qwen3(name, 504, seed=12)
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=True)
    batch = _batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad)
    want = om.rag_step(bert, ref, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    got = out["losses"].cpu()
    assert abs(got[2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    _check_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["qwen3-tiny", "qwen3-hd128"])
def test_full_finetune_qk_norm_gradients(cuda_dev, name):
    """full fine-tuning: every parameter's gradient, q_norm / k_norm included, against autograd through HF; the norm weights
    round-trip through hf_state_dict / load_hf_state_dict under their HF names"""
    from test_full_ft_gpu import _batch, _compare_full_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _qwen3(name, 504, seed=14)
    sd = {k: v.to(bf16).float() for k, v in sd.items()}                 # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=False)
    batch = _batch(5, 12, 24, 40, 600, 504, seed=21)
    want = om.rag_step(bert, ref, batch)
    enc.full.zero_grad(); dec.full.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["losses"][2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    norm_names = [n for parts in dec._rows.values() for n, _ in parts if n.endswith(("q_norm.weight", "k_norm.weight"))]
    assert len(norm_names) == 2 * cfg["num_hidden_layers"]
    got = {}
    for key, parts in dec._rows.items():
        gw, r = dec.full.g(key), 0
        for n, rows in parts:
            got[n] = gw[r:r + rows]
            r += rows
    for n in norm_names:
        assert got[n].abs().max() > 0 and _rel(got[n], want["grads"]["generator." + n]) < 6e-2, n
    checked = _compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 8 * cfg["num_hidden_layers"] + 2
    hf = dec.hf_state_dict()
    assert set(hf) == set(sd) and all(torch.equal(hf[k], sd[k].float()) for k in norm_names)
    moved = {k: (v + 1.0 if k in norm_names else v) for k, v in hf.items()}
    dec.load_hf_state_dict(moved)
    assert all(torch.equal(dec.hf_state_dict()[k], moved[k]) for k in norm_names)


def test_autoregressive_qwen3_retriever(cuda_dev):
    """`is_autoregressive=True` with a Qwen3 model: last hidden state, eos pooling, LoRA on q_proj / v_proj"""
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import losses, models as om
    V = 504
    cfg, sd = _qwen3("qwen3-hd128", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    ref = build_qwen3(cfg, sd)
    _lora_init(enc, ref, 32)
    g = torch.Generator().manual_seed(32)
    model = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, is_autoregressive=True, _model=enc, _load_tokenizer=False)
    B, Lq, Lp = 4, 12, 20
    mk = lambda L: torch.ones(B, L, dtype=torch.int64)
    rb = {"query_input_ids": torch.randint(3, V, (B, Lq), generator=g), "query_attention_mask": mk(Lq),
          "passage_input_ids": torch.randint(3, V, (B, Lp), generator=g), "passage_attention_mask": mk(Lp)}
    rb["query_attention_mask"][0, :3] = 0; rb["passage_attention_mask"][2, :6] = 0
    q = om.retrieval_forward_autoregressive(ref, rb["query_input_ids"], rb["query_attention_mask"])
    p = om.retrieval_forward_autoregressive(ref, rb["passage_input_ids"], rb["passage_attention_mask"])
    loss = losses.contrastive_loss(losses.get_cosine_sim(q, p, 100.0))
    loss.backward()
    enc.lora.zero_grad()
    out = fused_retriever_step(model, rb, 100.0)
    assert abs(out["loss"].item() - loss.item()) / abs(loss.item()) < 2e-2
    worst = 0.0
    for n, _, _ in enc.lora.specs:
        mod = om._get_module(ref, n)
        worst = max(worst, _rel(enc.lora.gA[n], mod.lora_A.grad), _rel(enc.lora.gB[n], mod.lora_B.grad))
    assert worst < 8e-2, worst


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,lora", [("qwen3-tiny", 4, True), ("qwen3-hd128", 4, False), ("qwen3-hd128", 20, False)])
def test_qwen3_generate(cuda_dev, monkeypatch, name, B, lora):
    """per-step logits and choices vs HF teacher-forced on our tokens, bookkeeping bit-exact, graph replay == eager; the prefill
    and every decode step run the row kernel at explicit positions; B <= 16 decodes through decode_gemm, B = 20 through wgmma"""
    from test_generate_gpu import _check_against_oracle

    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _qwen3(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = build_qwen3(cfg, sd)
    if lora:
        _lora_init(dec, ref, 9)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, V, (B, 12), generator=g)
    mask = torch.ones(B, 12, dtype=torch.int64)
    mask[1, :3] = 0
    mask[2, 9:] = 0
    free, _ = _check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert free.shape == (B, 30)
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    _check_against_oracle(dec, ref, ids, mask, 30, eos, eos[0], monkeypatch)


@pytest.mark.parametrize("B", [4, 20])
def test_qwen3_generate_sampling_instruct_config(cuda_dev, monkeypatch, B):
    """an Instruct-style generation config (temperature 0.6, top-k 20, top-p 0.95, two EOS ids): sampled tokens are reproducible
    under torch.manual_seed and graph replay gives exactly the eager launches' tokens"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import decoding
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _qwen3("qwen3-hd128", V, seed=5)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    dec.generation_config = dict(synthetic.QWEN3_GENERATION["instruct"])
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(3, V, (B, 12), generator=g)
    mask = torch.ones(B, 12, dtype=torch.int64)
    mask[1, :3] = 0

    def gen(seed, graph):
        monkeypatch.setenv("DALM_B200_DECODE_GRAPH", graph)
        torch.manual_seed(seed)
        return dec.generate(input_ids=ids.to(cuda_dev), attention_mask=mask.to(cuda_dev), max_length=34, eos_token_id=[]).cpu()

    eager = gen(7, "0")
    assert eager.shape == (B, 34) and torch.equal(eager[:, :12], ids)
    assert torch.equal(gen(7, "0"), eager)
    replayed = gen(7, "1")
    assert decoding.LAST_RUN["graph_replays"] >= 4 and torch.equal(replayed, eager)


# ----------------------------------------------------------------------------------------------------------------
# trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_qwen3_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Qwen3 directory writes PEFT adapters; eval_rag loads them and
    decodes under the base-style (greedy) and the Instruct-style (sampling) generation config"""
    import csv as _csv
    import json
    import shutil

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    words = synthetic.word_list()
    csv = str(tmp_path / "short.csv")
    with open(csv, "w", newline="") as f:
        w = _csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for i in range(12):
            w.writerow({"Abstract": " ".join(words[20 + 6 * i:26 + 6 * i]), "Question": " ".join(words[200 + 4 * i:204 + 4 * i]),
                        "Answer": " ".join(words[400 + i:402 + i])})
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "qwen3-tiny"), "qwen3", "qwen3-tiny", vocab_size=1200, qk_norm_std=NORM_STD,
                                     generation_config=synthetic.QWEN3_GENERATION["base"])
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64,
              num_train_epochs=1, output_dir=out, use_peft=Mode.BOTH, num_warmup_steps=1, with_tracking=False)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out, sub, "adapter_model.bin"))
    sd = torch.load(os.path.join(out, "generator", "adapter_model.bin"), weights_only=True)
    assert any(v.abs().max() > 0 for k, v in sd.items() if "lora_B" in k)
    idir = str(tmp_path / "qwen3-tiny-instruct")                               # differs only in generation_config.json
    shutil.copytree(gdir, idir)
    with open(os.path.join(idir, "generation_config.json"), "w") as f:
        json.dump(synthetic.QWEN3_GENERATION["instruct"], f)
    for d in (gdir, idir):
        capsys.readouterr()
        torch.manual_seed(0)
        res = evaluate_rag(csv, rdir, d, os.path.join(out, "retriever"), os.path.join(out, "generator"), "Abstract", "Question",
                           "Answer", embed_dim=64, max_length=160, test_batch_size=4, query_batch_size=4, top_k=3,
                           evaluate_generator=True)
        text = capsys.readouterr().out
        assert res.total_examples == 12 and "Generator evaluation:" in text and "Exact match:" in text
