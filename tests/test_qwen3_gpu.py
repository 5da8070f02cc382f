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
import pytest
import torch

from exact_helpers import (EPS, M_EDGE, NORM_STD, Guarded, _expect_close, _expect_equal, _ints, _norm_w, _poisoned, _ref_norm_rope,
                           _tables, _ulp_bf16, _ulp_f32)
from model_helpers import (attach_lora, check_against_oracle, check_autoregressive_retriever, check_decoder, check_rag_lora_grads,
                           compare_full_grads, draw_lora_B, eval_rag_generator, full_grads, instruct_copy, prompt, r16, r16_2d,
                           rag_batch, rag_models, rag_step_vs_oracle, rel, toy_rag_inputs, train_rag_lora)

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64


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
def _qwen3(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.qwen3_config(name, vocab_size=V)
    return cfg, r16_2d(params.random_state_dict("qwen3", cfg, seed=seed, qk_norm_std=NORM_STD))


@pytest.mark.parametrize("name,B,L,pad", [("qwen3-tiny", 3, 40, "right"), ("qwen3-tiny", 2, 33, "left"),
                                           ("qwen3-hd128", 2, 72, "left"), ("qwen3-hd128", 2, 130, "right")])
def test_qwen3_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF Qwen3ForCausalLM (qwen3-tiny: 5 q|k heads, the row kernel,
    tied head; qwen3-hd128: 8 q|k heads, q/k norm + RoPE in the QKV epilogue, untied)"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen3(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    assert dec.qk_norm and dec.fuse_rope and (((dec.nh + dec.nkv) * 128) % 256 == 0) == (name == "qwen3-hd128")
    ref = om.build_causal_lm(cfg, sd)
    draw_lora_B(dec, torch.Generator().manual_seed(9))
    attach_lora(ref, dec)
    check_decoder(dec, ref, torch.Generator().manual_seed(9), V, B, L, pad)


@pytest.mark.parametrize("name,pad", [("qwen3-tiny", "left"), ("qwen3-hd128", "right")])
def test_fused_rag_step_qwen3_lora(cuda_dev, name, pad):
    """bge + Qwen3 generator, LoRA on both: the fused training step against the reference loop body"""
    cfg, sd = _qwen3(name, 504, seed=12)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad))
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["qwen3-tiny", "qwen3-hd128"])
def test_full_finetune_qk_norm_gradients(cuda_dev, name):
    """full fine-tuning: every parameter's gradient, q_norm / k_norm included, against autograd through HF; the norm weights
    round-trip through hf_state_dict / load_hf_state_dict under their HF names"""
    cfg, sd = _qwen3(name, 504, seed=14)
    sd = r16(sd)                                                          # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, lora_r=False, lora_g=False)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 40, 600, 504, seed=21))
    norm_names = [n for parts in dec._rows.values() for n, _ in parts if n.endswith(("q_norm.weight", "k_norm.weight"))]
    assert len(norm_names) == 2 * cfg["num_hidden_layers"]
    got = full_grads(dec)
    for n in norm_names:
        assert got[n].abs().max() > 0 and rel(got[n], want["grads"]["generator." + n]) < 6e-2, n
    checked = compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 8 * cfg["num_hidden_layers"] + 2
    hf = dec.hf_state_dict()
    assert set(hf) == set(sd) and all(torch.equal(hf[k], sd[k].float()) for k in norm_names)
    moved = {k: (v + 1.0 if k in norm_names else v) for k, v in hf.items()}
    dec.load_hf_state_dict(moved)
    assert all(torch.equal(dec.hf_state_dict()[k], moved[k]) for k in norm_names)


def test_autoregressive_qwen3_retriever(cuda_dev):
    """`is_autoregressive=True` with a Qwen3 model: last hidden state, eos pooling, LoRA on q_proj / v_proj"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen3("qwen3-hd128", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    ref = om.build_causal_lm(cfg, sd)
    draw_lora_B(enc, torch.Generator().manual_seed(32))
    attach_lora(ref, enc)
    check_autoregressive_retriever(enc, ref, torch.Generator().manual_seed(32), V, 12, 20)


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,lora", [("qwen3-tiny", 4, True), ("qwen3-hd128", 4, False), ("qwen3-hd128", 20, False)])
def test_qwen3_generate(cuda_dev, monkeypatch, name, B, lora):
    """per-step logits and choices vs HF teacher-forced on our tokens, bookkeeping bit-exact, graph replay == eager; the prefill
    and every decode step run the row kernel at explicit positions; B <= 16 decodes through decode_gemm, B = 20 through wgmma"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen3(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = om.build_causal_lm(cfg, sd)
    if lora:
        draw_lora_B(dec, torch.Generator().manual_seed(9))
        attach_lora(ref, dec)
    ids, mask = prompt(B, 12, V, seed=1)
    free, _ = check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert free.shape == (B, 30)
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    check_against_oracle(dec, ref, ids, mask, 30, eos, eos[0], monkeypatch)


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
    from dalm_b200 import synthetic
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / "qwen3-tiny"), "qwen3", "qwen3-tiny", vocab_size=1200, qk_norm_std=NORM_STD,
                                     generation_config=synthetic.QWEN3_GENERATION["base"])
    out = train_rag_lora(csv, rdir, gdir, tmp_path)
    idir = instruct_copy(gdir, str(tmp_path / "qwen3-tiny-instruct"), synthetic.QWEN3_GENERATION["instruct"])
    for d in (gdir, idir):
        torch.manual_seed(0)
        eval_rag_generator(csv, rdir, d, out, capsys)
