"""-m gpu: Qwen2 generators (Llama + q/k/v biases) and Llama with `attention_bias`.

Kernels: the bias in the two QKV epilogues that gained one (gemm_bf16_rope, decode_gemm), element by element under the rules
of test_exact_tiles_gpu.py (integer operands and biases, NaN-poisoned padding, guard bands); an all-zero bias must give what
bias=None gives. Models: forward / backward against transformers' Qwen2ForCausalLM / LlamaForCausalLM on bf16-rounded weights
with N(0, 0.5) biases (a dropped bias moves the logits far beyond bf16 noise), the fused RAG step, an autoregressive Qwen2
retriever, `generate` on both decode-GEMM paths, and the trainer + eval-rag end to end.
"""
import pytest
import torch

from exact_helpers import M_EDGE, Guarded, _expect_close, _expect_equal, _gelu64, _ints, _poisoned, _ulp_bf16
from model_helpers import (attach_lora, check_against_oracle, check_autoregressive_retriever, check_decoder, check_rag_lora_grads,
                           compare_full_grads, draw_lora_B, eval_rag_generator, full_grads, instruct_copy, pad_mask, prompt, r16,
                           r16_2d, rag_batch, rag_models, rag_step_vs_oracle, rel, toy_rag_inputs, train_rag_lora)

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
BIAS_STD = 0.5


def _qwen2(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.qwen2_config(name, vocab_size=V)
    return cfg, r16_2d(params.random_state_dict("qwen2", cfg, seed=seed, bias_std=BIAS_STD))


def _llama_ab(name, V, seed, bias_std=BIAS_STD):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = dict(synthetic.llama_config(name, vocab_size=V), attention_bias=True)
    return cfg, r16_2d(params.random_state_dict("llama", cfg, seed=seed, bias_std=bias_std))


# ----------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------
def test_gemm_rope_bias_exact(cuda_dev):
    """bias added to the fp32 accumulator before the rotation: rotated columns within one bf16 ulp (+ the fp32 rounding of
    the sin product), v columns bit-exact; an all-zero bias gives what bias=None gives"""
    from dalm_b200 import ops
    dev = cuda_dev
    Lr = 37
    inv = 1.0 / (1e6 ** (torch.arange(0, 128, 2, dtype=f32) / 128))
    fr = torch.outer(torch.arange(Lr, dtype=f32), inv)
    cbuf = torch.full((Lr + 128, 64), float("nan"), device=dev); cbuf[:Lr] = fr.cos().to(dev)
    sbuf = torch.full((Lr + 128, 64), float("nan"), device=dev); sbuf[:Lr] = fr.sin().to(dev)
    cos_t, sin_t = cbuf[:Lr], sbuf[:Lr]
    i = 0
    for M in M_EDGE:
        for N, rope_cols in ((264, 256), (512, 512), (520, 512), (1792 + 256, 1792)):
            for K in (8, 72):
                g = torch.Generator().manual_seed(700 + i)
                a = _poisoned(_ints((M, K), g).to(dev, bf16))
                w = _poisoned(_ints((N, K), g).to(dev, bf16))
                bias = _poisoned(_ints((N,), g, hi=64).to(dev))
                out = Guarded(M, N, bf16, dev)
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=out.view, bias=bias)
                what = f"gemm_rope+bias M {M} N {N} K {K} rope_cols {rope_cols}"
                y = a.double() @ w.double().t() + bias.double()[None]                  # exact in fp32 too
                pos = torch.arange(M, device=dev) % Lr
                c, s = cos_t.double()[pos][:, None], sin_t.double()[pos][:, None]
                h = y[:, :rope_cols].reshape(M, rope_cols // 128, 2, 64)
                x1, x2 = h[:, :, 0], h[:, :, 1]
                rot = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).view(M, rope_cols)
                terms = torch.stack([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], 2).view(M, rope_cols)
                _expect_close(out.view[:, :rope_cols], rot, _ulp_bf16(rot) + 2.0 ** -22 * terms, what + " rotated", 128, 256)
                _expect_equal(out.view[:, rope_cols:], y[:, rope_cols:].to(bf16), what + " plain", 128, 256)
                out.check(what)
                # zero bias == no bias, element for element (+0 == -0)
                o0, o1 = Guarded(M, N, bf16, dev), Guarded(M, N, bf16, dev)
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=o0.view, bias=_poisoned(torch.zeros(N, device=dev)))
                ops.gemm_rope(a, w, cos_t, sin_t, Lr, rope_cols, out=o1.view)
                _expect_equal(o0.view, o1.view, what + " zero bias vs none", 128, 256)
                o0.check(what + " zero bias")
                i += 1


@pytest.mark.parametrize("M", [1, 7, 16])
def test_decode_gemm_bias_exact(cuda_dev, M):
    """out = act(A W^T + bias) + resid on ragged N / K: fp32 outputs equal fp64, bf16 outputs its rounding, GELU within one
    fp32-evaluation tolerance; an all-zero bias gives what bias=None gives"""
    from dalm_b200 import ops
    dev = cuda_dev
    for j, (N, K) in enumerate(((13, 8), (264, 72), (1000, 520), (2056, 3584))):
        g = torch.Generator().manual_seed(900 + 31 * M + j)
        a = _poisoned(_ints((M, K), g).to(dev, bf16))
        w = _poisoned(_ints((N, K), g).to(dev, bf16))
        bias = _poisoned(_ints((N,), g, hi=4096).to(dev))
        r32 = _poisoned(_ints((M, N), g, hi=2048).to(dev))
        y = a.double() @ w.double().t() + bias.double()[None]
        what = f"decode_gemm+bias M {M} N {N} K {K}"
        o = Guarded(M, N, f32, dev)
        ops.decode_gemm(a, w, out=o.view, bias=bias)
        _expect_equal(o.view, y.to(f32), what + " fp32", 16, 16); o.check(what + " fp32")
        o = Guarded(M, N, bf16, dev)
        ops.decode_gemm(a, w, out=o.view, bias=bias)
        _expect_equal(o.view, y.to(bf16), what + " bf16", 16, 16); o.check(what + " bf16")
        o = Guarded(M, N, f32, dev)
        ops.decode_gemm(a, w, out=o.view, bias=bias, resid=r32)
        _expect_equal(o.view, (y + r32.double()).to(f32), what + " +resid", 16, 16); o.check(what + " +resid")
        o = Guarded(M, N, f32, dev)
        ops.decode_gemm(a, w, out=o.view, bias=bias / 1024, act=1)                # GELU where it is not ~identity / zero
        pre = a.double() @ w.double().t() + (bias / 1024).double()[None]
        ref = _gelu64(pre)
        _expect_close(o.view, ref, 4 * 2.0 ** -23 * (pre.abs() + 1), what + " gelu", 16, 16); o.check(what + " gelu")
        o0, o1 = Guarded(M, N, bf16, dev), Guarded(M, N, bf16, dev)
        ops.decode_gemm(a, w, out=o0.view, bias=_poisoned(torch.zeros(N, device=dev)))
        ops.decode_gemm(a, w, out=o1.view)
        _expect_equal(o0.view, o1.view, what + " zero bias vs none", 16, 16); o0.check(what + " zero bias")
        # gemm_rows routes the bias to whichever row path it picks
        assert torch.equal(ops.gemm_rows(a, w, bias=bias, out_dtype=f32), y.to(f32))
    a = _poisoned(_ints((40, 72), g).to(dev, bf16))
    w = _poisoned(_ints((264, 72), g).to(dev, bf16))
    assert torch.equal(ops.gemm_rows(a, w, bias=bias[:264], out_dtype=f32), (a.double() @ w.double().t() + bias[:264].double()).to(f32))


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,L,pad", [("qwen2-tiny", 3, 40, "right"), ("qwen2-tiny", 2, 33, "left"),
                                           ("qwen2-hd128", 2, 72, "left"), ("qwen2-hd128", 2, 130, "right")])
def test_qwen2_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF Qwen2ForCausalLM (qwen2-tiny: head_dim 64, RoPE pass after
    the GEMM, tied head; qwen2-hd128: head_dim 128, RoPE in the QKV epilogue, untied)"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen2(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    assert dec.fuse_rope == (name == "qwen2-hd128")
    g = torch.Generator().manual_seed(9)
    draw_lora_B(dec, g)
    ref = om.build_causal_lm(cfg, sd)
    attach_lora(ref, dec)
    check_decoder(dec, ref, g, V, B, L, pad)                              # the ids continue the LoRA draws' generator


@pytest.mark.parametrize("name,pad", [("llama-tiny", "right"), ("llama-hd128", "left")])
def test_llama_attention_bias_forward(cuda_dev, name, pad):
    """a Llama config with attention_bias: q/k/v and o_proj biases are all applied (they used to be ignored)"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 512
    cfg, sd = _llama_ab(name, V, seed=4)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    assert dec.qkv_bias and dec.o_bias
    ref = om.build_llama(cfg, sd)
    g = torch.Generator().manual_seed(10)
    B, L = 2, 72
    ids = torch.randint(3, V, (B, L), generator=g)
    mask = pad_mask(B, L, pad)
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev))
    with torch.no_grad():
        ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2


@pytest.mark.parametrize("name,pad", [("qwen2-tiny", "left"), ("qwen2-hd128", "right")])
def test_fused_rag_step_qwen2_lora(cuda_dev, name, pad):
    """bge + Qwen2 generator, LoRA on both: the fused training step against the reference loop body"""
    cfg, sd = _qwen2(name, 504, seed=12)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad))
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("kind,name", [("qwen2", "qwen2-tiny"), ("qwen2", "qwen2-hd128"), ("llama", "llama-tiny")])
def test_full_finetune_bias_gradients(cuda_dev, kind, name):
    """full fine-tuning: every parameter's gradient, the attention biases included, against autograd through HF; the biases
    round-trip through hf_state_dict / load_hf_state_dict under their HF names"""
    # llama-tiny's q = h Wq is ~0.2 in size: biases of 0.5 would make every query alike and the k gradients vanish into
    # cancellation, so this case draws its biases at std 0.1
    cfg, sd = _qwen2(name, 504, seed=14) if kind == "qwen2" else _llama_ab(name, 504, seed=14, bias_std=0.1)
    sd = r16(sd)                                                          # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, lora_r=False, lora_g=False)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 40, 600, 504, seed=21))
    bias_names = [n for parts in dec._rows.values() for n, _ in parts if n.endswith(".bias")]
    expect = 3 if kind == "qwen2" else 4
    assert len(bias_names) == expect * cfg["num_hidden_layers"]
    got = full_grads(dec)
    for n in bias_names:
        if kind == "qwen2" or n.endswith("o_proj.bias"):
            assert rel(got[n], want["grads"]["generator." + n]) < 6e-2, n
        else:
            # llama-tiny's q/k/v bias gradients are sums over tokens that largely cancel, so the bf16 rounding of d(qkv) makes
            # their relative error large; their error is bounded against the o_proj bias gradient of the same layer
            o = n.rsplit(".", 2)[0] + ".o_proj.bias"
            err = (got[n].double().cpu() - want["grads"]["generator." + n].double()).norm()
            assert err / want["grads"]["generator." + o].double().norm() < 6e-2, n
    loose = () if kind == "qwen2" else tuple(n for n in bias_names if not n.endswith("o_proj.bias"))
    checked = compare_full_grads(dec, want["grads"], "generator.", skip=loose)
    assert checked >= 6 * cfg["num_hidden_layers"] + 2
    hf = dec.hf_state_dict()
    assert set(hf) == set(sd) and all(torch.equal(hf[k], sd[k].float()) for k in bias_names)
    moved = {k: (v + 1.0 if k.endswith(".bias") else v) for k, v in hf.items()}
    dec.load_hf_state_dict(moved)
    assert all(torch.equal(dec.hf_state_dict()[k], moved[k]) for k in bias_names)


def test_autoregressive_qwen2_retriever(cuda_dev):
    """`is_autoregressive=True` with a Qwen2 model: last hidden state, eos pooling, LoRA on q_proj / v_proj"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen2("qwen2-tiny", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    g = torch.Generator().manual_seed(32)
    draw_lora_B(enc, g)
    ref = om.build_causal_lm(cfg, sd)
    attach_lora(ref, enc)
    check_autoregressive_retriever(enc, ref, g, V, 12, 20)                # the ids continue the LoRA draws' generator


# ----------------------------------------------------------------------------------------------------------------
# generate
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,lora", [("qwen2-tiny", 4, True), ("qwen2-hd128", 4, False), ("qwen2-hd128", 20, False)])
def test_qwen2_generate(cuda_dev, monkeypatch, name, B, lora):
    """per-step logits and choices vs HF teacher-forced on our tokens, bookkeeping bit-exact, graph replay == eager; B <= 16
    decodes through decode_gemm's bias, B = 20 through the wgmma GEMM's"""
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen2(name, V, seed=2)
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


# ----------------------------------------------------------------------------------------------------------------
# trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_qwen2_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Qwen2 directory writes PEFT adapters; eval_rag loads them
    and decodes greedily under a base-style generation config; an Instruct-style config asks for repetition_penalty, which
    is refused by name"""
    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / "qwen2-tiny"), "qwen2", "qwen2-tiny", vocab_size=1200, bias_std=BIAS_STD,
                                     generation_config=synthetic.QWEN2_GENERATION["base"])
    out = train_rag_lora(csv, rdir, gdir, tmp_path)
    eval_rag_generator(csv, rdir, gdir, out, capsys)
    idir = instruct_copy(gdir, str(tmp_path / "qwen2-tiny-instruct"), synthetic.QWEN2_GENERATION["instruct"])
    with pytest.raises(NotImplementedError, match="repetition_penalty"):
        evaluate_rag(csv, rdir, idir, None, None, "Abstract", "Question", "Answer", embed_dim=64, max_length=160,
                     test_batch_size=4, query_batch_size=4, top_k=3, evaluate_generator=True)
