"""-m gpu: Qwen2 generators (Llama + q/k/v biases) and Llama with `attention_bias`.

Kernels: the bias in the two QKV epilogues that gained one (gemm_bf16_rope, decode_gemm), element by element under the rules
of test_exact_tiles_gpu.py (integer operands and biases, NaN-poisoned padding, guard bands); an all-zero bias must give what
bias=None gives. Models: forward / backward against transformers' Qwen2ForCausalLM / LlamaForCausalLM on bf16-rounded weights
with N(0, 0.5) biases (a dropped bias moves the logits far beyond bf16 noise), the fused RAG step, an autoregressive Qwen2
retriever, `generate` on both decode-GEMM paths, and the trainer + eval-rag end to end.
"""
import os

import pytest
import torch

from exact_helpers import Guarded, _expect_close, _expect_equal, _poisoned, _ulp_bf16
from test_exact_tiles_gpu import M_EDGE, _ints

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
BIAS_STD = 0.5


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def build_qwen2(cfg, sd):
    """transformers' Qwen2ForCausalLM, fp32, on the given HF-named weights (tied configs store no lm_head)"""
    from transformers import Qwen2Config, Qwen2ForCausalLM
    m = Qwen2ForCausalLM(Qwen2Config(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}))
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected and set(missing) <= ({"lm_head.weight"} if cfg.get("tie_word_embeddings") else set()), (missing, unexpected)
    return m.float().eval()


def _qwen2(name, V, seed):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.qwen2_config(name, vocab_size=V)
    sd = params.random_state_dict("qwen2", cfg, seed=seed, bias_std=BIAS_STD)
    return cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def _llama_ab(name, V, seed, bias_std=BIAS_STD):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = dict(synthetic.llama_config(name, vocab_size=V), attention_bias=True)
    sd = params.random_state_dict("llama", cfg, seed=seed, bias_std=bias_std)
    return cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}


def _ref_model(cfg, sd):
    from oracle import models as om
    return build_qwen2(cfg, sd) if cfg["model_type"] == "qwen2" else om.build_llama(cfg, sd)


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
    from test_exact_tiles_gpu import _gelu64
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
def _mask(B, L, pad):
    mask = torch.ones(B, L, dtype=torch.int64)
    if pad == "right":
        mask[0, L - 5:] = 0
    else:
        mask[0, :5] = 0; mask[1, :2] = 0
    return mask


@pytest.mark.parametrize("name,B,L,pad", [("qwen2-tiny", 3, 40, "right"), ("qwen2-tiny", 2, 33, "left"),
                                           ("qwen2-hd128", 2, 72, "left"), ("qwen2-hd128", 2, 130, "right")])
def test_qwen2_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs HF Qwen2ForCausalLM (qwen2-tiny: head_dim 64, RoPE pass after
    the GEMM, tied head; qwen2-hd128: head_dim 128, RoPE in the QKV epilogue, untied)"""
    from dalm_b200 import ops
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import losses, models as om
    V = 504
    cfg, sd = _qwen2(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    assert dec.fuse_rope == (name == "qwen2-hd128")
    g = torch.Generator().manual_seed(9)
    for n, _, _ in dec.lora.specs:
        dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(cuda_dev))
    dec.repack_lora()
    ref = build_qwen2(cfg, sd)
    om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})
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


@pytest.mark.parametrize("name,pad", [("llama-tiny", "right"), ("llama-hd128", "left")])
def test_llama_attention_bias_forward(cuda_dev, name, pad):
    """a Llama config with attention_bias: q/k/v and o_proj biases are all applied (they used to be ignored)"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 512
    cfg, sd = _llama_ab(name, V, seed=4)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    assert dec.qkv_bias and dec.o_bias
    ref = _ref_model(cfg, sd)
    g = torch.Generator().manual_seed(10)
    B, L = 2, 72
    ids = torch.randint(3, V, (B, L), generator=g)
    mask = _mask(B, L, pad)
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev))
    with torch.no_grad():
        ref_logits = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert _rel(logits.float().cpu()[valid], ref_logits[valid]) < 1.5e-2


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
    bert, ref = om.build_bert(bcfg, bsd), _ref_model(gcfg, gsd)
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


@pytest.mark.parametrize("name,pad", [("qwen2-tiny", "left"), ("qwen2-hd128", "right")])
def test_fused_rag_step_qwen2_lora(cuda_dev, name, pad):
    """bge + Qwen2 generator, LoRA on both: the fused training step against the reference loop body"""
    from test_step_gpu import _batch, _check_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _qwen2(name, 504, seed=12)
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=True)
    batch = _batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad)
    want = om.rag_step(bert, ref, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    got = out["losses"].cpu()
    assert abs(got[2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    _check_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("kind,name", [("qwen2", "qwen2-tiny"), ("qwen2", "qwen2-hd128"), ("llama", "llama-tiny")])
def test_full_finetune_bias_gradients(cuda_dev, kind, name):
    """full fine-tuning: every parameter's gradient, the attention biases included, against autograd through HF; the biases
    round-trip through hf_state_dict / load_hf_state_dict under their HF names"""
    from test_full_ft_gpu import _batch, _compare_full_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    # llama-tiny's q = h Wq is ~0.2 in size: biases of 0.5 would make every query alike and the k gradients vanish into
    # cancellation, so this case draws its biases at std 0.1
    cfg, sd = _qwen2(name, 504, seed=14) if kind == "qwen2" else _llama_ab(name, 504, seed=14, bias_std=0.1)
    sd = {k: v.to(bf16).float() for k, v in sd.items()}                 # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=False)
    batch = _batch(5, 12, 24, 40, 600, 504, seed=21)
    want = om.rag_step(bert, ref, batch)
    enc.full.zero_grad(); dec.full.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["losses"][2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    bias_names = [n for parts in dec._rows.values() for n, _ in parts if n.endswith(".bias")]
    expect = 3 if kind == "qwen2" else 4
    assert len(bias_names) == expect * cfg["num_hidden_layers"]
    got = dict(_full_grads(dec))
    for n in bias_names:
        if kind == "qwen2" or n.endswith("o_proj.bias"):
            assert _rel(got[n], want["grads"]["generator." + n]) < 6e-2, n
        else:
            # llama-tiny's q/k/v bias gradients are sums over tokens that largely cancel, so the bf16 rounding of d(qkv) makes
            # their relative error large; their error is bounded against the o_proj bias gradient of the same layer
            o = n.rsplit(".", 2)[0] + ".o_proj.bias"
            err = (got[n].double().cpu() - want["grads"]["generator." + n].double()).norm()
            assert err / want["grads"]["generator." + o].double().norm() < 6e-2, n
    loose = () if kind == "qwen2" else tuple(n for n in bias_names if not n.endswith("o_proj.bias"))
    checked = _compare_full_grads(dec, want["grads"], "generator.", skip=loose)
    assert checked >= 6 * cfg["num_hidden_layers"] + 2
    hf = dec.hf_state_dict()
    assert set(hf) == set(sd) and all(torch.equal(hf[k], sd[k].float()) for k in bias_names)
    moved = {k: (v + 1.0 if k.endswith(".bias") else v) for k, v in hf.items()}
    dec.load_hf_state_dict(moved)
    assert all(torch.equal(dec.hf_state_dict()[k], moved[k]) for k in bias_names)


def _full_grads(dec):
    for key, parts in dec._rows.items():
        gw, r = dec.full.g(key), 0
        for name, rows in parts:
            yield name, gw[r:r + rows]
            r += rows


def test_autoregressive_qwen2_retriever(cuda_dev):
    """`is_autoregressive=True` with a Qwen2 model: last hidden state, eos pooling, LoRA on q_proj / v_proj"""
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import losses, models as om
    V = 504
    cfg, sd = _qwen2("qwen2-tiny", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    g = torch.Generator().manual_seed(32)
    for n, _, _ in enc.lora.specs:
        enc.lora.B[n].copy_((torch.randn(enc.lora.B[n].shape, generator=g) * 0.02).to(cuda_dev))
    enc.repack_lora()
    model = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, is_autoregressive=True, _model=enc, _load_tokenizer=False)
    ref = build_qwen2(cfg, sd)
    om.attach_lora(ref, {n: {"A": enc.lora.A[n].cpu(), "B": enc.lora.B[n].cpu()} for n, _, _ in enc.lora.specs})
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
@pytest.mark.parametrize("name,B,lora", [("qwen2-tiny", 4, True), ("qwen2-hd128", 4, False), ("qwen2-hd128", 20, False)])
def test_qwen2_generate(cuda_dev, monkeypatch, name, B, lora):
    """per-step logits and choices vs HF teacher-forced on our tokens, bookkeeping bit-exact, graph replay == eager; B <= 16
    decodes through decode_gemm's bias, B = 20 through the wgmma GEMM's"""
    from test_generate_gpu import _check_against_oracle

    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 504
    cfg, sd = _qwen2(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = build_qwen2(cfg, sd)
    if lora:
        g = torch.Generator().manual_seed(9)
        for n, _, _ in dec.lora.specs:
            dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(cuda_dev))
        dec.repack_lora()
        om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, V, (B, 12), generator=g)
    mask = torch.ones(B, 12, dtype=torch.int64)
    mask[1, :3] = 0
    mask[2, 9:] = 0
    free, _ = _check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert free.shape == (B, 30)
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    _check_against_oracle(dec, ref, ids, mask, 30, eos, eos[0], monkeypatch)


# ----------------------------------------------------------------------------------------------------------------
# trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_qwen2_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Qwen2 directory writes PEFT adapters; eval_rag loads them
    and decodes greedily under a base-style generation config; an Instruct-style config asks for repetition_penalty, which
    is refused by name"""
    import csv as _csv
    import json
    import shutil

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    words = synthetic.word_list()
    csv = str(tmp_path / "short.csv")                                           # prompts well inside max_length
    with open(csv, "w", newline="") as f:
        w = _csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for i in range(12):
            w.writerow({"Abstract": " ".join(words[20 + 6 * i:26 + 6 * i]), "Question": " ".join(words[200 + 4 * i:204 + 4 * i]),
                        "Answer": " ".join(words[400 + i:402 + i])})
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "qwen2-tiny"), "qwen2", "qwen2-tiny", vocab_size=1200, bias_std=BIAS_STD,
                                     generation_config=synthetic.QWEN2_GENERATION["base"])
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64,
              num_train_epochs=1, output_dir=out, use_peft=Mode.BOTH, num_warmup_steps=1, with_tracking=False)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out, sub, "adapter_model.bin"))
    sd = torch.load(os.path.join(out, "generator", "adapter_model.bin"), weights_only=True)
    assert any(v.abs().max() > 0 for k, v in sd.items() if "lora_B" in k)
    capsys.readouterr()
    res = evaluate_rag(csv, rdir, gdir, os.path.join(out, "retriever"), os.path.join(out, "generator"), "Abstract", "Question",
                       "Answer", embed_dim=64, max_length=160, test_batch_size=4, query_batch_size=4, top_k=3,
                       evaluate_generator=True)
    text = capsys.readouterr().out
    assert res.total_examples == 12 and "Generator evaluation:" in text and "Exact match:" in text
    idir = str(tmp_path / "qwen2-tiny-instruct")                               # differs only in generation_config.json
    shutil.copytree(gdir, idir)
    with open(os.path.join(idir, "generation_config.json"), "w") as f:
        json.dump(synthetic.QWEN2_GENERATION["instruct"], f)
    with pytest.raises(NotImplementedError, match="repetition_penalty"):
        evaluate_rag(csv, rdir, idir, None, None, "Abstract", "Question", "Answer", embed_dim=64, max_length=160,
                     test_batch_size=4, query_batch_size=4, top_k=3, evaluate_generator=True)
