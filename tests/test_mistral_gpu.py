"""-m gpu: sliding-window causal attention (Mistral; Qwen2 / Qwen3 with use_sliding_window) in the training and decode kernels,
and Mistral generators and retrievers against transformers.

Kernels: query i sees key j iff j <= i and i - j < window (transformers' `sliding_window_overlay`, counted in the padded row).
Random inputs are checked row by row against fp64 with the bounds of test_exact_tiles_gpu.test_attention_rows_vs_fp64, on
poisoned inputs and guarded outputs. A window >= L is no window, and must give the bits of window = 0; the decode kernel must
give the bits of window = 0 while the window still covers every column.

Models: whole decoders against transformers' MistralForCausalLM (eager attention, fp32, the same bf16-rounded weights) at
sequence lengths 2-3x the window. The q / k projections are drawn 2.5x wider than initializer_range so that attention is
peaked and depends on which keys are visible: the same decoder without its window then misses the logits by 10x the tolerance
(the control). Tolerances are those of test_llama3_gpu.py.
"""
import math

import pytest
import torch

from exact_helpers import Guarded, _attn_bwd64, _attn_fns, _attn_ref64, _expect_close, _poisoned, _row_mask, dev, ops  # noqa: F401
from model_helpers import (attach_lora, check_against_oracle, check_autoregressive_retriever, check_decoder, check_rag_lora_grads,
                           compare_full_grads, draw_lora_B, eval_rag_generator, hf_generate_agreement, hf_grads, lora_grad_error,
                           pad_mask, prompt, r16, r16_2d, rag_batch, rag_models, rag_step_vs_oracle, rel, toy_rag_inputs,
                           train_rag_lora)

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64
QK_SCALE = 2.5


def _visible_win(mask, L, window):
    """[B, 1, Lq, Lk] visibility: key-padding mask, causal, and j > i - window when window > 0"""
    i = torch.arange(L, device=mask.device)
    band = i[None, :] <= i[:, None]
    if window > 0:
        band = band & (i[None, :] > i[:, None] - window)
    return mask.bool()[:, None, None, :] & band


# ----------------------------------------------------------------------------------------------------------------
# 1. attention kernels against fp64
# ----------------------------------------------------------------------------------------------------------------
KINDS = [("wg", 64), ("wg", 128), ("mma", 32), ("mma", 64), ("mma", 128)]
LENGTHS = (63, 65, 128, 200, 257)
PATTERNS = ("right64", "left64", "holes", "empty")
HEADS = ((4, 4), (4, 2), (4, 1))                          # MHA, GQA, MQA


def _window_params():
    out, n = [], 0
    for kind, D in KINDS:
        for L in LENGTHS:
            for w in (1, 17, 63, 64, 65, 100, L, L + 5):
                Hq, Hkv = HEADS[n % 3]
                out.append((kind, D, L, w, PATTERNS[n % 4], Hq, Hkv))
                n += 1
    return out


def _run_attn(ops, dev, kind, D, B, L, Hq, Hkv, mask, window, seed, scale=None):
    g = torch.Generator().manual_seed(seed)
    q0 = torch.randn(B * L, Hq * D, generator=g).to(bf16)
    k0 = torch.randn(B * L, Hkv * D, generator=g).to(bf16)
    v0 = torch.randn(B * L, Hkv * D, generator=g).to(bf16)
    do0 = torch.randn(B * L, Hq * D, generator=g).to(bf16)
    q, k, v, d_out = (_poisoned(t.to(dev)) for t in (q0, k0, v0, do0))
    fwd, bwd = _attn_fns(ops, kind)
    out = Guarded(B * L, Hq * D, bf16, dev)
    _, lse = fwd(q, k, v, mask, B, L, Hq, Hkv, D, True, out=out.view, scale=scale, window=window)
    dq, dk, dv = Guarded(B * L, Hq * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev), Guarded(B * L, Hkv * D, bf16, dev)
    bwd(q, k, v, mask, out.view, lse, d_out, B, L, Hq, Hkv, D, True, dq=dq.view, dk=dk.view, dv=dv.view, scale=scale, window=window)
    return (q, k, v, d_out), out, lse, dq, dk, dv


@pytest.mark.parametrize("kind,D,L,window,pattern,Hq,Hkv", _window_params())
def test_window_attention_rows_vs_fp64(ops, dev, kind, D, L, window, pattern, Hq, Hkv):
    """forward and backward with a sliding window, every row against fp64: windows shorter than one key tile, exactly one
    tile, across tile edges and wider than the sequence; fully masked KV tiles, >= 64 left-pad tokens, interior holes and
    a sample with every key masked (rows without a visible key: zero output, lse = +inf, zero gradients)"""
    B = 3
    g = torch.Generator().manual_seed(L * 131 + D + window)
    mask = _row_mask(B, L, pattern, g).to(dev)
    sc = 1.0 / math.sqrt(D)
    (q, k, v, d_out), out, lse, dq, dk, dv = _run_attn(ops, dev, kind, D, B, L, Hq, Hkv, mask, window, seed=L + 7 * window)
    what = f"{kind} attention D {D} L {L} window {window} {pattern} Hq {Hq} Hkv {Hkv}"
    vis = _visible_win(mask, L, window)
    qd, kd, vd = (t.double() for t in (q, k, v))
    ref, lse_ref = _attn_ref64(qd, kd, vd, vis, B, L, Hq, Hkv, D, sc)
    for name, t in (("out", out.view), ("lse", lse), ("dq", dq.view), ("dk", dk.view), ("dv", dv.view)):
        assert not torch.isnan(t).any(), f"{what}: NaN in {name}"
    vmax = v.double().abs().view(B, L, Hkv, D).amax((1, 3)).repeat_interleave(Hq // Hkv, 1)
    tol = (vmax[:, None, :, None] / 128).expand(B, L, Hq, D).reshape(B * L, Hq * D)
    _expect_close(out.view, ref, tol, what + " out", 64)
    valid = vis.expand(B, Hq, L, L).any(-1)
    assert (torch.isinf(lse[~valid]) & (lse[~valid] > 0)).all(), f"{what}: rows without a visible key need lse = +inf"
    lerr = (lse.double() - lse_ref).abs()[valid]
    assert lerr.max() < 1e-4, f"{what}: lse off by {lerr.max().item():.3e}"
    # backward: the kernels' algorithm in fp64, including delta = rowsum(dO * O) from the bf16 output the forward wrote. With
    # one or two visible keys dP - delta cancels, and the exact-O gradient would measure that rounding of O, not the kernel.
    want = _attn_bwd64(qd, kd, vd, d_out.double(), out.view.double(), vis, B, L, Hq, Hkv, D, sc)
    no_query = (~valid).permute(0, 2, 1).reshape(B * L, Hq)
    # key j is always visible to query j itself, so only masked keys have zero dK / dV
    masked_key = (mask == 0).reshape(B * L, 1).expand(B * L, Hkv)
    floor = None
    for name, got, w, H, zero in (("dv", dv.view, want[2], Hkv, masked_key), ("dq", dq.view, want[0], Hq, no_query),
                                  ("dk", dk.view, want[1], Hkv, masked_key)):
        gr, wr = got.double().view(B * L, H, D), w.view(B * L, H, D)
        err, nrm = (gr - wr).norm(dim=-1), wr.norm(dim=-1)
        med = nrm[~zero].median()
        if floor is None:        # dV never cancels; 1e-4 of its median row bounds the fp32 noise where dS is exactly 0 (window 1)
            floor = 1e-4 * med
        lim = 0.04 * nrm + 0.01 * med + floor
        bad = err > lim
        if bad.any():
            r, h = bad.nonzero()[0].tolist()
            pytest.fail(f"{what}: {name} {int(bad.sum())} bad rows; first token {r} (sample {r // L}, position {r % L}) head {h}: "
                        f"error {err[r, h].item():.3e} vs row norm {nrm[r, h].item():.3e}")
        assert (gr[zero] == 0).all(), f"{what}: {name} nonzero where every contribution is masked"
    for name, gd in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
        gd.check(f"{what} {name}")


@pytest.mark.parametrize("kind,D", KINDS)
@pytest.mark.parametrize("L", [65, 200, 257])
def test_wide_window_is_bit_identical_to_none(ops, dev, kind, D, L):
    """window >= L masks nothing and skips no tile: out, lse, dq, dk, dv bit-equal to window = 0"""
    B, Hq, Hkv = 3, 4, 2
    mask = _row_mask(B, L, "holes", torch.Generator().manual_seed(L)).to(dev)
    base = _run_attn(ops, dev, kind, D, B, L, Hq, Hkv, mask, 0, seed=L)
    for w in (L, L + 5, 1 << 30):
        got = _run_attn(ops, dev, kind, D, B, L, Hq, Hkv, mask, w, seed=L)
        for name, a, b in (("out", got[1].view, base[1].view), ("lse", got[2], base[2]), ("dq", got[3].view, base[3].view),
                           ("dk", got[4].view, base[4].view), ("dv", got[5].view, base[5].view)):
            assert torch.equal(a, b), f"{kind} D {D} L {L} window {w}: {name} differs from window 0"


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("L,window", [(200, 65), (257, 17), (130, 64)])
def test_window_wg_agrees_with_mma(ops, dev, D, L, window):
    """the wgmma / TMA kernels and the mma.sync kernels compute the same windowed attention"""
    B, Hq, Hkv = 2, 4, 2
    mask = _row_mask(B + 1, L, "left64", torch.Generator().manual_seed(3))[:B].to(dev).contiguous()
    a = _run_attn(ops, dev, "wg", D, B, L, Hq, Hkv, mask, window, seed=5)
    b = _run_attn(ops, dev, "mma", D, B, L, Hq, Hkv, mask, window, seed=5)
    assert rel(a[1].view.float(), b[1].view.float()) < 1e-2
    fin = torch.isfinite(b[2])
    assert torch.equal(fin, torch.isfinite(a[2])) and (a[2][fin] - b[2][fin]).abs().max() < 1e-4
    for i in (3, 4, 5):
        assert rel(a[i].view.float(), b[i].view.float()) < 2e-2


def test_window_argument_checks(ops, dev):
    from dalm_b200 import _lib
    B, L, H, D = 1, 64, 2, 64
    x = torch.zeros(B * L, H * D, dtype=bf16, device=dev)
    with pytest.raises(_lib.DalmB200Error, match="window"):
        ops.attention_tc_fwd(x, x, x, None, B, L, H, H, D, False, window=8)       # a window needs causal
    with pytest.raises(_lib.DalmB200Error, match="window"):
        ops.attention_fwd(x, x, x, None, B, L, H, H, D, True, window=-1)
    with pytest.raises(_lib.DalmB200Error, match="dropout"):
        ops.attention_tc_fwd(x, x, x, None, B, L, H, H, D, True, window=8, drop=ops.Drop(0.1, 1, 1, None))


# ----------------------------------------------------------------------------------------------------------------
# 2. decode kernel
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,Hq,Hkv,T,cur,window", [(128, 4, 2, 300, 299, 37), (64, 4, 1, 130, 128, 64), (32, 8, 4, 80, 50, 1),
                                                    (128, 8, 8, 1024, 1000, 129), (64, 2, 2, 64, 63, 17)])
def test_attention_decode_window(cuda_dev, D, Hq, Hkv, T, cur, window):
    """one query against the cache with a window shorter than the prefix, against fp64, in host-column and device-column
    modes; while cur < window the result is the bits of window = 0"""
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(T + cur + window)
    B = 3
    Nq, Nkv = Hq * D, Hkv * D
    qkv = (torch.randn(B, Nq + 2 * Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    ck = (torch.randn(B, T, Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    cv = (torch.randn(B, T, Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    mask = (torch.rand(B, T, generator=g) > 0.3).to(i64).to(cuda_dev)
    mask[0, max(0, cur - window):cur] = 0                      # row 0: the window holds nothing but the token itself
    mask[:, cur:] = 0
    ck0, cv0 = ck.clone(), cv.clone()
    out = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck, cv, mask, cur, Hq, Hkv, D, window=window)
    q = qkv[:, :Nq].double().view(B, Hq, D)
    K = ck[:, :cur + 1].double().view(B, cur + 1, Hkv, D).repeat_interleave(Hq // Hkv, dim=2)
    V = cv[:, :cur + 1].double().view(B, cur + 1, Hkv, D).repeat_interleave(Hq // Hkv, dim=2)
    s = torch.einsum("bhd,bthd->bht", q, K) / math.sqrt(D)
    vis = mask[:, :cur + 1].bool().clone()
    vis[:, cur] = True
    vis[:, :max(0, cur - window + 1)] = False
    s = s.masked_fill(~vis[:, None, :], float("-inf"))
    ref = torch.einsum("bht,bthd->bhd", torch.softmax(s, -1), V).reshape(B, Nq)
    assert rel(out.double(), ref) < 5e-3 and (out.double() - ref).abs().max().item() < 2e-2
    assert torch.equal(out[0].view(Hq, D), qkv[0, Nq + Nkv:].view(Hkv, D).repeat_interleave(Hq // Hkv, 0))
    full = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck0.clone(), cv0.clone(), mask, cur, Hq, Hkv, D)
    assert rel(full.double(), ref) > 1e-2                      # the window matters at this column
    ck2, cv2 = ck0.clone(), cv0.clone()
    dcol = torch.full((B,), cur, dtype=torch.int32, device=cuda_dev)
    out2 = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck2, cv2, mask, dcol, Hq, Hkv, D, window=window)
    assert torch.equal(out2, out) and torch.equal(ck2, ck) and torch.equal(cv2, cv)
    # columns the window still covers entirely: the bits of window = 0, in both modes
    c = min(cur, window - 1)
    for col in (c, torch.full((B,), c, dtype=torch.int32, device=cuda_dev)):
        a = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck0.clone(), cv0.clone(), mask, col, Hq, Hkv, D, window=window)
        b = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck0.clone(), cv0.clone(), mask, col, Hq, Hkv, D)
        assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------------------
# 3. decoders against transformers
# ----------------------------------------------------------------------------------------------------------------
def _hf(cfg, sd, headless=False):
    """transformers' MistralForCausalLM (or MistralModel), eager attention"""
    from oracle import models as om
    m = om.build_causal_lm(cfg, sd, headless=headless, attn_implementation="eager")
    assert m.config.sliding_window == cfg.get("sliding_window")
    return m


def _mistral(name, V, seed, headless=False):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.mistral_config(name, vocab_size=V)
    sd = params.random_state_dict("mistral", cfg, seed=seed)
    sd = {k: (v * QK_SCALE if k.endswith(("q_proj.weight", "k_proj.weight")) else v) for k, v in sd.items()}
    sd = r16_2d(sd)
    if headless:
        sd = synthetic.headless_state_dict(sd)
    return cfg, sd


def _no_window(dec):
    """turn `dec` into the control: the same weights with full causal attention"""
    dec.windows = [0] * dec.nl


@pytest.mark.parametrize("name,B,L,pad", [("mistral-tiny", 3, 110, "right"), ("mistral-tiny", 2, 140, "left"),
                                           ("mistral-hd64", 3, 80, "left"), ("mistral-hd64", 2, 111, "right")])
def test_mistral_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits and the marginalised loss vs HF MistralForCausalLM at 2-3x the window, and the LoRA gradients with right
    padding; then the control: the same decoder without its window fails the logits tolerance. With left padding these tiny
    models' LoRA gradients differ from HF's by 6-12 % with and without the window alike (measured on an H100), so that
    comparison says nothing about the window and is made on right-padded batches only."""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _mistral(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    w = cfg["sliding_window"]
    assert dec.windows == [w] * dec.nl and 2 * w <= L <= 3 * w + 3
    assert dec.fuse_rope == (name == "mistral-tiny") and dec.nkv < dec.nh
    ref = _hf(cfg, sd)
    draw_lora_B(dec, torch.Generator().manual_seed(9))
    attach_lora(ref, dec)
    ids, mask, ref_logits = check_decoder(dec, ref, torch.Generator().manual_seed(9), V, B, L, pad, lora_tol=None)
    valid = mask.bool()
    if pad == "right":
        worst = lora_grad_error(dec, hf_grads(ref))
        assert worst < 5e-2, worst
    _no_window(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert rel(control.float().cpu()[valid], ref_logits[valid]) > 10 * 1.5e-2


@pytest.mark.parametrize("name,pad", [("mistral-tiny", "left"), ("mistral-hd64", "right")])
def test_fused_rag_step_mistral_lora(cuda_dev, name, pad):
    """bge + Mistral generator, LoRA on both, generator length 100 (past the window): the fused training step against the
    reference loop body"""
    cfg, sd = _mistral(name, 504, seed=12)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, attn_implementation="eager")
    assert ref.config.sliding_window == cfg.get("sliding_window")
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, rag_batch(5, 12, 24, 100, 600, 504, seed=21, pad=pad))
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["mistral-tiny", "mistral-hd64"])
def test_full_finetune_mistral_gradients(cuda_dev, name):
    """full fine-tuning with a window: every parameter's gradient against autograd through HF (generator rows right-padded,
    see test_mistral_decoder_fwd_bwd_lora)"""
    cfg, sd = _mistral(name, 504, seed=14)
    sd = r16(sd)                                                          # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, lora_r=False, lora_g=False, attn_implementation="eager")
    assert ref.config.sliding_window == cfg.get("sliding_window")
    batch = rag_batch(5, 12, 24, 100, 600, 504, seed=21)
    gm = batch["generator_input_attention_mask"]
    gm[0, :5] = 1
    gm[0, -5:] = 0
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, batch)
    checked = compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 7 * cfg["num_hidden_layers"] + 2
    assert set(dec.hf_state_dict()) == set(sd)


def test_autoregressive_headless_mistral_retriever(cuda_dev):
    """`is_autoregressive=True` with an e5-mistral-shaped headless checkpoint (MistralModel keys, no lm_head): last hidden
    state, eos pooling, LoRA on q_proj / v_proj, passages of 2x the window, against transformers' AutoModel class"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd = _mistral("mistral-tiny", V, seed=31, headless=True)
    assert not any(k.startswith(("model.", "lm_head")) for k in sd)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    assert enc.headless
    ref = _hf(cfg, sd, headless=True)
    draw_lora_B(enc, torch.Generator().manual_seed(32))
    attach_lora(ref, enc, strip="model.")
    check_autoregressive_retriever(enc, ref, torch.Generator().manual_seed(32), V, 24, 100, strip="model.")


@pytest.mark.parametrize("name,B,lora", [("mistral-tiny", 4, False), ("mistral-hd64", 4, True)])
def test_mistral_generate_greedy(cuda_dev, monkeypatch, name, B, lora):
    """greedy decoding to position 139 (3-4x the window): per-step logits and choices vs HF teacher-forced on our tokens, graph
    replay == eager, and the tokens equal HF `generate`'s wherever HF's own choice is not a near tie"""
    from dalm_b200.engine.llama import LlamaDecoder
    V, L0, T = 504, 12, 140
    cfg, sd = _mistral(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = _hf(cfg, sd)
    if lora:
        draw_lora_B(dec, torch.Generator().manual_seed(9))
        attach_lora(ref, dec)
    ids, mask = prompt(B, L0, V, seed=1, low=4)
    out, _ = check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert out.shape == (B, T)
    _, agree = hf_generate_agreement(ref, ids, mask, out, T)
    assert max(agree) == T and L0 + 2 * cfg["sliding_window"] < T


def test_qwen2_sliding_window_layers(cuda_dev):
    """Qwen2 with use_sliding_window and max_window_layers = 1: layer 0 full, layer 1 windowed, against Qwen2ForCausalLM"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from transformers import Qwen2Config, Qwen2ForCausalLM
    V = 504
    cfg = dict(synthetic.qwen2_config("qwen2-tiny", vocab_size=V), use_sliding_window=True, sliding_window=24, max_window_layers=1)
    sd = params.random_state_dict("qwen2", cfg, seed=4)
    sd = {k: (v * QK_SCALE if k.endswith(("q_proj.weight", "k_proj.weight")) else v) for k, v in sd.items()}
    sd = r16_2d(sd)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    assert dec.windows == [0, 24]
    conf = Qwen2Config(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    ref = Qwen2ForCausalLM._from_config(conf, attn_implementation="eager")
    assert ref.config.layer_types == ["full_attention", "sliding_attention"]
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not unexpected and set(missing) <= {"lm_head.weight"}, (missing, unexpected)      # tied head
    ref = ref.float().eval()
    B, L = 3, 70
    ids = torch.randint(3, V, (B, L), generator=torch.Generator().manual_seed(4))
    mask = pad_mask(B, L, "left")
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    with torch.no_grad():
        want = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert rel(logits.float().cpu()[valid], want[valid]) < 1.5e-2
    _no_window(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert rel(control.float().cpu()[valid], want[valid]) > 1.5e-2


# ----------------------------------------------------------------------------------------------------------------
# 4. trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_mistral_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Mistral directory (window 37, generator length 80)
    writes PEFT adapters; eval_rag loads them and generates"""
    from dalm_b200 import synthetic
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / "mistral-hd64"), "mistral", "mistral-hd64", vocab_size=1200)
    out = train_rag_lora(csv, rdir, gdir, tmp_path, generator_max_len=80)
    eval_rag_generator(csv, rdir, gdir, out, capsys)
