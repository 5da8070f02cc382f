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
import os

import pytest
import torch

from exact_helpers import Guarded, _expect_close, _poisoned
from test_exact_tiles_gpu import _attn_fns, _attn_ref64, _row_mask, dev, ops  # noqa: F401  (module fixtures)

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64
QK_SCALE = 2.5


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _visible_win(mask, L, window):
    """[B, 1, Lq, Lk] visibility: key-padding mask, causal, and j > i - window when window > 0"""
    i = torch.arange(L, device=mask.device)
    band = i[None, :] <= i[:, None]
    if window > 0:
        band = band & (i[None, :] > i[:, None] - window)
    return mask.bool()[:, None, None, :] & band


def _attn_bwd64(q, k, v, d_out, o, vis, B, L, Hq, Hkv, D, scale):
    """fp64 flash-attention backward: P from fp64 scores, delta = rowsum(dO * O) from the given output,
    dS = P (dP - delta) scale; -> dq [B*L, Hq*D], dk / dv [B*L, Hkv*D] (summed over the q heads of each kv head)"""
    G = Hq // Hkv
    qh = q.view(B, L, Hq, D).transpose(1, 2)
    kh = k.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(G, 1)
    vh = v.view(B, L, Hkv, D).transpose(1, 2).repeat_interleave(G, 1)
    doh = d_out.view(B, L, Hq, D).transpose(1, 2)
    oh = o.view(B, L, Hq, D).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    dp = doh @ vh.transpose(-1, -2)
    delta = (doh * oh).sum(-1, keepdim=True)
    ds = p * (dp - delta) * scale
    dq = ds @ kh
    dk = (ds.transpose(-1, -2) @ qh).view(B, Hkv, G, L, D).sum(2)
    dv = (p.transpose(-1, -2) @ doh).view(B, Hkv, G, L, D).sum(2)
    flat = lambda t, H: t.transpose(1, 2).reshape(B * L, H * D)
    return flat(dq, Hq), flat(dk, Hkv), flat(dv, Hkv)


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
    assert _rel(a[1].view.float(), b[1].view.float()) < 1e-2
    fin = torch.isfinite(b[2])
    assert torch.equal(fin, torch.isfinite(a[2])) and (a[2][fin] - b[2][fin]).abs().max() < 1e-4
    for i in (3, 4, 5):
        assert _rel(a[i].view.float(), b[i].view.float()) < 2e-2


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
    assert _rel(out.double(), ref) < 5e-3 and (out.double() - ref).abs().max().item() < 2e-2
    assert torch.equal(out[0].view(Hq, D), qkv[0, Nq + Nkv:].view(Hkv, D).repeat_interleave(Hq // Hkv, 0))
    full = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck0.clone(), cv0.clone(), mask, cur, Hq, Hkv, D)
    assert _rel(full.double(), ref) > 1e-2                      # the window matters at this column
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
def build_mistral(cfg, sd, headless=False):
    """transformers' MistralForCausalLM (or MistralModel), fp32, eager attention, on the given HF-named weights"""
    from transformers import MistralConfig, MistralForCausalLM, MistralModel
    conf = MistralConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    cls = MistralModel if headless else MistralForCausalLM
    m = cls._from_config(conf, attn_implementation="eager")
    assert m.config.sliding_window == cfg.get("sliding_window")
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return m.float().eval()


def _mistral(name, V, seed, headless=False):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.mistral_config(name, vocab_size=V)
    sd = params.random_state_dict("mistral", cfg, seed=seed)
    sd = {k: (v * QK_SCALE if k.endswith(("q_proj.weight", "k_proj.weight")) else v) for k, v in sd.items()}
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}
    if headless:
        sd = synthetic.headless_state_dict(sd)
    return cfg, sd


def _no_window(dec):
    """turn `dec` into the control: the same weights with full causal attention"""
    dec.windows = [0] * dec.nl


def _mask(B, L, pad):
    mask = torch.ones(B, L, dtype=i64)
    if pad == "right":
        mask[0, L - 5:] = 0
    else:
        mask[0, :5] = 0; mask[1, :2] = 0
    return mask


def _lora_init(dec, ref, seed, strip=""):
    from oracle import models as om
    g = torch.Generator().manual_seed(seed)
    for n, _, _ in dec.lora.specs:
        dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(dec.dev))
    dec.repack_lora()
    om.attach_lora(ref, {n[len(strip):]: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})


@pytest.mark.parametrize("name,B,L,pad", [("mistral-tiny", 3, 110, "right"), ("mistral-tiny", 2, 140, "left"),
                                           ("mistral-hd64", 3, 80, "left"), ("mistral-hd64", 2, 111, "right")])
def test_mistral_decoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    """logits and the marginalised loss vs HF MistralForCausalLM at 2-3x the window, and the LoRA gradients with right
    padding; then the control: the same decoder without its window fails the logits tolerance. With left padding these tiny
    models' LoRA gradients differ from HF's by 6-12 % with and without the window alike (measured on an H100), so that
    comparison says nothing about the window and is made on right-padded batches only."""
    from dalm_b200 import ops
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import losses, models as om
    V = 504
    cfg, sd = _mistral(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    w = cfg["sliding_window"]
    assert dec.windows == [w] * dec.nl and 2 * w <= L <= 3 * w + 3
    assert dec.fuse_rope == (name == "mistral-tiny") and dec.nkv < dec.nh
    ref = build_mistral(cfg, sd)
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
    if pad == "right":
        worst = 0.0
        for n, _, _ in dec.lora.specs:
            mod = om._get_module(ref, n)
            worst = max(worst, _rel(dec.lora.gA[n], mod.lora_A.grad), _rel(dec.lora.gB[n], mod.lora_B.grad))
        assert worst < 5e-2, worst
    _no_window(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert _rel(control.float().cpu()[valid], ref_logits[valid]) > 10 * 1.5e-2


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
    bert, ref = om.build_bert(bcfg, bsd), build_mistral(gcfg, gsd)
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


@pytest.mark.parametrize("name,pad", [("mistral-tiny", "left"), ("mistral-hd64", "right")])
def test_fused_rag_step_mistral_lora(cuda_dev, name, pad):
    """bge + Mistral generator, LoRA on both, generator length 100 (past the window): the fused training step against the
    reference loop body"""
    from test_step_gpu import _batch, _check_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _mistral(name, 504, seed=12)
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=True)
    batch = _batch(5, 12, 24, 100, 600, 504, seed=21, pad=pad)
    want = om.rag_step(bert, ref, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    got = out["losses"].cpu()
    assert abs(got[2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    _check_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["mistral-tiny", "mistral-hd64"])
def test_full_finetune_mistral_gradients(cuda_dev, name):
    """full fine-tuning with a window: every parameter's gradient against autograd through HF (generator rows right-padded,
    see test_mistral_decoder_fwd_bwd_lora)"""
    from test_full_ft_gpu import _batch, _compare_full_grads

    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd = _mistral(name, 504, seed=14)
    sd = {k: v.to(bf16).float() for k, v in sd.items()}                 # fp32 master == bf16 shadow at the start
    model, enc, dec, bert, ref = _rag_models(cuda_dev, cfg, sd, lora=False)
    batch = _batch(5, 12, 24, 100, 600, 504, seed=21)
    gm = batch["generator_input_attention_mask"]
    gm[0, :5] = 1
    gm[0, -5:] = 0
    want = om.rag_step(bert, ref, batch)
    enc.full.zero_grad(); dec.full.zero_grad()
    out = fused_rag_step(model, batch, 100.0)
    assert abs(out["losses"][2].item() - want["loss"].item()) / abs(want["loss"].item()) < 1e-3
    checked = _compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 7 * cfg["num_hidden_layers"] + 2
    assert set(dec.hf_state_dict()) == set(sd)


def test_autoregressive_headless_mistral_retriever(cuda_dev):
    """`is_autoregressive=True` with an e5-mistral-shaped headless checkpoint (MistralModel keys, no lm_head): last hidden
    state, eos pooling, LoRA on q_proj / v_proj, passages of 2x the window, against transformers' AutoModel class"""
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    from oracle import losses, models as om
    V = 504
    cfg, sd = _mistral("mistral-tiny", V, seed=31, headless=True)
    assert not any(k.startswith(("model.", "lm_head")) for k in sd)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    assert enc.headless
    ref = build_mistral(cfg, sd, headless=True)
    _lora_init(enc, ref, 32, strip="model.")
    g = torch.Generator().manual_seed(32)
    model = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, is_autoregressive=True, _model=enc, _load_tokenizer=False)
    B, Lq, Lp = 4, 24, 100
    mk = lambda L: torch.ones(B, L, dtype=i64)
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
        mod = om._get_module(ref, n[len("model."):])
        worst = max(worst, _rel(enc.lora.gA[n], mod.lora_A.grad), _rel(enc.lora.gB[n], mod.lora_B.grad))
    assert worst < 8e-2, worst


@pytest.mark.parametrize("name,B,lora", [("mistral-tiny", 4, False), ("mistral-hd64", 4, True)])
def test_mistral_generate_greedy(cuda_dev, monkeypatch, name, B, lora):
    """greedy decoding to position 139 (3-4x the window): per-step logits and choices vs HF teacher-forced on our tokens, graph
    replay == eager, and the tokens equal HF `generate`'s wherever HF's own choice is not a near tie"""
    from test_generate_gpu import _check_against_oracle

    from dalm_b200.engine.llama import LlamaDecoder
    V, L0, T = 504, 12, 140
    cfg, sd = _mistral(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = build_mistral(cfg, sd)
    if lora:
        _lora_init(dec, ref, 9)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(4, V, (B, L0), generator=g)
    mask = torch.ones(B, L0, dtype=i64)
    mask[1, :3] = 0
    mask[2, 9:] = 0
    out, _ = _check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert out.shape == (B, T)
    ref.generation_config.eos_token_id = None
    with torch.no_grad():
        hf = ref.generate(input_ids=ids, attention_mask=mask, max_length=T, do_sample=False, pad_token_id=0)
        am = torch.ones(B, T, dtype=i64)
        am[:, :L0] = mask
        pos = (am.cumsum(-1) - 1).masked_fill(am == 0, 1)
        want = ref(input_ids=out, attention_mask=am, position_ids=pos).logits.float()
    agree = []
    for r in range(B):
        diff = (out[r] != hf[r]).nonzero()
        if diff.numel():
            c = int(diff[0])
            top2 = want[r, c - 1].topk(2).values
            assert float(top2[0] - top2[1]) < 0.05, (r, c)
        agree.append(int(diff[0]) if diff.numel() else T)
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
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}
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
    mask = _mask(B, L, "left")
    logits, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    with torch.no_grad():
        want = ref(input_ids=ids, attention_mask=mask).logits
    valid = mask.bool()
    assert _rel(logits.float().cpu()[valid], want[valid]) < 1.5e-2
    _no_window(dec)
    control, _ = dec.forward_logits(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert _rel(control.float().cpu()[valid], want[valid]) > 1.5e-2


# ----------------------------------------------------------------------------------------------------------------
# 4. trainer and evaluation end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_eval_rag_with_mistral_directory(cuda_dev, tmp_path, capsys):
    """train_e2e (`dalm train-rag-e2e`) on a toy CSV with a synthetic Mistral directory (window 37, generator length 80)
    writes PEFT adapters; eval_rag loads them and generates"""
    import csv as _csv

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
    gdir = synthetic.write_model_dir(str(tmp_path / "mistral-hd64"), "mistral", "mistral-hd64", vocab_size=1200)
    out = str(tmp_path / "out")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=80,
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
