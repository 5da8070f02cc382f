"""GPU: OLMo 2 / OLMo 3 / OLMoE. The full-width q/k RMSNorm + RoPE kernels, their deterministic weight gradient and the
post-sublayer norm kernels against fp64 (poisoned padding, guarded outputs); then the models against transformers'
Olmo2ForCausalLM / Olmo3ForCausalLM / OlmoeForCausalLM: logits, loss and gradients, the fused RAG step, the CUDA-graph step,
`generate`, the autoregressive retriever, and the CLI trainer + eval-rag on a synthetic directory."""
import pytest
import torch

from exact_helpers import Guarded, _expect_close, _expect_equal, _poisoned, _ulp_bf16, _ulp_f32
from model_helpers import (attach_lora, check_against_oracle, check_autoregressive_retriever, check_decoder, check_rag_lora_grads,
                           compare_full_grads, draw_lora_B, eval_rag_generator, pad_mask, prompt, r16_2d, rag_batch, rag_models,
                           rag_step_vs_oracle, toy_rag_inputs, train_rag_lora)

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
EPS = 1e-6


# ----------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------
def _tables(dev, T, hd):
    """poisoned fp32 cos / sin [T, hd/2] (NaN rows after T)"""
    inv = 1.0 / (5e5 ** (torch.arange(0, hd, 2, dtype=f32) / hd))
    fr = torch.outer(torch.arange(T, dtype=f32), inv)
    out = []
    for t in (fr.cos() * 1.13, fr.sin() * 1.13):                  # a YaRN-like attention factor on both tables
        buf = torch.full((T + 128, hd // 2), float("nan"), device=dev)
        buf[:T] = t.to(dev)
        out.append(buf[:T])
    return out


def _rot64(n, c, s, hd):
    """rotate_half RoPE of [M, heads, hd] (fp64) with per-row cos / sin [M, 1, hd/2]"""
    a, b = n[..., :hd // 2], n[..., hd // 2:]
    return torch.cat([a * c - b * s, b * c + a * s], -1), torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], -1)


WIDTHS = [(16, 16, 128), (32, 8, 128), (40, 8, 128), (40, 40, 128), (32, 8, 64)]      # (q heads, k heads, head_dim)


def _fullnorm_case(dev, nq, nk, hd, M, seed):
    g = torch.Generator().manual_seed(seed)
    Nq, Nk = nq * hd, nk * hd
    W = Nq + 2 * Nk
    x = (torch.randn(M, W, generator=g) * torch.rand(M, 1, generator=g) * 3).to(bf16).to(dev)
    wq = (1 + torch.randn(Nq, generator=g) * 0.5).to(dev)
    wk = (1 + torch.randn(Nk, generator=g) * 0.5).to(dev)
    return x, _poisoned(wq), _poisoned(wk)


@pytest.mark.parametrize("nq,nk,hd", WIDTHS)
@pytest.mark.parametrize("mode", ["rows", "pos"])
@pytest.mark.parametrize("round_first", [False, True])
def test_qk_fullnorm_rope_vs_fp64(cuda_dev, nq, nk, hd, mode, round_first):
    """rotated q|k against fp64 (one bf16 step of the rounded norm output allowed, per transformers' rounding point), v and
    the padding untouched, pre = the input bits, rstd within fp32 rounding; positions row % L or explicit, out of range
    clamped"""
    from dalm_b200 import ops
    M, L, T = 301, 43, 64
    x, wq, wk = _fullnorm_case(cuda_dev, nq, nk, hd, M, seed=nq + nk + hd)
    Nq, Nk = nq * hd, nk * hd
    cos_t, sin_t = _tables(cuda_dev, T, hd)
    buf = _poisoned(x)
    pos = None
    if mode == "pos":
        p = torch.randint(0, T, (M,), generator=torch.Generator().manual_seed(3))
        p[:3] = torch.tensor([-3, T, T + 9])
        pbuf = torch.full((M + 256,), 1 << 40, dtype=torch.int64, device=cuda_dev)     # far out of range after the view
        pbuf[:M] = p.to(cuda_dev)
        pos = pbuf[:M]
        eff = p.clamp(0, T - 1)
    else:
        eff = torch.arange(M) % L
    pre = Guarded(M, Nq + Nk, bf16, cuda_dev)
    rstd = Guarded(M, 2, f32, cuda_dev)
    ops.qk_fullnorm_rope_(buf, nq, nk, hd, wq, wk, EPS, cos_t, sin_t, L=L if pos is None else 0, pos=pos, pre=pre.view,
                          rstd=rstd.view, round_first=round_first)
    pre.check("pre"); rstd.check("rstd")
    _expect_equal(pre.view, x[:, :Nq + Nk], "pre")
    _expect_equal(buf[:, Nq + Nk:], x[:, Nq + Nk:], "v columns")
    assert torch.isnan(buf.as_strided((M, 64), (buf.stride(0), 1), buf.storage_offset() + buf.shape[1])).all()
    x64 = x.double().cpu()
    out, terms, ulps = [], [], []
    for c0, w, wt, j in ((0, Nq, wq, 0), (Nq, Nk, wk, 1)):
        h = x64[:, c0:c0 + w]
        r = 1.0 / torch.sqrt((h * h).mean(-1, keepdim=True) + EPS)
        _expect_close(rstd.view[:, j:j + 1].cpu(), r, r * 2e-6, f"rstd[{j}]")
        xh = h * r
        if round_first:
            xh = xh.to(bf16).double()
        n = (wt.double().cpu() * xh).to(bf16).double()
        c, s = cos_t.double().cpu()[eff][:, None], sin_t.double().cpu()[eff][:, None]
        rot, t = _rot64(n.view(M, -1, hd), c, s, hd)
        u = _ulp_bf16(n).view(M, -1, hd)
        ua, ub = u[..., :hd // 2], u[..., hd // 2:]
        flip = torch.cat([ua * c.abs() + ub * s.abs(), ub * c.abs() + ua * s.abs()], -1) * (2 if round_first else 1)
        out.append(rot.reshape(M, w)); terms.append(t.reshape(M, w)); ulps.append(flip.reshape(M, w))
    ref, terms, flip = torch.cat(out, 1), torch.cat(terms, 1), torch.cat(ulps, 1)
    _expect_close(buf[:, :Nq + Nk].cpu(), ref, flip + _ulp_bf16(ref) + terms * 2.0 ** -21, "rotated q|k")


def _fullnorm_bwd_ref(x, dy, wq, wk, cos_t, sin_t, Nq, Nk, hd, L):
    """fp64 autograd of rope(w * x rstd) over the q and the k widths: (dx, dwq, dwk, bound). bound: the magnitudes dx's fp32
    arithmetic rounds, rstd (|w g| + |x_hat| mean|w g x_hat|); the second term bounds the fp32 row dot, whose own sum can
    cancel to far below its terms"""
    M = x.shape[0]
    c, s = cos_t.double().cpu()[torch.arange(M) % L][:, None], sin_t.double().cpu()[torch.arange(M) % L][:, None]
    dxs, dws, bounds = [], [], []
    for c0, w, wt in ((0, Nq, wq), (Nq, Nk, wk)):
        h = x[:, c0:c0 + w].double().cpu().requires_grad_(True)
        ww = wt.double().cpu().requires_grad_(True)
        r = 1.0 / torch.sqrt((h * h).mean(-1, keepdim=True) + EPS)
        y, _ = _rot64((ww * h * r).view(M, -1, hd), c, s, hd)
        y.reshape(M, w).backward(dy[:, c0:c0 + w].double().cpu())
        dxs.append(h.grad); dws.append(ww.grad)
        with torch.no_grad():
            g = dy[:, c0:c0 + w].double().cpu().view(M, -1, hd)
            a, b = g[..., :hd // 2], g[..., hd // 2:]
            gu = torch.cat([a * c + b * s, b * c - a * s], -1).reshape(M, w)     # the un-rotated gradient
            xh = h.detach() * r
            m = (ww.detach() * gu * xh).abs().mean(-1, keepdim=True)
            bounds.append((r * ((ww.detach() * gu).abs() + xh.abs() * m)))
            dws[-1] = (dws[-1], (gu * xh).abs().sum(0))
    return torch.cat(dxs, 1), dws, torch.cat(bounds, 1)


@pytest.mark.parametrize("nq,nk,hd", WIDTHS)
def test_qk_fullnorm_rope_bwd_vs_fp64(cuda_dev, nq, nk, hd):
    """d(pre-norm q|k) and the norm weights' gradients against fp64 autograd; v gradients and padding untouched; a second run
    gives the same bits (no atomics)"""
    from dalm_b200 import ops
    M, L = 300, 50
    x, wq, wk = _fullnorm_case(cuda_dev, nq, nk, hd, M, seed=7 + hd)
    Nq, Nk = nq * hd, nk * hd
    cos_t, sin_t = _tables(cuda_dev, L, hd)
    pre, rstd = torch.empty(M, Nq + Nk, dtype=bf16, device=cuda_dev), torch.empty(M, 2, device=cuda_dev)
    ops.qk_fullnorm_rope_(x.clone(), nq, nk, hd, wq, wk, EPS, cos_t, sin_t, L=L, pre=pre, rstd=rstd)
    dy = torch.randn(M, Nq + 2 * Nk, generator=torch.Generator().manual_seed(5)).to(bf16).to(cuda_dev)
    runs = []
    for _ in range(2):
        d = _poisoned(dy)
        gq, gk = Guarded(1, Nq, f32, cuda_dev, init=torch.full((1, Nq), 0.25)), Guarded(1, Nk, f32, cuda_dev, init=torch.full((1, Nk), -0.5))
        ops.qk_fullnorm_rope_bwd_(d, nq, nk, hd, wq, wk, cos_t, sin_t, L, _poisoned(pre), _poisoned(rstd),
                                  dw_q=gq.view[0], dw_k=gk.view[0])
        gq.check("dw_q"); gk.check("dw_k")
        runs.append((d.clone(), gq.view.clone(), gk.view.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    d, gq, gk = runs[0]
    _expect_equal(d[:, Nq + Nk:], dy[:, Nq + Nk:], "v gradient")
    dx, ((dwq, bq), (dwk, bk)), bound = _fullnorm_bwd_ref(x, dy, wq, wk, cos_t, sin_t, Nq, Nk, hd, L)
    _expect_close(d[:, :Nq + Nk].cpu(), dx, _ulp_bf16(dx) + bound * 2.0 ** -17, "d(q|k)")
    _expect_close(gq.cpu(), (dwq + 0.25)[None], bq[None] * 2.0 ** -18 + 1e-6, "dw_q")
    _expect_close(gk.cpu(), (dwk - 0.5)[None], bk[None] * 2.0 ** -18 + 1e-6, "dw_k")


@pytest.mark.parametrize("H", [256, 2048, 4096, 5120, 8192])
def test_postnorm_fwd_bwd_vs_fp64(cuda_dev, H):
    """x_out = resid + bf16(w y rstd(y)) and bf16(x_out); backward d = dres + dh (exact in fp32) and dy against fp64; the
    weight gradient (norm_wgrad, fp32 dy) against fp64 and bit-identical on a second run"""
    from dalm_b200 import ops
    M = 333
    g = torch.Generator().manual_seed(H)
    y = (torch.randn(M, H, generator=g) * torch.rand(M, 1, generator=g) * 4).to(bf16).to(cuda_dev)
    w = (1 + torch.randn(H, generator=g) * 0.5).to(cuda_dev)
    resid = (torch.randn(M, H, generator=g) * 2).to(cuda_dev)
    out16 = Guarded(M, H, bf16, cuda_dev)
    out, rstd = ops.postnorm_fwd(_poisoned(y), _poisoned(w), resid, EPS, out16=out16.view)
    out16.check("out16")
    y64 = y.double().cpu()
    r = 1.0 / torch.sqrt((y64 * y64).mean(-1, keepdim=True) + EPS)
    _expect_close(rstd.cpu()[:, None], r, r * 2e-6, "rstd")
    n = w.double().cpu() * y64 * r
    ref = resid.double().cpu() + n.to(bf16).double()
    _expect_close(out.cpu(), ref, _ulp_bf16(n) + 2 * _ulp_f32(ref), "x_out")
    _expect_equal(out16.view, out.to(bf16), "bf16(x_out)")
    dres = torch.randn(M, H, generator=g).to(cuda_dev)
    dh = torch.randn(M, H, generator=g).to(bf16).to(cuda_dev)
    d, dy = ops.postnorm_bwd(_poisoned(y), _poisoned(w), rstd, dres, dh=_poisoned(dh))
    _expect_equal(d, (dres.double() + dh.double()).float(), "residual gradient")
    yv = y64.clone().requires_grad_(True)
    rr = 1.0 / torch.sqrt((yv * yv).mean(-1, keepdim=True) + EPS)
    (w.double().cpu() * yv * rr).backward(d.double().cpu())
    wd, yh = w.double().cpu() * d.double().cpu(), y64 * r
    m = (wd * yh).abs().mean(-1, keepdim=True)                     # bounds the fp32 row dot (see _fullnorm_bwd_ref)
    _expect_close(dy.cpu(), yv.grad, _ulp_bf16(yv.grad) + r * (wd.abs() + yh.abs() * m) * 2.0 ** -17, "dy")
    dws = []
    for _ in range(2):
        dw = torch.zeros(H, device=cuda_dev)
        ops.norm_wgrad_(d, _poisoned(y), rstd, dw)
        dws.append(dw)
    assert torch.equal(dws[0], dws[1])
    want = (d.double().cpu() * yh).sum(0)
    _expect_close(dws[0].cpu()[None], want[None], (d.double().cpu() * yh).abs().sum(0)[None] * 2.0 ** -18 + 1e-6, "dw")


# ----------------------------------------------------------------------------------------------------------------
# models against transformers
# ----------------------------------------------------------------------------------------------------------------
KIND = {"olmo2-tiny": "olmo2", "olmo2-hd128-gqa": "olmo2", "olmo3-tiny": "olmo3", "olmoe-tiny": "olmoe"}
ROUTER_STD, ROUTE_MARGIN = 0.2, 0.1


@pytest.fixture
def olmo_oracle(monkeypatch):
    """oracle.models.build_causal_lm for the OLMo kinds (transformers' Olmo2 / Olmo3 / OlmoeForCausalLM)"""
    from oracle import models as om
    for k, fam in (("olmo2", "Olmo2"), ("olmo3", "Olmo3"), ("olmoe", "Olmoe")):
        monkeypatch.setitem(om._CAUSAL_LM, k, fam)
    return om


def _olmo(name, V, seed):
    """(cfg, hub-layout state dict, the oracle's layout: OLMoE experts fused) of a bf16-rounded random model"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.olmo_config(name, vocab_size=V)
    sd = r16_2d(params.random_state_dict(KIND[name], cfg, seed=seed, qk_norm_std=0.5, router_std=ROUTER_STD))
    sd = {k: (v.to(bf16).float() if v.dim() >= 2 else v) for k, v in sd.items()}
    if KIND[name] != "olmoe":
        return cfg, sd, sd
    fused = {k: v for k, v in sd.items() if ".mlp.experts." not in k}
    for l in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{l}.mlp.experts."
        fused[p + "gate_up_proj"] = torch.stack([torch.cat([sd[p + f"{e}.gate_proj.weight"], sd[p + f"{e}.up_proj.weight"]])
                                                 for e in range(cfg["num_experts"])])
        fused[p + "down_proj"] = torch.stack([sd[p + f"{e}.down_proj.weight"] for e in range(cfg["num_experts"])])
    return cfg, sd, fused


def _pin_routing(monkeypatch, dec, ref, cfg, ids, mask):
    """OLMoE: the engine's experts are the oracle's top-k wherever the k-th / (k+1)-th router-logit gap exceeds ROUTE_MARGIN
    (at least 80% of the valid tokens); then the oracle's routers take the engine's experts, leaving the comparison to the
    rest of the layer"""
    import torch.nn.functional as F
    from dalm_b200.engine import moe
    if cfg["model_type"] != "olmoe":
        return
    got, real = [], moe.forward

    def recording(*a, **kw):
        out, s = real(*a, **kw)
        got.append(s.ids.long().cpu())
        return out, s
    monkeypatch.setattr(moe, "forward", recording)
    dec.forward_final(ids.to(dec.dev), mask.to(dec.dev), save=False)
    monkeypatch.setattr(moe, "forward", real)
    gates = [layer.mlp.gate for layer in ref.model.layers]
    k, caught = cfg["num_experts_per_tok"], []
    hooks = [gt.register_forward_hook(lambda m, i, o: caught.append(i[0].detach().double().reshape(-1, m.hidden_dim)
                                                                    @ m.weight.double().t())) for gt in gates]
    with torch.no_grad():
        ref(input_ids=ids, attention_mask=mask)
    for h in hooks:
        h.remove()
    valid = mask.bool().view(-1)
    for l, (lg, mine) in enumerate(zip(caught, got)):
        top = lg.topk(k + 1, -1)
        clear = valid & (top.values[:, k - 1] - top.values[:, k] > ROUTE_MARGIN)
        assert clear.sum() >= 0.8 * valid.sum(), f"layer {l}: only {int(clear.sum())} of {int(valid.sum())} tokens clear"
        assert not (clear & (mine.sort(-1).values != top.indices[:, :k].sort(-1).values).any(-1)).any(), f"layer {l}"
    for gate, sel in zip(gates, got):
        def fwd(h, gate=gate, sel=sel):
            h = h.reshape(-1, gate.hidden_dim)
            probs = F.softmax(F.linear(h, gate.weight), dtype=torch.float, dim=-1)
            w = probs.gather(1, sel)
            if gate.norm_topk_prob:
                w = w / w.sum(-1, keepdim=True)
            return probs, w.to(probs.dtype), sel
        monkeypatch.setattr(gate, "forward", fwd)


@pytest.mark.parametrize("name,B,L,pad", [("olmo2-tiny", 3, 40, "right"), ("olmo2-hd128-gqa", 2, 72, "left"),
                                          ("olmo3-tiny", 3, 56, "left"), ("olmo3-tiny", 2, 48, "right"),
                                          ("olmoe-tiny", 3, 40, "right"), ("olmoe-tiny", 2, 72, "left")])
def test_olmo_decoder_fwd_bwd_lora(cuda_dev, monkeypatch, olmo_oracle, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients (q_proj / v_proj) against transformers; OLMo 3's sequences cross
    its 16-token window"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd, osd = _olmo(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    ref = olmo_oracle.build_causal_lm(cfg, osd)
    draw_lora_B(dec, torch.Generator().manual_seed(9))
    attach_lora(ref, dec)
    g = torch.Generator().manual_seed(9)
    ids, mask = torch.randint(3, V, (B, L), generator=g), pad_mask(B, L, pad)         # what check_decoder draws from g first
    _pin_routing(monkeypatch, dec, ref, cfg, ids, mask)
    check_decoder(dec, ref, torch.Generator().manual_seed(9), V, B, L, pad)


@pytest.mark.parametrize("name", ["olmo2-tiny", "olmo3-tiny", "olmo2-hd128-gqa"])
def test_olmo_full_finetune_gradients(cuda_dev, olmo_oracle, name):
    """full fine-tuning: every parameter's gradient (q_norm / k_norm, both post-sublayer norms included) against autograd
    through transformers, and the same bits on a second backward; hf_state_dict writes the checkpoint layout back"""
    cfg, sd, _ = _olmo(name, 504, seed=14)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, sd, lora_r=False, lora_g=False)
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=21)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, batch)
    checked = compare_full_grads(dec, want["grads"], "generator.")
    assert checked >= 9 * cfg["num_hidden_layers"] + 2
    hf = dec.hf_state_dict()
    assert set(hf) == set(sd) and all(torch.equal(hf[k], sd[k].float()) for k in sd)


@pytest.mark.parametrize("name,pad", [("olmo2-hd128-gqa", "left"), ("olmo3-tiny", "right"), ("olmoe-tiny", "left")])
def test_fused_rag_step_olmo_lora(cuda_dev, monkeypatch, olmo_oracle, name, pad):
    """bge-tiny + an OLMo generator, LoRA on both: the fused training step against the reference loop body"""
    cfg, _, osd = _olmo(name, 504, seed=12)
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, osd)              # the engine loads OLMoE's fused layout here
    _pin_routing(monkeypatch, dec, ref, cfg, batch["generator_input_input_ids"], batch["generator_input_attention_mask"])
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, batch)
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.parametrize("name", ["olmo2-tiny", "olmoe-tiny"])
def test_graphed_step_bit_identical(cuda_dev, olmo_oracle, name):
    """the step captured as one CUDA graph gives the eager step's loss and LoRA gradients bit for bit"""
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_rag_step
    cfg, _, osd = _olmo(name, 504, seed=12)
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=22)
    model, enc, dec, _, _ = rag_models(cuda_dev, cfg, osd)
    zero = lambda: (enc.zero_grad_buffers(), dec.zero_grad_buffers())
    zero()
    eager = fused_rag_step(model, batch, 100.0)
    want = [eager["losses"].clone(), enc.lora.grad.clone(), dec.lora.grad.clone()]
    graphed = GraphedStep(fused_rag_step, model, batch, 100.0, zero_grads=zero)
    assert isinstance(graphed.graph, torch.cuda.CUDAGraph)
    for _ in range(2):
        zero()
        out = graphed(batch)
        torch.cuda.synchronize()
        for a, b in zip([out["losses"], enc.lora.grad, dec.lora.grad], want):
            assert torch.equal(a, b)


@pytest.mark.parametrize("name,B,L0,T", [("olmo2-tiny", 4, 12, 30), ("olmo2-hd128-gqa", 20, 12, 30), ("olmo3-tiny", 4, 30, 60),
                                          ("olmoe-tiny", 4, 12, 30)])
def test_olmo_generate(cuda_dev, monkeypatch, olmo_oracle, name, B, L0, T):
    """greedy decoding: per-step logits and choices vs the oracle teacher-forced on our tokens, and the decode step replayed
    as a CUDA graph gives the eager tokens; OLMo 3's prompt and generation run past its 16-token window"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd, osd = _olmo(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    ref = olmo_oracle.build_causal_lm(cfg, osd)
    ids, mask = prompt(B, L0, V, seed=1)
    out, _ = check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert out.shape == (B, T)


@pytest.mark.parametrize("name", ["olmo3-tiny", "olmoe-tiny"])
def test_olmo_generate_sampling_graph(cuda_dev, monkeypatch, name):
    """sampling (temperature / top-k / top-p): reproducible under torch.manual_seed, graph replay == eager launches"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import decoding
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd, _ = _olmo(name, V, seed=5)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    dec.generation_config = dict(synthetic.QWEN3_GENERATION["instruct"])
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(3, V, (8, 12), generator=g)
    mask = torch.ones(8, 12, dtype=torch.int64)
    mask[1, :3] = 0

    def gen(seed, graph):
        monkeypatch.setenv("DALM_B200_DECODE_GRAPH", graph)
        torch.manual_seed(seed)
        return dec.generate(input_ids=ids.to(cuda_dev), attention_mask=mask.to(cuda_dev), max_length=34, eos_token_id=[]).cpu()

    eager = gen(7, "0")
    assert eager.shape == (8, 34) and torch.equal(eager[:, :12], ids)
    assert torch.equal(gen(7, "0"), eager)
    replayed = gen(7, "1")
    assert decoding.LAST_RUN["graph_replays"] > 0 and torch.equal(replayed, eager)


def test_autoregressive_olmo2_retriever(cuda_dev, olmo_oracle):
    """`is_autoregressive=True` with an OLMo 2 model: last hidden state, eos pooling, LoRA on q_proj / v_proj"""
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd, _ = _olmo("olmo2-hd128-gqa", V, seed=31)
    enc = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True, lora_seed=0)
    ref = olmo_oracle.build_causal_lm(cfg, sd)
    draw_lora_B(enc, torch.Generator().manual_seed(32))
    attach_lora(ref, enc)
    check_autoregressive_retriever(enc, ref, torch.Generator().manual_seed(32), V, 12, 20)


@pytest.mark.parametrize("name", ["olmo3-tiny", "olmoe-tiny"])
def test_train_and_eval_rag_with_olmo_directory(cuda_dev, tmp_path, capsys, name):
    """`dalm train-rag-e2e --use-peft both` on a toy CSV with a synthetic OLMo directory writes adapters; eval-rag loads them
    and decodes"""
    from dalm_b200 import synthetic
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / name), KIND[name], name, vocab_size=1200, router_std=ROUTER_STD,
                                     generation_config=synthetic.QWEN3_GENERATION["base"])
    out = train_rag_lora(csv, rdir, gdir, tmp_path)
    torch.manual_seed(0)
    eval_rag_generator(csv, rdir, gdir, out, capsys)
