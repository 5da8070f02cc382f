"""Qwen3-MoE's routed MLP on the GPU: the grouped wgmma GEMM, the routing kernels and the layer they make.

Grouped GEMM: integer operands, so every sum is exact in fp32 and each expert's rows are compared bit for bit with an fp64
per-expert reference (bf16 outputs: its round-to-nearest-even image). Operands carry NaN padding columns and rows; the
padding rows inside each expert's segment are NaN too, so a tile that mixes rows or experts shows. Outputs sit in guard
bands, and the rows of the unused tail tiles must come back untouched. max_ctas forces several tiles per CTA.

Routing kernels: the router against torch.topk and fp64 softmax; the permutation against its definition; gather, combine,
the down-projection and router backwards against fp64 autograd; the whole layer forward + backward against fp64 autograd
on the same routing, and bit-identical from run to run.
"""
import pytest
import torch

from exact_helpers import (Guarded, _expect_close, _expect_equal, _ints, _poisoned, _ulp_bf16, _ulp_f32,  # noqa: F401
                           dev, ops)

bf16, f32, f64, i32 = torch.bfloat16, torch.float32, torch.float64, torch.int32


# ----------------------------------------------------------------------------------------------------------------
# grouped GEMM
# ----------------------------------------------------------------------------------------------------------------
def _segments(counts):
    """padded row offsets of segments with these row counts"""
    off, o = [], 0
    for c in counts:
        off.append(o)
        o += -(-c // 128) * 128
    return off, o


# per-expert row counts: empty experts, segments of 1 row and of 128 n rows, everything on one expert; `extra` unused tail
# tiles past the live ones
COUNT_CASES = [
    ([0, 1, 128, 0, 300, 256, 0, 5], 2),
    ([0, 0, 0, 700, 0, 0], 1),
    ([1, 1, 1, 1, 1, 1, 1, 1, 1, 1], 3),
    ([128, 384, 0, 129, 127], 0),
]


def _grouped_case(ops, dev, counts, extra, layout, swiglu, N, K, max_ctas, seed):
    g = torch.Generator().manual_seed(seed)
    E = len(counts)
    off, live_rows = _segments(counts)
    n_tiles = live_rows // 128 + extra
    rows = 128 * n_tiles
    a_host = torch.full((rows, K), float("nan"))
    for e, c in enumerate(counts):
        a_host[off[e]:off[e] + c] = _ints((c, K), g)
    a = _poisoned(a_host.to(dev, bf16))
    wshape = (E, N, K) if layout == 0 else (E, K, N)
    wbuf = torch.full((E + 1,) + wshape[1:], float("nan"), dtype=bf16, device=dev)   # a NaN expert after the last one
    wbuf[:E] = _ints(wshape, g).to(dev, bf16)
    w = wbuf[:E]
    tiles = torch.full((n_tiles,), -1, dtype=i32)
    for e, c in enumerate(counts):
        tiles[off[e] // 128:(off[e] + -(-c // 128) * 128) // 128] = e
    tile_expert = tiles.to(dev)
    live = torch.tensor([live_rows // 128], dtype=i32, device=dev)
    out = Guarded(rows, N, bf16, dev)
    act = Guarded(rows, N // 2, bf16, dev) if swiglu else None
    ops.gemm_grouped(a, w, tile_expert, live, out=out.view, layout=layout, swiglu=swiglu, act=act.view if swiglu else None,
                     max_ctas=max_ctas)
    what = f"gemm_grouped layout {layout} swiglu {swiglu} counts {counts} +{extra} tiles N {N} K {K} max_ctas {max_ctas}"
    w64 = w.double().cpu()
    got, got_act = out.view.cpu(), act.view.cpu() if swiglu else None
    for e, c in enumerate(counts):
        if c == 0:
            continue
        x = a_host[off[e]:off[e] + c].double()
        acc = x @ (w64[e].t() if layout == 0 else w64[e])
        _expect_equal(got[off[e]:off[e] + c], acc.to(bf16), f"{what} expert {e}", 128, 256)
        if swiglu:
            blk = acc.view(c, N // 256, 2, 128)
            gate, up = blk[:, :, 0].reshape(c, N // 2), blk[:, :, 1].reshape(c, N // 2)
            ref = gate * torch.sigmoid(gate) * up
            _expect_close(got_act[off[e]:off[e] + c], ref, _ulp_bf16(ref) + 2.0 ** -20 * ref.abs() + 2.0 ** -100,
                          f"{what} act expert {e}", 128, 128)
    # the tail tiles past the live count are not computed: their rows keep the sentinel
    for v, nm in ((out, "out"), (act, "act")):
        if v is None:
            continue
        tail = v.view[live_rows:].contiguous().view(torch.int16)
        assert bool((tail == v.bits).all()), f"{what}: {nm} rows past the live tiles were written"
        v.check(f"{what} {nm}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["tn", "nn", "swiglu"])
def test_grouped_gemm_exact(ops, dev, kind):
    """each grouped instance, per expert bit-exact against fp64, over empty / 1-row / 128 n-row / single-expert segments"""
    layout, swiglu = (1, False) if kind == "nn" else (0, kind == "swiglu")
    shapes = {"tn": [(200, 72), (1024, 64), (64, 8)], "nn": [(200, 64), (768, 128), (64, 192)],
              "swiglu": [(256, 72), (512, 128)]}[kind]
    i = 0
    for counts, extra in COUNT_CASES:
        for N, K in shapes:
            for max_ctas in (0, 3):
                _grouped_case(ops, dev, counts, extra, layout, swiglu, N, K, max_ctas, seed=i)
                i += 1


@pytest.mark.gpu
def test_grouped_gemm_refusals(ops, dev):
    a = torch.zeros(256, 72, dtype=bf16, device=dev)
    te, live = torch.zeros(2, dtype=i32, device=dev), torch.ones(1, dtype=i32, device=dev)
    with pytest.raises(ops._lib.DalmB200Error, match="multiple of 64"):
        ops.gemm_grouped(a, torch.zeros(2, 72, 64, dtype=bf16, device=dev), te, live, layout=1)
    with pytest.raises(ops._lib.DalmB200Error, match="multiple of 256"):
        ops.gemm_grouped(a, torch.zeros(2, 128, 72, dtype=bf16, device=dev), te, live, swiglu=True)


# ----------------------------------------------------------------------------------------------------------------
# routing kernels
# ----------------------------------------------------------------------------------------------------------------
def _probs64(logits):
    return torch.softmax(logits.double(), -1)


@pytest.mark.gpu
@pytest.mark.parametrize("E,k", [(8, 2), (60, 4), (128, 8), (256, 16)])
@pytest.mark.parametrize("norm", [False, True])
def test_router(ops, dev, E, k, norm):
    """ids == torch.topk of the same fp32 logits; weights within a few fp32 ulps of fp64"""
    g = torch.Generator().manual_seed(E * 31 + k)
    M = 1000
    logits = (torch.randn(M, E, generator=g) * 3).to(dev)
    ids, w = ops.moe_router(_poisoned(logits), k, norm)
    want = torch.topk(logits, k, dim=-1)
    assert torch.equal(ids.long(), want.indices), "router ids differ from torch.topk"
    p = _probs64(logits).gather(1, ids.long())
    ref = p / p.sum(-1, keepdim=True) if norm else p
    _expect_close(w, ref, 8 * _ulp_f32(ref), f"router weights E {E} k {k} norm {norm}")


def _check_routing(r, ids, E):
    ids = ids.cpu().long().view(-1)
    P = ids.numel()
    counts = torch.bincount(ids, minlength=E)
    assert torch.equal(r.counts.cpu().long(), counts)
    pad = (counts + 127) // 128 * 128
    off = torch.cat([torch.zeros(1, dtype=torch.long), pad.cumsum(0)])
    assert torch.equal(r.seg_off.cpu().long(), off)
    live = int(off[-1]) // 128
    assert int(r.live.item()) == live
    te = torch.full((r.n_tiles,), -1, dtype=torch.long)
    for e in range(E):
        te[int(off[e]) // 128:int(off[e + 1]) // 128] = e
    assert torch.equal(r.tile_expert.cpu().long(), te)
    pr = r.pair_row.cpu().long()
    want = torch.empty(P, dtype=torch.long)
    for e in range(E):
        sel = (ids == e).nonzero().view(-1)                 # pair order: by token, then slot
        want[sel] = off[e] + torch.arange(sel.numel())
    assert torch.equal(pr, want), "pair -> row map"
    rp = r.row_pair.cpu().long()[:live * 128]
    wrp = torch.full((live * 128,), -1, dtype=torch.long)
    wrp[want] = torch.arange(P)
    assert torch.equal(rp, wrp), "row -> pair map"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random", "one_expert", "skewed"])
def test_permute(ops, dev, case):
    g = torch.Generator().manual_seed(7)
    M, k, E = 3000, 8, 128
    if case == "random":
        ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)])
    elif case == "one_expert":
        M, k = 2500, 1
        ids = torch.full((M, 1), 77)
    else:                                                   # most pairs on a few experts, many experts empty
        ids = torch.stack([torch.randperm(12, generator=g)[:k] for _ in range(M)]) * 3
    ids = ids.to(dev, i32).contiguous()
    r = ops.moe_permute(ids, E)
    _check_routing(r, ids, E)


def _routed(ops, dev, M, E, k, norm, seed, H=256):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(M, E, generator=g) * 2).to(dev)
    ids, w = ops.moe_router(logits, k, norm)
    return g, logits, ids, w, ops.moe_permute(ids, E)


@pytest.mark.gpu
def test_gather_combine(ops, dev):
    """gather: rows exact (0 on padding); combine: fp32 sums in slot order against fp64"""
    M, E, k, H = 777, 16, 4, 264
    g, _, ids, w, r = _routed(ops, dev, M, E, k, True, 3)
    x = _poisoned(torch.randn(M, H, generator=g).to(dev, bf16))
    rows = ops.moe_gather(x, r)
    live = int(r.live.item()) * 128
    rp = r.row_pair[:live].long()
    want = torch.where((rp >= 0)[:, None], x[rp.clamp_min(0) // k], torch.zeros((), dtype=bf16, device=dev))
    _expect_equal(rows[:live], want, "moe_gather")
    xf = _poisoned(torch.randn(M, H, generator=g).to(dev))
    rows32 = ops.moe_gather(xf, r)
    _expect_equal(rows32[:live], torch.where((rp >= 0)[:, None], xf[rp.clamp_min(0) // k], torch.zeros((), device=dev)).to(bf16),
                  "moe_gather fp32 source")
    y = torch.randn(r.rows, H, generator=g).to(dev, bf16)
    resid = torch.randn(M, H, generator=g).to(dev)
    yp = y[r.pair_row.long()].double().view(M, k, H)
    ref = resid.double() + (w.double()[..., None] * yp).sum(1)
    terms = resid.double().abs() + (w.double()[..., None] * yp).abs().sum(1)
    out = Guarded(M, H, f32, dev)
    ops.moe_combine(y, r, w, resid=_poisoned(resid), out=out.view)
    _expect_close(out.view, ref, (k + 2) * _ulp_f32(terms), "moe_combine")
    out.check("moe_combine")
    o16 = ops.moe_combine(y, r, None, resid=resid.to(bf16))            # weights of 1, bf16 in place of fp32
    ref1 = resid.to(bf16).double() + yp.sum(1)
    _expect_close(o16, ref1, _ulp_bf16(ref1) + (k + 2) * _ulp_f32(ref1.abs() + yp.abs().sum(1)), "moe_combine w=None bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
def test_down_bwd_and_router_bwd(ops, dev, norm):
    """dw = <da, act> and d_act = w da per pair; dlogits against fp64 autograd of softmax, top-k gather and renormalisation"""
    M, E, k, I = 500, 32, 4, 200
    g, logits, ids, w, r = _routed(ops, dev, M, E, k, norm, 11)
    da = torch.randn(r.rows, I, generator=g).to(dev, bf16)
    act = torch.randn(r.rows, I, generator=g).to(dev, bf16)
    dw, d_act = ops.moe_down_bwd(da, act, r, w)
    pr = r.pair_row.long()
    ref_dw = (da[pr].double() * act[pr].double()).sum(-1).view(M, k)
    tol = (I / 8 + 8) * _ulp_f32((da[pr].double() * act[pr].double()).abs().sum(-1)).view(M, k)
    _expect_close(dw, ref_dw, tol, "moe_down_bwd dw")
    ref_da = (w.view(-1)[:, None] * da[pr].float()).to(bf16)           # one fp32 product, then RNE, as the kernel
    _expect_equal(d_act[pr], ref_da, "moe_down_bwd d_act")
    # router backward
    lg = logits.double().clone().requires_grad_(True)
    p = torch.softmax(lg, -1).gather(1, ids.long())
    wt = p / p.sum(-1, keepdim=True) if norm else p
    (wt * dw.double()).sum().backward()
    ref = lg.grad
    got = ops.moe_router_bwd(logits, ids, w, dw, norm)
    S = torch.softmax(logits.double(), -1).gather(1, ids.long()).sum(-1, keepdim=True)
    scale = dw.double().abs().sum(-1, keepdim=True) / (S if norm else 1.0)
    _expect_close(got, ref, _ulp_bf16(ref) + 2.0 ** -18 * scale, f"moe_router_bwd norm {norm}")


# ----------------------------------------------------------------------------------------------------------------
# the layer
# ----------------------------------------------------------------------------------------------------------------
def _layer(dev, E, k, H, I, seed, norm=True):
    from dalm_b200.engine import moe
    g = torch.Generator().manual_seed(seed)
    gate = torch.randn(E, H, generator=g) * 0.3
    gp, up = torch.randn(E, I, H, generator=g) * H ** -0.5, torch.randn(E, I, H, generator=g) * H ** -0.5
    down = torch.randn(E, H, I, generator=g) * I ** -0.5
    mw = moe.pack_experts(gate, gp, up, down, k, norm, dev)
    host = {n: t.to(bf16).double() for n, t in (("gate", gate), ("gp", gp), ("up", up), ("down", down))}
    return moe, mw, host, g


def _ref_layer(x, resid, host, ids, k, norm):
    """fp64 Qwen3MoeSparseMoeBlock on the given expert choice (autograd-ready in x)"""
    logits = x @ host["gate"].t()
    p = torch.softmax(logits, -1).gather(1, ids)
    w = p / p.sum(-1, keepdim=True) if norm else p
    out = resid.clone()
    for s in range(k):
        e = ids[:, s]
        gt = torch.einsum("mh,mih->mi", x, host["gp"][e])
        u = torch.einsum("mh,mih->mi", x, host["up"][e])
        y = torch.einsum("mi,mhi->mh", torch.nn.functional.silu(gt) * u, host["down"][e])
        out = out + w[:, s:s + 1] * y
    return out, logits


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [True, False])
def test_moe_layer_vs_fp64(ops, dev, norm):
    """forward and dx against fp64 autograd with the engine's expert choice, after checking that choice is not a near-tie"""
    M, E, k, H, I = 600, 16, 4, 256, 256
    moe, mw, host, g = _layer(dev, E, k, H, I, 5, norm)
    x = (torch.randn(M, H, generator=g)).to(dev, bf16)
    resid = torch.randn(M, H, generator=g).to(dev)
    out, saved = moe.forward(x, mw, resid=resid.clone())
    ids = saved.ids.long().cpu()
    x64 = x.double().cpu().requires_grad_(True)
    ref, logits = _ref_layer(x64, resid.double().cpu(), host, ids, k, norm)
    # the choice flips only where the k-th and (k+1)-th logits are closer than the fp32 logits' error (~1e-5 here): tokens
    # closer than 1e-3 are left out of the comparison
    lg = logits.detach().sort(-1, descending=True).values
    keep = lg[:, k - 1] - lg[:, k] > 1e-3
    assert keep.float().mean() > 0.97
    assert torch.equal(ids[keep], torch.topk(logits.detach(), k, -1).indices[keep]), "engine routing differs from fp64"
    err = (out.double().cpu() - ref.detach())[keep].abs().max().item()
    assert err < 3e-2 * ref.detach().abs().max().item(), f"forward: max err {err}"
    dy = torch.randn(M, H, generator=g).to(dev)
    dx = moe.backward(dy, saved, mw)
    ref.backward(dy.double().cpu())
    gref = x64.grad
    derr = (dx.double().cpu() - gref)[keep].abs().max().item()
    assert derr < 3e-2 * gref.abs().max().item(), f"dx: max err {derr} (max |dx| {gref.abs().max().item()})"


@pytest.mark.gpu
def test_moe_layer_bit_reproducible(ops, dev):
    """forward + backward twice: the same bits (no atomics, fixed orders)"""
    M, E, k, H, I = 2000, 64, 8, 512, 256
    moe, mw, _, g = _layer(dev, E, k, H, I, 9)
    x = torch.randn(M, H, generator=g).to(dev, bf16)
    resid = torch.randn(M, H, generator=g).to(dev)
    dy = torch.randn(M, H, generator=g).to(dev)
    runs = []
    for _ in range(2):
        out, s = moe.forward(x, mw, resid=resid.clone())
        dx = moe.backward(dy, s, mw)
        runs.append((out.clone(), dx.clone(), s.ids.clone(), s.w.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a, b.view(torch.uint8) if b.is_floating_point() else b)


# ----------------------------------------------------------------------------------------------------------------
# decoders against transformers' Qwen3MoeForCausalLM
# ----------------------------------------------------------------------------------------------------------------
# Routing: a token whose k-th and (k+1)-th router logits are closer than the engine's bf16 activations can resolve may pick
# another expert than the fp32 oracle, and its output then differs by far more than any tolerance. So each model test first
# runs the engine, checks that it picks the oracle's experts on every valid token whose oracle gap exceeds ROUTE_MARGIN (and
# that at least 80% of the tokens do), and then runs the oracle on the engine's choice of experts (with the oracle's own
# softmax weights), which leaves every other difference to the tolerances of test_qwen3_gpu.py.
# router logits: their spread is ~4 here (router_std 0.2, H 384 / 512); the bf16 activations before the router move them by
# a few hundredths
ROUTE_MARGIN = 0.1
ROUTER_STD = 0.2


def _moe_model(name, V, seed):
    """(cfg, hub-layout state dict, fused-layout state dict) of a bf16-rounded random Qwen3-MoE"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from model_helpers import r16_2d
    cfg = synthetic.qwen3_moe_config(name, vocab_size=V)
    sd = {k: (v.to(bf16).float() if v.dim() >= 2 else v)
          for k, v in r16_2d(params.random_state_dict("qwen3_moe", cfg, seed=seed, qk_norm_std=0.5, router_std=ROUTER_STD)).items()}
    fused = {k: v for k, v in sd.items() if ".mlp.experts." not in k}
    for l, sparse in enumerate(params.moe_layers(cfg)):
        if sparse:
            p = f"model.layers.{l}.mlp.experts."
            E = cfg["num_experts"]
            fused[p + "gate_up_proj"] = torch.stack([torch.cat([sd[p + f"{e}.gate_proj.weight"], sd[p + f"{e}.up_proj.weight"]])
                                                     for e in range(E)])
            fused[p + "down_proj"] = torch.stack([sd[p + f"{e}.down_proj.weight"] for e in range(E)])
    return cfg, sd, fused


@pytest.fixture
def moe_oracle(monkeypatch):
    """oracle.models.build_causal_lm for qwen3_moe (transformers' Qwen3MoeForCausalLM, fused expert parameters)"""
    from oracle import models as om
    monkeypatch.setitem(om._CAUSAL_LM, "qwen3_moe", "Qwen3Moe")
    return om


def _engine_routing(monkeypatch, dec, ids, mask):
    """the engine's expert choice (int64 [B*L, k] per sparse layer, in layer order) on one forward"""
    from dalm_b200.engine import moe
    got, real = [], moe.forward

    def recording(*a, **kw):
        out, s = real(*a, **kw)
        got.append(s.ids.long().cpu())
        return out, s
    monkeypatch.setattr(moe, "forward", recording)
    dec.forward_final(ids.to(dec.dev), mask.to(dec.dev), save=False)
    monkeypatch.setattr(moe, "forward", real)
    return got


def _sparse_gates(ref, cfg):
    from dalm_b200.engine import params
    return [ref.model.layers[l].mlp.gate for l, s in enumerate(params.moe_layers(cfg)) if s]


def _check_routing_agreement(ref, cfg, ids, mask, engine_ids):
    """the oracle's own router logits on every sparse layer: the engine's experts are the oracle's top-k wherever the
    k-th / (k+1)-th gap exceeds ROUTE_MARGIN, and that covers at least 80% of the valid tokens"""
    k = cfg["num_experts_per_tok"]
    caught = []
    hooks = [g.register_forward_hook(lambda m, i, o: caught.append(i[0].detach().double() @ m.weight.double().t()))
             for g in _sparse_gates(ref, cfg)]
    with torch.no_grad():
        ref(input_ids=ids, attention_mask=mask)
    for h in hooks:
        h.remove()
    valid = mask.bool().view(-1)
    for l, (lg, mine) in enumerate(zip(caught, engine_ids)):
        top = lg.topk(k + 1, -1)
        clear = valid & (top.values[:, k - 1] - top.values[:, k] > ROUTE_MARGIN)
        assert clear.sum() >= 0.8 * valid.sum(), f"sparse layer {l}: only {int(clear.sum())} of {int(valid.sum())} tokens clear"
        bad = clear & (mine.sort(-1).values != top.indices[:, :k].sort(-1).values).any(-1)   # the same set of experts
        assert not bad.any(), f"sparse layer {l}: the engine routes {int(bad.sum())} clear tokens elsewhere"


def _force_routing(monkeypatch, ref, cfg, engine_ids):
    """make the oracle's routers take the engine's experts (weights: the oracle's own fp32 softmax, renormalised as
    configured)"""
    import torch.nn.functional as F
    for gate, sel in zip(_sparse_gates(ref, cfg), engine_ids):
        def fwd(h, gate=gate, sel=sel):
            h = h.reshape(-1, gate.hidden_dim)
            probs = F.softmax(F.linear(h, gate.weight), dtype=torch.float, dim=-1)
            w = probs.gather(1, sel)
            if gate.norm_topk_prob:
                w = w / w.sum(-1, keepdim=True)
            return probs, w.to(probs.dtype), sel
        monkeypatch.setattr(gate, "forward", fwd)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,L,pad", [("qwen3-moe-tiny", 3, 40, "right"), ("qwen3-moe-hd128", 2, 72, "left")])
def test_qwen3_moe_decoder_fwd_bwd_lora(cuda_dev, monkeypatch, moe_oracle, name, B, L, pad):
    """logits, the marginalised loss and the LoRA gradients vs Qwen3MoeForCausalLM (qwen3-moe-tiny: a dense layer between two
    sparse ones, renormalised top-2 of 8, the q/k norm row kernel; qwen3-moe-hd128: every layer sparse, top-4 of 16 not
    renormalised, q/k norm + RoPE in the QKV epilogue). The engine loads the hub layout, the oracle the fused one."""
    from dalm_b200.engine.llama import LlamaDecoder
    from model_helpers import attach_lora, check_decoder, draw_lora_B, pad_mask
    V = 504
    cfg, sd, fused = _moe_model(name, V, seed=3)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=True)
    assert sum("moe" in W for W in dec.layers) == sum(dec.sparse) == (2 if name == "qwen3-moe-tiny" else 2)
    ref = moe_oracle.build_causal_lm(cfg, fused)
    draw_lora_B(dec, torch.Generator().manual_seed(9))
    attach_lora(ref, dec)
    g = torch.Generator().manual_seed(9)
    ids, mask = torch.randint(3, V, (B, L), generator=g), pad_mask(B, L, pad)         # what check_decoder draws from g first
    eng = _engine_routing(monkeypatch, dec, ids, mask)
    _check_routing_agreement(ref, cfg, ids, mask, eng)
    _force_routing(monkeypatch, ref, cfg, eng)
    check_decoder(dec, ref, torch.Generator().manual_seed(9), V, B, L, pad)


def _moe_rag(cuda_dev, monkeypatch, moe_oracle, name, batch):
    from model_helpers import rag_models
    cfg, _, fused = _moe_model(name, 504, seed=12)
    model, enc, dec, bert, ref = rag_models(cuda_dev, cfg, fused)                  # the engine loads the fused layout here
    ids, mask = batch["generator_input_input_ids"], batch["generator_input_attention_mask"]
    eng = _engine_routing(monkeypatch, dec, ids, mask)
    _check_routing_agreement(ref, cfg, ids, mask, eng)
    _force_routing(monkeypatch, ref, cfg, eng)
    return model, enc, dec, bert, ref


@pytest.mark.gpu
@pytest.mark.parametrize("name,pad", [("qwen3-moe-tiny", "left"), ("qwen3-moe-hd128", "right")])
def test_fused_rag_step_qwen3_moe_lora(cuda_dev, monkeypatch, moe_oracle, name, pad):
    """bge-tiny + Qwen3-MoE generator, LoRA on both: the fused training step against the reference loop body"""
    from model_helpers import check_rag_lora_grads, rag_batch, rag_step_vs_oracle
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=21, pad=pad)
    model, enc, dec, bert, ref = _moe_rag(cuda_dev, monkeypatch, moe_oracle, name, batch)
    want, _ = rag_step_vs_oracle(model, enc, dec, bert, ref, batch)
    check_rag_lora_grads(enc, dec, want, tol=6e-2)


@pytest.mark.gpu
def test_graphed_step_bit_identical(cuda_dev, monkeypatch, moe_oracle):
    """the step captured as one CUDA graph (GraphedStep: a capture that fails raises here) gives the eager step's loss and
    LoRA gradients bit for bit"""
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_rag_step
    from model_helpers import rag_batch
    batch = rag_batch(5, 12, 24, 40, 600, 504, seed=22)
    model, enc, dec, _, _ = _moe_rag(cuda_dev, monkeypatch, moe_oracle, "qwen3-moe-tiny", batch)
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
        got = [out["losses"], enc.lora.grad, dec.lora.grad]
        for a, b in zip(got, want):
            assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------------------
# generate, and the trainer + eval-rag through the CLI
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [("qwen3-moe-tiny", 4), ("qwen3-moe-hd128", 20)])
def test_qwen3_moe_generate(cuda_dev, monkeypatch, moe_oracle, name, B):
    """greedy decoding: per-step logits and choices vs the oracle teacher-forced on our tokens, and the decode step replayed
    as a CUDA graph gives the eager tokens (check_against_oracle)"""
    from dalm_b200.engine.llama import LlamaDecoder
    from model_helpers import check_against_oracle, prompt
    V = 504
    cfg, sd, fused = _moe_model(name, V, seed=2)
    dec = LlamaDecoder(cfg, sd, device=cuda_dev)
    ref = moe_oracle.build_causal_lm(cfg, fused)
    ids, mask = prompt(B, 12, V, seed=1)
    out, _ = check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert out.shape == (B, 30)


@pytest.mark.gpu
def test_qwen3_moe_generate_sampling_graph(cuda_dev, monkeypatch):
    """sampling under an Instruct-style config: reproducible under torch.manual_seed, graph replay == eager launches"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import decoding
    from dalm_b200.engine.llama import LlamaDecoder
    V = 504
    cfg, sd, _ = _moe_model("qwen3-moe-hd128", V, seed=5)
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


@pytest.mark.gpu
def test_train_and_eval_rag_with_qwen3_moe_directory(cuda_dev, tmp_path, capsys):
    """`dalm train-rag-e2e --use-peft both` on a toy CSV with a synthetic Qwen3-MoE directory writes adapters; eval-rag loads
    them and decodes"""
    from dalm_b200 import synthetic
    from model_helpers import eval_rag_generator, toy_rag_inputs, train_rag_lora
    csv, rdir = toy_rag_inputs(tmp_path)
    gdir = synthetic.write_model_dir(str(tmp_path / "qwen3-moe-tiny"), "qwen3_moe", "qwen3-moe-tiny", vocab_size=1200,
                                     router_std=ROUTER_STD, generation_config=synthetic.QWEN3_GENERATION["base"])
    out = train_rag_lora(csv, rdir, gdir, tmp_path)
    torch.manual_seed(0)
    eval_rag_generator(csv, rdir, gdir, out, capsys)
