"""The routed-expert path at the widths production runs: Qwen3-30B-A3B (H 2048, I 768, 128 experts), OLMoE-1B-7B (H 2048,
I 1024, 64 experts) and a Qwen3-235B-A22B-wide grouped GEMM (H 4096, I 1536, 128 experts), on 4608-token steps routed top-8.

1. The grouped GEMM, all four instances (gate|up with SwiGLU, down, and the two dgrads in the NN layout) at full K, on the
   segment counts of a real routing and of a skewed one (most pairs on three experts, more than half the experts empty, one
   segment of hundreds of tiles), sized for the engine's static tile bound. Integer operands in [-2, 2]: every partial sum
   stays below 2^24, so each segment's rows are bit-exact against fp64. max_ctas 0 (a full wave) and 7 (one CTA crosses
   many expert boundaries, its stage ring wrapping inside every tile). Together with small-bound cases the list reaches
   every tile width (BN 64 / 128 / 256) in both layouts. A tile table that is not in expert order, and the raster / L2
   hint settings, must not change a bit.
2. The routing kernels at production counts: the router's tie rule (lower index first) against a stable sort, the
   permutation at 36 864 and 65 537 pairs and at a tile bound filled exactly, the launchers' refusals, and gather /
   combine / down backward / router backward at H 2048.
3. The layer forward and backward at M 4608 against fp64 on the engine's expert choice, within a bound derived from the
   path's rounding points (see _layer_ref), with a control that drops one expert slot.
4. The layer captured once as a CUDA graph and replayed on batches whose live tile count and tile table differ from the
   captured one: bit-equal to eager runs, and within the fp64 bound.

Inputs are NaN-poisoned views and outputs sit inside sentinel guard bands (exact_helpers). The fp64 references run on the
GPU, per expert or per segment. U = 2^-24 is the fp32 unit roundoff, u = 2^-8 the bf16 one (8 significant bits).
"""
import math

import pytest
import torch

from exact_helpers import (Guarded, _check_routing, _expect_close, _expect_equal, _grouped_case, _pick_block_n, _poisoned,
                           _segments, _silu_tol, _ulp_bf16, _ulp_f32)

pytestmark = pytest.mark.gpu
bf16, f32, f64, i32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
U = 2.0 ** -24
UB = 2.0 ** -8
TOKENS, TOP_K = 4608, 8                          # a cfg-3 step: 36 864 (token, slot) pairs


@pytest.fixture(scope="module")
def ops(cuda_dev):
    from dalm_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _free(cuda_dev):
    """the buffers here are large: give them back to the allocator between tests"""
    yield
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------
# 1. grouped GEMM at production widths
# ----------------------------------------------------------------------------------------------------------------
MODELS = {"qwen3-30b-a3b": (2048, 768, 128), "olmoe-1b-7b": (2048, 1024, 64), "qwen3-235b-a22b": (4096, 1536, 128)}
# instance -> (layout, swiglu, (N, K) at hidden H / intermediate I), as engine/moe.py calls them
INSTANCES = {
    "gate_up": (0, True, lambda H, I: (2 * I, H)),
    "down": (0, False, lambda H, I: (H, I)),
    "down_dgrad": (1, False, lambda H, I: (I, H)),
    "gate_up_dgrad": (1, False, lambda H, I: (H, 2 * I)),
}
# small static bounds, where the tile-width rule picks 64 or 128: (counts, extra tiles, layout, N, K)
SMALL = {
    "small_tn_bn128": ([0, 1, 128, 0, 300, 256, 0, 5], 2, 0, 1024, 2048),
    "small_nn_bn128": ([0, 1, 128, 0, 300, 256, 0, 5], 2, 1, 1024, 2048),
    "small_tn_bn64": ([0, 0, 0, 700, 0, 0], 1, 0, 200, 2048),
    "small_nn_bn64": ([0, 0, 0, 700, 0, 0], 1, 1, 192, 2048),
}
GROUPED = [(m, inst, rt) for m in MODELS for inst in INSTANCES for rt in ("router", "skewed")] + [(s, None, None) for s in SMALL]


def _router_counts(ops, dev, E, seed):
    """per-expert pair counts of a 4608-token step routed top-8 by the router kernel"""
    g = torch.Generator(device=dev).manual_seed(seed)
    ids, _ = ops.moe_router(torch.randn(TOKENS, E, generator=g, device=dev) * 2, TOP_K, True)
    return torch.bincount(ids.view(-1).long(), minlength=E).tolist()


def _skewed_counts(E):
    """36 864 pairs: 30 000 on one expert (235 tiles), 4 000 and 2 000 on two more, 864 over 20 others, the rest empty"""
    c = [0] * E
    c[5], c[E - 40], c[E - 1] = 30000, 4000, 2000
    for j in range(20):
        c[7 + 2 * j] = 43 + (j < 4)
    assert sum(c) == TOKENS * TOP_K
    return c


def _grouped_shape(name, inst):
    """(layout, swiglu, N, K, E, static bound of tiles or None)"""
    if inst is None:
        counts, extra, layout, N, K = SMALL[name]
        return layout, False, N, K, len(counts), _segments(counts)[1] // 128 + extra
    H, I, E = MODELS[name]
    layout, swiglu, nk = INSTANCES[inst]
    return (layout, swiglu) + nk(H, I) + (E, -(-(TOKENS * TOP_K + 127 * E) // 128))


def _block_n(case, sms):
    layout, swiglu, N, _, _, tiles = _grouped_shape(*case[:2])
    return layout, 256 if swiglu else _pick_block_n(128 * tiles, N, sms)


def test_grouped_cases_reach_every_block_n(ops):
    """the case list below makes pick_block_n (restated in exact_helpers._pick_block_n) choose each of BN 64, 128 and 256 in
    both layouts; at the production bounds it picks 256 for every instance"""
    sms = ops.num_sms()
    reached = {_block_n(c, sms) for c in GROUPED}
    assert reached >= {(lay, bn) for lay in (0, 1) for bn in (64, 128, 256)}, f"{sms} SMs: reached {sorted(reached)}"
    assert all(_block_n(c, sms)[1] == 256 for c in GROUPED if c[1] is not None), "production bounds pick BN 256"


@pytest.mark.parametrize("name,inst,routing", GROUPED, ids=[f"{m}-{i}-{r}" if i else m for m, i, r in GROUPED])
def test_grouped_gemm_production_widths(ops, cuda_dev, name, inst, routing):
    """every segment bit-exact against fp64, rows past the live tiles untouched, at max_ctas 0 and 7"""
    layout, swiglu, N, K, E, tiles = _grouped_shape(name, inst)
    if inst is None:
        counts, extra = SMALL[name][:2]
    else:
        counts = _router_counts(ops, cuda_dev, E, seed=E) if routing == "router" else _skewed_counts(E)
        extra = tiles - _segments(counts)[1] // 128
        assert extra >= 0
        if routing == "skewed":
            assert sum(c == 0 for c in counts) > E // 2 and max(counts) > 200 * 128
    for i, max_ctas in enumerate((0, 7)):
        _grouped_case(ops, cuda_dev, counts, extra, layout, swiglu, N, K, max_ctas, seed=17 * i + N + K, E=E, device_ref=True)


def _shuffled_segments(counts, seed):
    """the routing's segments in a random expert order, ten of them split in two parts placed far apart: the tile table
    repeats experts in non-adjacent tiles and is not monotone"""
    g = torch.Generator().manual_seed(seed)
    order = [e for e in torch.randperm(len(counts), generator=g).tolist() if counts[e] > 0]
    segs = [(e, counts[e]) for e in order]
    for j in range(10):
        e, c = segs[j]
        segs[j] = (e, c // 3)
        segs.insert(len(segs) - 3 * j, (e, c - c // 3))
    return [c for _, c in segs], [e for e, _ in segs]


@pytest.mark.parametrize("inst", ["down", "gate_up_dgrad"])
def test_grouped_gemm_shuffled_tile_table(ops, cuda_dev, inst):
    """tile m uses expert tile_expert[m], whatever the order of the segments"""
    H, I, E = MODELS["qwen3-30b-a3b"]
    layout, swiglu, nk = INSTANCES[inst]
    N, K = nk(H, I)
    counts, experts = _shuffled_segments(_router_counts(ops, cuda_dev, E, seed=3), seed=4)
    assert len(set(experts)) < len(experts) and experts != sorted(experts)
    for max_ctas in (0, 7):
        _grouped_case(ops, cuda_dev, counts, 3, layout, swiglu, N, K, max_ctas, seed=5 + max_ctas, experts=experts, E=E,
                      device_ref=True)


def test_grouped_gemm_raster_and_l2_hints_do_not_change_results(ops, cuda_dev):
    """raster order and TMA L2 eviction hints are performance hints: the Qwen3-30B-A3B down projection and gate|up dgrad
    stay bit-exact under every setting"""
    from dalm_b200 import _lib
    H, I, E = MODELS["qwen3-30b-a3b"]
    counts = _router_counts(ops, cuda_dev, E, seed=E)
    extra = -(-(TOKENS * TOP_K + 127 * E) // 128) - _segments(counts)[1] // 128
    lib = _lib.load()
    try:
        for raster in (0, -1, -2):
            for hints in (0, 1, 2, 7):
                lib.dalm_b200_gemm_set_raster(raster)
                lib.dalm_b200_gemm_set_l2_hints(hints)
                for layout, (N, K) in ((0, (H, I)), (1, (H, 2 * I))):
                    _grouped_case(ops, cuda_dev, counts, extra, layout, False, N, K, 0, seed=1, E=E, device_ref=True)
    finally:
        lib.dalm_b200_gemm_set_raster(0)
        lib.dalm_b200_gemm_set_l2_hints(-1)


# ----------------------------------------------------------------------------------------------------------------
# 2. routing kernels at production counts
# ----------------------------------------------------------------------------------------------------------------
def _tied_logits(M, E, dev, seed):
    """logits from seven values (each row ties inside its top k and across the k-th place), every 7th row continuous,
    every 97th row all equal"""
    g = torch.Generator(device=dev).manual_seed(seed)
    lg = torch.randint(-3, 4, (M, E), generator=g, device=dev).float() * 0.75
    lg[1::7] = torch.randn(lg[1::7].shape, generator=g, device=dev) * 2
    lg[3::97] = 0.5
    return lg


@pytest.mark.parametrize("E,k", [(128, 8), (64, 8), (256, 16)])
@pytest.mark.parametrize("norm", [False, True])
def test_router_ties_production_counts(ops, cuda_dev, E, k, norm):
    """ids == the first k of a stable descending sort (ties to the lower index); rows of equal logits pick experts 0..k-1.
    Weights against fp64: expf within 2 ulp (own term and the sum), a sum of E / 32 serial terms per lane and a 5-level
    butterfly, one division, and the argument's rounding (U |l - max| <= U span): relative (E/32 + 14 + 2 span) U; the
    renormalised weight twice that plus k + 1 roundings"""
    M = TOKENS
    lg = _tied_logits(M, E, cuda_dev, seed=E + k)
    ids, w = ops.moe_router(_poisoned(lg), k, norm)
    want = torch.sort(-lg, dim=1, stable=True).indices[:, :k]
    bad = (ids.long() != want).any(1)
    assert not bad.any(), f"E {E} k {k}: {int(bad.sum())} rows differ from the stable order; first row {int(bad.nonzero()[0])}: " \
                          f"{ids[bad][0].tolist()} vs {want[bad][0].tolist()}"
    assert torch.equal(ids[3::97].long(), torch.arange(k, device=cuda_dev).expand(ids[3::97].shape[0], k))
    ties = (lg.gather(1, want[:, k - 1:k]) == lg).sum(1) > 1
    assert ties.float().mean() > 0.5, "most rows tie at the k-th place"
    p = torch.softmax(lg.double(), -1).gather(1, ids.long())
    span = (lg.amax(1, keepdim=True) - lg.amin(1, keepdim=True)).double()
    rel = (E / 32 + 14 + 2 * span) * U
    ref, tol = (p / p.sum(-1, keepdim=True), (2 * rel + (k + 1) * U) * p / p.sum(-1, keepdim=True)) if norm else (p, rel * p)
    _expect_close(w, ref, tol, f"router weights E {E} k {k} norm {norm}")


@pytest.mark.parametrize("case", ["router", "single_pair_chunk", "one_expert", "full_bound"])
def test_permute_production_counts(ops, cuda_dev, case):
    """router: 36 864 pairs (36 chunks of 1024) over 128 experts; single_pair_chunk: 65 537 pairs of k = 1, the last chunk
    one pair; one_expert: 36 864 pairs on one expert; full_bound: every expert's count 1 mod 128, so the live tiles fill
    n_tiles = moe_tiles(P, E) exactly (P + 127 E a multiple of 128)"""
    dev, E = cuda_dev, 128
    g = torch.Generator(device=dev).manual_seed(23)
    if case == "router":
        ids, _ = ops.moe_router(torch.randn(TOKENS, E, generator=g, device=dev), TOP_K, True)
    elif case == "single_pair_chunk":
        ids = torch.randint(0, E, (65537, 1), generator=g, device=dev, dtype=i32)
    elif case == "one_expert":
        ids = torch.full((TOKENS, TOP_K), 77, dtype=i32, device=dev)
    else:
        cnt = 1 + 128 * torch.randint(0, 5, (E,), generator=g, device=dev)
        flat = torch.repeat_interleave(torch.arange(E, device=dev), cnt)
        ids = flat[torch.randperm(flat.numel(), generator=g, device=dev)].view(-1, TOP_K).to(i32)
        assert (ids.numel() + 127 * E) % 128 == 0
    ids = ids.contiguous()
    r = ops.moe_permute(ids, E)
    assert r.n_tiles == ops.moe_tiles(ids.numel(), E)
    _check_routing(r, ids, E)
    if case == "full_bound":
        assert int(r.live.item()) == r.n_tiles


def test_routing_refusals(ops, cuda_dev):
    """a tile bound one short of moe_tiles(P, E), and router shapes past its limits, are refused by name"""
    Err = ops._lib.DalmB200Error
    dev, E, P = cuda_dev, 128, TOKENS * TOP_K
    ids = torch.zeros(TOKENS, TOP_K, dtype=i32, device=dev)
    short = ops.MoeRouting(TOKENS, TOP_K, E, dev, n_tiles=ops.moe_tiles(P, E) - 1)
    with pytest.raises(Err, match=f"moe_permute: {ops.moe_tiles(P, E) - 1} M tiles cannot hold {P} pairs"):
        ops.moe_permute(ids, E, short)
    with pytest.raises(Err, match="moe_router: E=257"):
        ops.moe_router(torch.zeros(8, 257, device=dev), 8, True)
    with pytest.raises(Err, match="moe_router: top-k=17"):
        ops.moe_router(torch.zeros(8, 64, device=dev), 17, True)
    with pytest.raises(Err, match="moe_router: top-k=5"):
        ops.moe_router(torch.zeros(8, 4, device=dev), 5, True)
    torch.cuda.synchronize()


def _routed(ops, dev, E, norm, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    logits = torch.randn(TOKENS, E, generator=g, device=dev) * 2
    ids, w = ops.moe_router(logits, TOP_K, norm)
    return g, logits, ids, w, ops.moe_permute(ids, E)


def _nan_padding(t, r):
    """t [rows, n] with every row that holds no pair (segment padding, tail tiles) set to NaN"""
    t[r.row_pair.long() < 0] = float("nan")
    t[int(r.live.item()) * 128:] = float("nan")
    return t


@pytest.mark.parametrize("I,E,norm", [(768, 128, True), (1024, 64, False)], ids=["qwen3-30b-a3b", "olmoe-1b-7b"])
def test_row_kernels_production_widths(ops, cuda_dev, I, E, norm):
    """gather (bf16 / fp32 sources), combine (weighted / unweighted, fp32 / bf16, out aliased to the residual), the down
    backward (separate d_act and d_act = act, the engine's call) and the router backward at H 2048, k 8, 4608 tokens"""
    dev, H, k, M = cuda_dev, 2048, TOP_K, TOKENS
    g, logits, ids, w, r = _routed(ops, dev, E, norm, seed=I)
    live = int(r.live.item()) * 128
    rp = r.row_pair[:live].long()
    has = (rp >= 0)[:, None]
    # gather: every live row its token's row (0 on padding rows), rows past the live tiles untouched
    for dt in (bf16, f32):
        x = torch.randn(M, H, generator=g, device=dev).to(dt)
        out = Guarded(r.rows, H, bf16, dev)
        ops.moe_gather(_poisoned(x), r, out=out.view)
        _expect_equal(out.view[:live], torch.where(has, x[rp.clamp_min(0) // k], torch.zeros((), dtype=dt, device=dev)).to(bf16),
                      f"moe_gather {dt} E {E}")
        assert bool((out.view[live:].contiguous().view(torch.int16) == out.bits).all()), "moe_gather wrote past the live tiles"
        out.check(f"moe_gather {dt}")
    # combine: fp32 fma chain over the slots, then the residual: (k + 2) U of the magnitudes, plus bf16's rounding
    y = _poisoned(_nan_padding(torch.randn(r.rows, H, generator=g, device=dev).to(bf16), r))
    yp = y[r.pair_row.long()].double().view(M, k, H)
    for weighted, dt, alias in ((True, f32, False), (True, bf16, True), (False, f32, True), (False, bf16, False)):
        resid = torch.randn(M, H, generator=g, device=dev).to(dt)
        wt = w.double()[..., None] if weighted else torch.ones(M, k, 1, dtype=f64, device=dev)
        ref = resid.double() + (wt * yp).sum(1)
        tol = (k + 2) * _ulp_f32(resid.double().abs() + (wt * yp).abs().sum(1)) + (_ulp_bf16(ref) if dt == bf16 else 0)
        what = f"moe_combine weighted {weighted} {dt} aliased {alias}"
        if alias:
            out = Guarded(M, H, dt, dev, init=resid)
            ops.moe_combine(y, r, w if weighted else None, resid=out.view, out=out.view)
        else:
            out = Guarded(M, H, dt, dev)
            ops.moe_combine(y, r, w if weighted else None, resid=_poisoned(resid), out=out.view)
        _expect_close(out.view, ref, tol, what)
        out.check(what)
    # down backward: dw = <da, act> (fp32, I / 256 chunks of 8 per lane and a butterfly), d_act = bf16(w da)
    da = _poisoned(_nan_padding(torch.randn(r.rows, I, generator=g, device=dev).to(bf16), r))
    act0 = _nan_padding(torch.randn(r.rows, I, generator=g, device=dev).to(bf16), r)
    pr = r.pair_row.long()
    ref_dw = (da[pr].double() * act0[pr].double()).sum(-1).view(M, k)
    tol_dw = (I / 8 + 8) * _ulp_f32((da[pr].double() * act0[pr].double()).abs().sum(-1)).view(M, k)
    ref_da = (w.view(-1)[:, None] * da[pr].float()).to(bf16)
    sep = Guarded(r.rows, I, bf16, dev)
    dw, _ = ops.moe_down_bwd(da, _poisoned(act0), r, w, d_act=sep.view)
    _expect_close(dw, ref_dw, tol_dw, "moe_down_bwd dw")
    _expect_equal(sep.view[pr], ref_da, "moe_down_bwd d_act")
    pad = torch.ones(r.rows, dtype=torch.bool, device=dev)
    pad[pr] = False
    assert bool((sep.view[pad].view(torch.int16) == sep.bits).all()), "moe_down_bwd wrote rows that hold no pair"
    sep.check("moe_down_bwd d_act")
    inp = Guarded(r.rows, I, bf16, dev, init=act0)
    dw2, _ = ops.moe_down_bwd(da, inp.view, r, w, d_act=inp.view)
    assert torch.equal(dw2, dw), "moe_down_bwd in place: dw differs from the separate call"
    _expect_equal(inp.view[pr], ref_da, "moe_down_bwd d_act in place")
    assert torch.equal(inp.view[pad].view(torch.int16), act0[pad].view(torch.int16)), "moe_down_bwd in place: rows without a pair changed"
    inp.check("moe_down_bwd in place")
    # router backward against fp64 autograd of softmax, top-k gather and renormalisation
    lg = logits.double().clone().requires_grad_(True)
    p = torch.softmax(lg, -1).gather(1, ids.long())
    wt = p / p.sum(-1, keepdim=True) if norm else p
    (wt * dw.double()).sum().backward()
    ref = lg.grad
    out = Guarded(M, E, bf16, dev)
    ops.moe_router_bwd(_poisoned(logits), ids, w, dw, norm, out=out.view)
    S = torch.softmax(logits.double(), -1).gather(1, ids.long()).sum(-1, keepdim=True)
    scale = dw.double().abs().sum(-1, keepdim=True) / (S if norm else 1.0)
    _expect_close(out.view, ref, _ulp_bf16(ref) + 2.0 ** -18 * scale, f"moe_router_bwd E {E} norm {norm}")
    out.check("moe_router_bwd")


# ----------------------------------------------------------------------------------------------------------------
# 3. the layer against fp64
# ----------------------------------------------------------------------------------------------------------------
LAYERS = {"qwen3-30b-a3b": (2048, 768, 128, True), "olmoe-1b-7b": (2048, 1024, 64, False)}


def _gam(n):
    """bound on the fp32 tensor-core sum of n products, relative to the sum of their magnitudes: one block FMA per 16
    products (a wgmma k-step) added to the accumulator, each within 2 U, and 8 more for the epilogue"""
    return 2 * (n / 16 + 8) * U


def _r2(v):
    """variance of v's round-to-nearest bf16 rounding error, at most (u v)^2 / 3"""
    return (UB * v).square() / 3


Z_BWD = 6                                        # standard deviations of the backward's rounding noise: ~2e-9 per element


def _layer_weights(dev, name, seed):
    """bf16 weights of one sparse layer of this model's widths (router logits of spread ~2 on unit-variance inputs)"""
    from dalm_b200.engine import moe
    H, I, E, norm = LAYERS[name]
    g = torch.Generator(device=dev).manual_seed(seed)
    gate = torch.randn(E, H, generator=g, device=dev) * (2 / math.sqrt(H))
    gp = torch.randn(E, I, H, generator=g, device=dev) * H ** -0.5
    up = torch.randn(E, I, H, generator=g, device=dev) * H ** -0.5
    down = torch.randn(E, H, I, generator=g, device=dev) * I ** -0.5
    mw = moe.pack_experts(gate, gp, up, down, TOP_K, norm, dev)
    w16 = {"gate": gate.to(bf16), "gp": gp.to(bf16), "up": up.to(bf16), "down": down.to(bf16)}
    return mw, w16


def _layer_ref(x, resid, dy, w16, ids, norm):
    """fp64 Qwen3MoeSparseMoeBlock forward and input gradient on the given expert choice, one expert at a time, with
    first-order bounds on the engine's error. Rounding points of the engine and the bound terms they give (|.| element-wise,
    products of magnitudes through the weights' magnitudes, gam(n) = _gam(n)):
      router     fp32 logits: dl = gam(H) |x| |Wr|; softmax within eps_p = 2 max dl + (E/32 + 14 + 2 span) U (the router
                 test), weights eps_w = eps_p (renormalised: 2 eps_p + (k + 1) U)
      gate|up    fp32 sums: dG = gam(H) |x| |Wg|, dV = gam(H) |x| |Wu|; stored as bf16 gu (+ u |G|, u |V| in the backward)
      act        silu(G) V from the fp32 sums, rounded to bf16: dA = u |A| + |dA/dG| dG + |silu G| dV + silu_tol |A|
      y          bf16 of the fp32 sum over I: dY = u |Y| + dA |Wd| + gam(I) |A| |Wd|
      combine    fp32: dout = sum_s (|w_s| dY_s + eps_w |w_s Y_s|) + (k + 2) U (|resid| + sum_s |w_s Y_s|)
    The backward chains two contractions (over H into da, over I into dw and over 2I into dx), where worst-case sums of the
    bf16 roundings exceed |dx| itself. So there each bf16 rounding of v counts as an independent error of variance
    (u v)^2 / 3 (round to nearest: uniform within half an ulp <= u |v|), carried through the weights' squares, and dx may
    be off by Z_BWD standard deviations plus the worst-case sum of the fp32 and approximation terms (a*):
      da         bf16(bf16(dy) W_down): a = gam(H) |dy| |Wd|, var from dy's and da's roundings
      dw         fp32 <da, act>: a = sum_i (aDa |A| + |Da| aA) + (I/8 + 8) U sum |Da A| (aA: dA without its u |A|)
      d_act      bf16(w da): a = eps_w |w Da| + |w| aDa + U |w Da|
      swiglu_bwd bf16 dgate = Dact V h(G), dup = Dact silu(G), h = sigma (1 + G (1 - sigma)), from the bf16 gu (its
                 rounding a variance, dG / dV worst-case), with __expf's sigmoid (silu_tol)
      dxr        bf16 of the fp32 sum over 2I: a = aDg |Wg| + aDu |Wu| + gam(2I) (|Dg| |Wg| + |Du| |Wu|)
      router bwd g_s = (dw_s - sum_r dw_r w_r) / S, dlogit_j = p_j (g_j - sum_s P_s g_s), rounded to bf16; eps_p and a few
                 U worst-case, dw's deviation carried through (standard deviations add)
      dx         fp32 dlogits W_gate (gam(E)) and the fp32 sum with the k dxr rows ((k + 2) U)
    -> (out, dx, out_tol, dx_tol, contribution of slot 0 [M, H], fp64 router logits), fp64"""
    M, H = x.shape
    E, I = w16["gp"].shape[0], w16["gp"].shape[1]
    k = ids.shape[1]
    X = x.double()
    Wr = w16["gate"].double()
    l = X @ Wr.t()
    dl = _gam(H) * (X.abs() @ Wr.abs().t())
    span = l.amax(1, keepdim=True) - l.amin(1, keepdim=True)
    eps_p = 2 * dl.amax(1, keepdim=True) + (E / 32 + 14 + 2 * span) * U                               # [M, 1]
    p = torch.softmax(l, -1)
    P = p.gather(1, ids)
    S = P.sum(-1, keepdim=True)
    w = P / S if norm else P
    eps_w = 2 * eps_p + (k + 1) * U if norm else eps_p
    out = resid.double().clone()
    out_err = torch.zeros(M, H, dtype=f64, device=x.device)
    mag = resid.double().abs()
    slot0 = torch.zeros(M, H, dtype=f64, device=x.device)
    dxr_sum = torch.zeros(M, H, dtype=f64, device=x.device)
    dxr_a, dxr_s, dxr_mag = (torch.zeros(M, H, dtype=f64, device=x.device) for _ in range(3))
    dw, adw, sdw = (torch.zeros(M, k, dtype=f64, device=x.device) for _ in range(3))
    gy_all = dy.to(bf16).double()
    for e in range(E):
        tok, slot = (ids == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        Wg, Wu, Wd = w16["gp"][e].double(), w16["up"][e].double(), w16["down"][e].double()
        aWg, aWu, aWd = Wg.abs(), Wu.abs(), Wd.abs()
        Xe = X[tok]
        G, V = Xe @ Wg.t(), Xe @ Wu.t()
        aX = Xe.abs()
        dG, dV = _gam(H) * (aX @ aWg.t()), _gam(H) * (aX @ aWu.t())
        sg = torch.sigmoid(G)
        silu = G * sg
        h = sg * (1 + G * (1 - sg))
        A = silu * V
        dA = UB * A.abs() + (V * h).abs() * dG + silu.abs() * dV + (_silu_tol(G) + U) * A.abs()
        Y = A @ Wd.t()
        dY = UB * Y.abs() + dA @ aWd.t() + _gam(I) * (A.abs() @ aWd.t())
        we, ew = w[tok, slot][:, None], eps_w[tok]
        out.index_add_(0, tok, we * Y)
        out_err.index_add_(0, tok, we.abs() * dY + ew * (we * Y).abs())
        mag.index_add_(0, tok, (we * Y).abs())
        first = slot == 0
        slot0[tok[first]] = (we * Y)[first]
        # backward: worst-case parts a*, variances s* of the bf16 roundings
        gy = gy_all[tok]
        Da = gy @ Wd
        aDa = _gam(H) * (gy.abs() @ aWd)
        sDa = _r2(gy) @ Wd.square() + _r2(Da)
        aA, sA = dA - UB * A.abs(), _r2(A)
        dw[tok, slot] = (Da * A).sum(-1)
        adw[tok, slot] = (aDa * A.abs() + Da.abs() * aA).sum(-1) + (I / 8 + 8) * U * (Da * A).abs().sum(-1)
        sdw[tok, slot] = (sDa * A.square() + Da.square() * sA).sum(-1)
        Dact = we * Da
        aDact = ew * Dact.abs() + we.abs() * aDa + U * Dact.abs()
        sDact = we.square() * sDa + _r2(Dact)
        sG, sV = _r2(G), _r2(V)                                                   # gu is read back as bf16
        hp = sg * (1 - sg) * (2 + G * (1 - 2 * sg))
        Dg, Du = Dact * V * h, Dact * silu
        st = _silu_tol(G)
        aDg = aDact * (V * h).abs() + (Dact * h).abs() * dV + (Dact * V * hp).abs() * dG \
            + 4 * st * (Dact * V * sg).abs() * (1 + G.abs())
        sDg = (V * h).square() * sDact + (Dact * h).square() * sV + (Dact * V * hp).square() * sG + _r2(Dg)
        aDu = aDact * silu.abs() + (Dact * h).abs() * dG + st * Du.abs()
        sDu = silu.square() * sDact + (Dact * h).square() * sG + _r2(Du)
        Dxr = Dg @ Wg + Du @ Wu
        dxr_sum.index_add_(0, tok, Dxr)
        dxr_a.index_add_(0, tok, aDg @ aWg + aDu @ aWu + _gam(2 * I) * (Dg.abs() @ aWg + Du.abs() @ aWu))
        dxr_s.index_add_(0, tok, sDg @ Wg.square() + sDu @ Wu.square() + _r2(Dxr))
        dxr_mag.index_add_(0, tok, Dxr.abs())
    out_tol = out_err + (k + 2) * U * mag
    # router backward (standard deviations add: std(a + b) <= std a + std b)
    sd = sdw.sqrt()
    if norm:
        dot = (dw * w).sum(-1, keepdim=True)
        gs = (dw - dot) / S
        ags = (adw + (adw * w.abs() + eps_w * (dw * w).abs()).sum(-1, keepdim=True)) / S + (eps_p + k * U) * gs.abs() \
            + 4 * U * (dw.abs() + (dw * w).abs().sum(-1, keepdim=True)) / S
        sgs = (sd + (w.abs() * sd).sum(-1, keepdim=True)) / S
    else:
        gs, ags, sgs = dw, adw, sd
    pg = (P * gs).sum(-1, keepdim=True)
    apg = (P * ags + eps_p * (P * gs).abs()).sum(-1, keepdim=True) + k * U * (P * gs).abs().sum(-1, keepdim=True)
    spg = (P * sgs).sum(-1, keepdim=True)
    gj = torch.zeros(M, E, dtype=f64, device=x.device).scatter_(1, ids, gs)
    agj = torch.zeros(M, E, dtype=f64, device=x.device).scatter_(1, ids, ags)
    sgj = torch.zeros(M, E, dtype=f64, device=x.device).scatter_(1, ids, sgs)
    Dl = p * (gj - pg)
    aDl = p * (agj + apg) + (eps_p + 3 * U) * p * (gj.abs() + pg.abs())
    sDl = (p * (sgj + spg)).square() + _r2(Dl)
    dx_router = Dl @ Wr
    dx = dx_router + dxr_sum
    dx_a = dxr_a + aDl @ Wr.abs() + _gam(E) * (Dl.abs() @ Wr.abs()) + (k + 2) * U * (dx_router.abs() + dxr_mag)
    dx_tol = dx_a + Z_BWD * (dxr_s + sDl @ Wr.square()).sqrt()
    return out, dx, out_tol, dx_tol, slot0, l


def _check_layer(what, ids, out, dx, ref, min_keep=0.97, control=True):
    """the engine's choice on the tokens that are not near-ties, then out and dx within the bounds, on those tokens; the
    control: the reference without slot 0's contribution must miss the forward bound on most of them"""
    ro, rdx, otol, dxtol, slot0, l = ref
    k = ids.shape[1]
    # a choice flips only where the k-th and (k+1)-th logits are closer than the fp32 logits' error (~1e-5): tokens closer
    # than 1e-3 are left out of the comparison
    top = l.topk(k + 1, -1)
    keep = top.values[:, k - 1] - top.values[:, k] > 1e-3
    assert keep.float().mean() >= min_keep, f"{what}: only {int(keep.sum())} of {keep.numel()} tokens clear"
    same = ids.long()[keep].sort(-1).values == top.indices[keep, :k].sort(-1).values
    assert bool(same.all()), f"{what}: the engine routes {int((~same.all(1)).sum())} clear tokens to other experts than fp64"
    for nm, got, want, tol in (("out", out, ro, otol), ("dx", dx, rdx, dxtol)):
        err = (got.double() - want).abs()[keep]
        print(f"[moe] {what} {nm}: max err / bound {(err / tol[keep]).max().item():.3f}, max err {err.max().item():.3e}")
        _expect_close(got[keep], want[keep], tol[keep], f"{what} {nm}")
    if control:
        miss = ((out.double() - (ro - slot0)).abs() > otol).any(1)[keep]
        print(f"[moe] {what} control: slot 0 dropped misses the bound on {miss.float().mean().item():.1%} of the tokens")
        assert miss.float().mean() > 0.99, f"{what}: a lost expert slot stays within the bound on {int((~miss).sum())} tokens"


@pytest.mark.parametrize("name", list(LAYERS))
def test_moe_layer_production_widths(ops, cuda_dev, name):
    """moe.forward and moe.backward at M 4608 against fp64 on the engine's expert choice, within _layer_ref's bound"""
    from dalm_b200.engine import moe
    dev = cuda_dev
    mw, w16 = _layer_weights(dev, name, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    H = w16["gate"].shape[1]
    x = torch.randn(TOKENS, H, generator=g, device=dev).to(bf16)
    resid = torch.randn(TOKENS, H, generator=g, device=dev)
    dy = torch.randn(TOKENS, H, generator=g, device=dev)
    out, saved = moe.forward(x, mw, resid=resid.clone())
    dx = moe.backward(dy, saved, mw)
    ids = saved.ids.long()
    ref = _layer_ref(x, resid, dy, w16, ids, mw.norm_topk)
    _check_layer(name, ids, out, dx, ref)
    print(f"[moe] {name}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


# ----------------------------------------------------------------------------------------------------------------
# 4. graph replay under changing routes
# ----------------------------------------------------------------------------------------------------------------
def _direction(w16, experts, H, dev):
    """a unit-variance token direction whose router logits rank exactly these experts first"""
    v = w16["gate"].float()[experts].sum(0)
    return v * (math.sqrt(H) / v.norm())


def _replay_inputs(w16, M, H, dev, seed):
    """(a) random tokens, (b) every token a power-of-two multiple of one direction (the same k experts everywhere: k full
    segments, E - k empty), (c) two populations on disjoint expert sets, (a) again"""
    g = torch.Generator(device=dev).manual_seed(seed)
    E = w16["gate"].shape[0]
    s1, s2 = list(range(0, 2 * TOP_K, 2)), list(range(E - 2 * TOP_K + 1, E, 2))
    v1, v2 = _direction(w16, s1, H, dev), _direction(w16, s2, H, dev)
    scale = 2.0 ** (torch.arange(M, device=dev) % 3 - 1).float()[:, None]
    rand = torch.randn(M, H, generator=g, device=dev).to(bf16)
    pop = torch.where((torch.arange(M, device=dev) % 2 == 0)[:, None], v1, v2)
    return [("random", rand, None), ("one_direction", (scale * v1).to(bf16), [s1]), ("two_populations", pop.to(bf16), [s1, s2]),
            ("random_again", rand, None)]


@pytest.mark.parametrize("M,max_ctas", [(1024, 0), (20, 7)])
def test_moe_graph_replay_changing_routes(ops, cuda_dev, M, max_ctas):
    """moe.forward + moe.backward captured once at Qwen3-30B-A3B widths, replayed on batches with other live tile counts
    and tile tables: out, dx, ids and weights bit-equal to eager runs with the same max_ctas; at the decode size also
    within the fp64 bound of test_moe_layer_production_widths"""
    from dalm_b200.engine import moe
    dev = cuda_dev
    mw, w16 = _layer_weights(dev, "qwen3-30b-a3b", seed=3)
    H, E = w16["gate"].shape[1], w16["gate"].shape[0]
    g = torch.Generator(device=dev).manual_seed(4)
    cases = _replay_inputs(w16, M, H, dev, seed=5)
    x_s = torch.randn(M, H, generator=g, device=dev).to(bf16)     # the captured batch: none of the replayed ones
    r_s = torch.randn(M, H, generator=g, device=dev)
    dy_s = torch.randn(M, H, generator=g, device=dev)

    def step():
        out, saved = moe.forward(x_s, mw, resid=r_s, max_ctas=max_ctas)
        dx = moe.backward(dy_s, saved, mw, max_ctas=max_ctas)
        return out, dx, saved.ids, saved.w, saved.routing.live, saved.routing.tile_expert

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    torch.cuda.synchronize()
    tables = [static[5].clone()]
    lives = []
    for nm, x, sets in cases:
        out_e, saved_e = moe.forward(x, mw, resid=r_s.clone(), max_ctas=max_ctas)
        dx_e = moe.backward(dy_s, saved_e, mw, max_ctas=max_ctas)
        want = (out_e, dx_e, saved_e.ids, saved_e.w)
        if sets is not None:                                       # the inputs route as constructed
            for i, s in enumerate(sets):
                rows = saved_e.ids[i::len(sets)].long().sort(-1).values
                assert bool((rows == torch.tensor(s, device=dev)).all()), f"{nm}: tokens do not route to {s}"
        x_s.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        live = int(static[4].item())
        lives.append(live)
        tables.append(static[5].clone())
        assert live == int(saved_e.routing.live.item()) and torch.equal(static[5], saved_e.routing.tile_expert)
        for part, a, b in zip(("out", "dx", "ids", "w"), static[:4], want):
            assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a, b.view(torch.uint8) if b.is_floating_point() else b), \
                f"M {M} {nm}: replayed {part} differs from the eager run"
        if M <= 20:
            ref = _layer_ref(x, r_s, dy_s, w16, static[2].long(), mw.norm_topk)
            _check_layer(f"replay M {M} {nm}", static[2], static[0], static[1], ref, min_keep=0.9, control=False)
    assert lives[1] == TOP_K * -(-M // 128), "one direction: k full segments"
    for i in range(4):                                             # captured, (a), (b), (c): four different tile tables
        for j in range(i):
            assert not torch.equal(tables[i], tables[j]), f"M {M}: tile tables {j} and {i} are the same"
