"""-m gpu: greedy decoding (the generator half of `dalm eval-rag`, reference dalm/eval/eval_rag.py:126-140).

Kernel level: `rope_pos`, `attention_decode`, `greedy_step` against plain torch fp32 / integer references of the same op.
Model level: `LlamaDecoder.generate` / `FalconDecoder.generate` against the CPU oracle (oracle/generate.py, pinned to the
installed transformers' `generate` by tests/test_generate_host.py) on identical bf16-rounded weights:
  * the logits of EVERY decode step (KV-cache path) against the oracle's full re-run of the emitted prefix: relative L2
    <= 3e-2 per step (bf16 forward through the layers; the training-forward logits in test_engine_gpu.py get 1.5e-2 over
    hundreds of rows, a decode step has only the B live rows);
  * every emitted token is the oracle's argmax up to the bf16 noise of the logits: oracle margin <= 0.05 (random-init
    logits have std ~0.25 and a top-1 / top-2 gap that is often < 0.002, far below bf16 rounding of the logits (~0.01), so
    token-for-token equality with an fp32 run is not a meaningful bar for a bf16 forward; a wrong position id, mask or cache
    slot gives margins of ~0.5);
  * integer bookkeeping (prompt copied through, pads after EOS, stop column, output length) is bit-exact against the
    oracle re-run on the emitted tokens;
  * the default launch mode (decode step captured once as a CUDA graph, replayed per token) emits exactly the tokens of
    the eager launch sequence.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ----------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,heads", [(32, 3), (64, 5), (128, 2)])
def test_rope_pos(cuda_dev, D, heads):
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(D)
    M, T, col0 = 37, 50, 16
    buf = torch.randn(M, col0 + heads * D + 8, generator=g).to(bf16).to(cuda_dev)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=f32) / D))
    fr = torch.outer(torch.arange(T, dtype=f32), inv)
    cos_t, sin_t = fr.cos().to(cuda_dev).contiguous(), fr.sin().to(cuda_dev).contiguous()
    pos = torch.randint(0, T, (M,), generator=g).to(cuda_dev)
    want = buf.clone()
    x = buf[:, col0:col0 + heads * D].float().view(M, heads, D)
    c, s = cos_t[pos][:, None, :], sin_t[pos][:, None, :]
    x1, x2 = x[..., :D // 2], x[..., D // 2:]
    want[:, col0:col0 + heads * D] = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).view(M, heads * D).to(bf16)
    got = ops.rope_pos_(buf.clone(), col0, heads, D, cos_t, sin_t, pos)
    # untouched columns bit-exact; rotated ones within one bf16 rounding of the fp32 reference (fma contraction may differ)
    assert torch.equal(got[:, :col0], want[:, :col0]) and torch.equal(got[:, col0 + heads * D:], want[:, col0 + heads * D:])
    assert ((got.float() - want.float()).abs() <= want.float().abs() * 2 ** -7 + 1e-6).all()      # one bf16 ulp
    assert _rel(got.float(), want.float()) < 2e-3
    # arange positions == the training kernel (position = row % L)
    L = 10
    b2 = torch.randn(3 * L, heads * D, generator=g).to(bf16).to(cuda_dev)
    a = ops.rope_(b2.clone(), 0, heads, D, cos_t[:L].contiguous(), sin_t[:L].contiguous(), L)
    p = ops.rope_pos_(b2.clone(), 0, heads, D, cos_t, sin_t, torch.arange(L, device=cuda_dev).repeat(3))
    assert ((a.float() - p.float()).abs() <= a.float().abs() * 2 ** -7 + 1e-6).all() and _rel(p.float(), a.float()) < 2e-3


@pytest.mark.parametrize("D,Hq,Hkv,T,cur", [(128, 4, 4, 40, 17), (128, 4, 2, 300, 299), (64, 7, 1, 64, 0), (64, 2, 2, 130, 128),
                                             (32, 8, 4, 33, 20), (128, 8, 8, 1024, 1000)])
def test_attention_decode(cuda_dev, D, Hq, Hkv, T, cur):
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(T + cur)
    B = 3
    Nq, Nkv = Hq * D, Hkv * D
    qkv = (torch.randn(B, Nq + 2 * Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    ck = (torch.randn(B, T, Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    cv = (torch.randn(B, T, Nkv, generator=g) * 0.8).to(bf16).to(cuda_dev)
    mask = (torch.rand(B, T, generator=g) > 0.3).to(i64).to(cuda_dev)
    mask[0, :cur] = 0                                           # a row whose only visible key is the token itself
    mask[:, cur:] = 0                                           # columns >= cur are not part of the prefix yet
    ck0, cv0 = ck.clone(), cv.clone()
    out = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck, cv, mask, cur, Hq, Hkv, D)
    # the token's K / V rows were appended at column cur, nothing else in the cache moved
    assert torch.equal(ck[:, cur], qkv[:, Nq:Nq + Nkv]) and torch.equal(cv[:, cur], qkv[:, Nq + Nkv:])
    keep = torch.ones(T, dtype=torch.bool, device=cuda_dev); keep[cur] = False
    assert torch.equal(ck[:, keep], ck0[:, keep]) and torch.equal(cv[:, keep], cv0[:, keep])
    # fp32 reference
    q = qkv[:, :Nq].float().view(B, Hq, D)
    K = ck[:, :cur + 1].float().view(B, cur + 1, Hkv, D).repeat_interleave(Hq // Hkv, dim=2)   # [B,t,Hq,D]
    V = cv[:, :cur + 1].float().view(B, cur + 1, Hkv, D).repeat_interleave(Hq // Hkv, dim=2)
    s = torch.einsum("bhd,bthd->bht", q, K) / math.sqrt(D)
    vis = mask[:, :cur + 1].bool().clone(); vis[:, cur] = True
    s = s.masked_fill(~vis[:, None, :], float("-inf"))
    ref = torch.einsum("bht,bthd->bhd", torch.softmax(s, -1), V).reshape(B, Nq)
    assert _rel(out.float(), ref) < 5e-3                        # bf16 output rounding
    assert (out.float() - ref).abs().max().item() < 2e-2
    # device-column mode (what a CUDA-graph replay uses): same launch, the column comes from an int32 [B] device tensor
    ck2, cv2 = ck0.clone(), cv0.clone()
    out2 = ops.attention_decode(qkv, 0, Nq, Nq + Nkv, ck2, cv2, mask, torch.full((B,), cur, dtype=torch.int32, device=cuda_dev),
                                Hq, Hkv, D)
    assert torch.equal(out2, out) and torch.equal(ck2, ck) and torch.equal(cv2, cv)


@pytest.mark.parametrize("M,N,K", [(16, 4096, 4096), (5, 24, 72), (1, 8, 8), (13, 1000, 1048), (16, 512, 11008), (3, 32008, 256)])
def test_decode_gemm(cuda_dev, M, N, K):
    """weight-streaming GEMM of the decode step (M <= 16 rows) vs torch fp32, every epilogue; ragged N, K tails (K % 32 != 0),
    strided operands (the LoRA-augmented activation / weight buffers have a padded row stride)"""
    from dalm_b200 import _lib, ops
    g = torch.Generator().manual_seed(M * 1000 + N + K)
    a_buf = (torch.randn(M, K + 64, generator=g) * 0.5).to(bf16).to(cuda_dev)
    w_buf = (torch.randn(N, K + 64, generator=g) * 0.5).to(bf16).to(cuda_dev)
    a, w = a_buf[:, :K], w_buf[:, :K]                                          # row stride K + 64
    ref = a.float() @ w.float().t()
    out = ops.decode_gemm(a, w)
    assert out.dtype == bf16 and _rel(out.float(), ref) < 4e-3                 # bf16 output rounding
    out32 = ops.decode_gemm(a, w, out_dtype=f32)
    assert _rel(out32, ref) < 1e-4                                             # fp32 tensor-core accumulate over up to 11 008 terms
    r32 = torch.randn(M, N, generator=g).to(cuda_dev)
    assert _rel(ops.decode_gemm(a, w, out_dtype=f32, resid=r32), ref + r32) < 1e-4
    r16 = r32.to(bf16)
    assert _rel(ops.decode_gemm(a, w, out_dtype=bf16, resid=r16).float(), ref + r16.float()) < 4e-3
    gelu = torch.nn.functional.gelu(ref)
    assert _rel(ops.decode_gemm(a, w, out_dtype=f32, act=1), gelu) < 1e-4
    # the same numbers as the wgmma GEMM the rest of the engine uses (bf16 outputs agree to rounding)
    if M == 16:
        assert _rel(ops.gemm(a, w).float(), out.float()) < 4e-3
    wide = torch.zeros(M, N + 16, dtype=f32, device=cuda_dev)                  # output into a column slice
    ops.decode_gemm(a, w, out=wide[:, 8:8 + N])
    assert _rel(wide[:, 8:8 + N], ref) < 1e-4 and (wide[:, :8] == 0).all() and (wide[:, 8 + N:] == 0).all()
    with pytest.raises(_lib.DalmB200Error):
        ops.decode_gemm(torch.zeros(17, K, dtype=bf16, device=cuda_dev), w)   # more than one 16-row tile: use ops.gemm


def test_greedy_step(cuda_dev):
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, V, Vp, T = 6, 1000, 1008, 12
    logits = torch.randn(B, Vp, generator=g).to(bf16).to(cuda_dev)
    logits[:, V:] = 100.0                                       # padded vocabulary columns must never win
    logits[0, 700] = 50.0; logits[0, 123] = 50.0                # tie -> lowest index
    logits[1, 999] = 60.0                                       # last valid column
    logits[2, 5] = 60.0                                         # emits an EOS id this step
    logits[4, 0] = 60.0                                         # first column
    logits[5, 333] = 60.0
    eos = torch.tensor([5, 9], device=cuda_dev)
    unfinished = torch.tensor([1, 1, 1, 0, 1, 1], dtype=torch.int32, device=cuda_dev)     # row 3 finished earlier
    tokens = torch.full((B, T), -1, dtype=i64, device=cuda_dev)
    mask = torch.zeros(B, T, dtype=i64, device=cuda_dev)
    next_ids = torch.zeros(B, dtype=i64, device=cuda_dev)
    pos = torch.arange(B, dtype=i64, device=cuda_dev) * 3
    alive = torch.zeros(T, dtype=torch.int32, device=cuda_dev)
    col = 7
    ops.greedy_step_(logits, V, eos, 77, unfinished, tokens, mask, col, next_ids, pos, alive)
    want = torch.tensor([123, 999, 5, 77, 0, 333], device=cuda_dev)          # row 0: lowest index of the tie; row 3: pad
    assert torch.equal(tokens[:, col], want) and torch.equal(next_ids, want)
    assert (tokens[:, :col] == -1).all() and (tokens[:, col + 1:] == -1).all()
    assert torch.equal(mask[:, col], torch.ones(B, dtype=i64, device=cuda_dev)) and int(mask.sum()) == B
    assert torch.equal(pos, torch.arange(B, dtype=i64, device=cuda_dev) * 3 + 1)
    assert unfinished.tolist() == [1, 1, 0, 0, 1, 1]
    assert alive.tolist() == [0] * col + [4] + [0] * (T - col - 1)
    # no EOS list: nobody finishes; small vocabulary (V < 256 threads)
    small = torch.randn(2, 40, generator=g).to(bf16).to(cuda_dev)
    small[0, 17] = 9.0; small[1, 32] = 9.0; small[:, 33:] = 50.0
    unf2 = torch.ones(2, dtype=torch.int32, device=cuda_dev)
    t2, m2 = torch.zeros(2, 3, dtype=i64, device=cuda_dev), torch.zeros(2, 3, dtype=i64, device=cuda_dev)
    n2, p2, a2 = torch.zeros(2, dtype=i64, device=cuda_dev), torch.zeros(2, dtype=i64, device=cuda_dev), torch.zeros(3, dtype=torch.int32, device=cuda_dev)
    ops.greedy_step_(small, 33, None, 0, unf2, t2, m2, 1, n2, p2, a2)
    assert n2.tolist() == [17, 32] and t2[:, 1].tolist() == [17, 32] and a2.tolist() == [0, 2, 0] and unf2.tolist() == [1, 1]
    # device-column mode: each row's own counter names the column (current + 1) and advances; past the end it is a no-op
    cur = torch.tensor([1, 0], dtype=torch.int32, device=cuda_dev)
    ops.greedy_step_(small, 33, None, 0, unf2, t2, m2, cur, n2, p2, a2)
    assert cur.tolist() == [2, 1] and t2.tolist() == [[0, 17, 17], [0, 32, 0]] and a2.tolist() == [0, 3, 1] and p2.tolist() == [2, 2]
    ops.greedy_step_(small, 33, None, 0, unf2, t2, m2, cur, n2, p2, a2)
    assert cur.tolist() == [2, 2] and t2.tolist() == [[0, 17, 17], [0, 32, 32]] and a2.tolist() == [0, 3, 2] and p2.tolist() == [2, 3]


# ----------------------------------------------------------------------------------------------------------------
# whole decoders
# ----------------------------------------------------------------------------------------------------------------
def _prompt(B, L0, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, V, (B, L0), generator=g)
    mask = torch.ones(B, L0, dtype=i64)
    mask[1, :3] = 0          # left padding
    mask[2, L0 - 3:] = 0     # right padding
    return ids, mask


def _check_against_oracle(dec, ref, ids, mask, T, eos, pad, monkeypatch):
    """runs dec.generate with every step's logits recorded, then replays the emitted tokens through the oracle"""
    from dalm_b200 import ops
    from oracle import generate as og
    rec = []
    real = ops.greedy_step_

    def recording(logits, V, *a, **k):
        rec.append(logits[:, :V].float().cpu())
        return real(logits, V, *a, **k)

    from dalm_b200.engine import decoding
    eos_list = [] if eos is None else list(eos)
    gen = lambda: dec.generate(input_ids=ids.to(dec.dev), attention_mask=mask.to(dec.dev), max_length=T, early_stopping=True,
                               eos_token_id=eos_list, pad_token_id=pad).cpu()       # [] = no EOS (None would mean the config's)
    # pass 1: eager launches with every step's logits recorded (the recorder reads them back, which a graph capture cannot)
    monkeypatch.setenv("DALM_B200_DECODE_GRAPH", "0")
    monkeypatch.setattr(ops, "greedy_step_", recording)
    out = gen()
    monkeypatch.setattr(ops, "greedy_step_", real)
    assert decoding.LAST_RUN["graph_replays"] == 0
    # pass 2: the default launch mode — the decode step captured once as a CUDA graph and replayed; same kernels, same
    # arguments, so the tokens must be IDENTICAL to the eager pass
    monkeypatch.setenv("DALM_B200_DECODE_GRAPH", "1")
    replayed = gen()
    assert decoding.LAST_RUN["graph_replays"] >= min(4, out.shape[1] - ids.shape[1] - 2), decoding.LAST_RUN
    assert torch.equal(replayed, out)
    B, L0 = ids.shape
    assert out.dtype == i64 and out.shape[0] == B and L0 < out.shape[1] <= T
    assert torch.equal(out[:, :L0], ids)                                    # prompt passes through untouched
    n_new = out.shape[1] - L0
    assert len(rec) >= n_new
    # oracle logits for every generated column, teacher-forced on OUR tokens (full re-run of the prefix, no cache)
    am = torch.cat([mask, torch.ones(B, n_new, dtype=i64)], 1)
    pos = (am.cumsum(-1) - 1).masked_fill(am == 0, 1)
    with torch.no_grad():
        want = ref(input_ids=out, attention_mask=am, position_ids=pos).logits.float()
    finished = torch.zeros(B, dtype=torch.bool)
    worst_rel, worst_margin = 0.0, 0.0
    for j in range(n_new):
        col = L0 + j
        live = ~finished
        w, g = want[:, col - 1], rec[j]
        if live.any():
            worst_rel = max(worst_rel, _rel(g[live], w[live]))
            margin = w.max(-1).values - w.gather(1, out[:, col:col + 1]).squeeze(1)
            worst_margin = max(worst_margin, float(margin[live].max()))
        assert (out[finished, col] == pad).all()                             # finished rows emit the pad id
        for e in eos_list:
            finished |= live & (out[:, col] == e)
    assert worst_rel < 3e-2, worst_rel
    assert worst_margin < 0.05, worst_margin
    if eos_list and out.shape[1] < T:
        assert finished.all()                                                # stopped early only because every row hit EOS
        # ... and not a step later than HF would: before the last column someone was still generating
        f2 = torch.zeros(B, dtype=torch.bool)
        for col in range(L0, out.shape[1] - 1):
            for e in eos_list:
                f2 |= out[:, col] == e
        assert not f2.all()
    # the oracle generating from the same prompt: identical wherever its own top-1 / top-2 gap exceeds the bf16 noise
    mine = og.greedy_generate(ref, ids, mask, T, eos_token_ids=eos_list, pad_token_id=pad)
    return out, mine


@pytest.mark.parametrize("name,lora,rows_gemm", [("llama-tiny", True, "1"), ("llama-hd128", False, "1"), ("llama-hd128", True, "0")])
def test_llama_generate(cuda_dev, monkeypatch, name, lora, rows_gemm):
    monkeypatch.setenv("DALM_B200_DECODE_GEMM", rows_gemm)                    # "0": decode-step GEMMs on the training tcgen05 kernel
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 512
    cfg = synthetic.llama_config(name, vocab_size=V)
    sd = params.random_state_dict("llama", cfg, seed=2)
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = om.build_llama(cfg, sd)
    if lora:
        g = torch.Generator().manual_seed(9)
        for n, _, _ in dec.lora.specs:
            dec.lora.B[n].copy_((torch.randn(dec.lora.B[n].shape, generator=g) * 0.02).to(cuda_dev))
        dec.repack_lora()
        om.attach_lora(ref, {n: {"A": dec.lora.A[n].cpu(), "B": dec.lora.B[n].cpu()} for n, _, _ in dec.lora.specs})
        dec.train()                                                          # generate must not apply adapter dropout
    ids, mask = _prompt(4, 12, V, seed=1)
    T = 34
    free, _ = _check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert free.shape == (4, T)
    assert dec.training == bool(lora)
    # EOS ids taken from the free run so that rows finish at different steps (and all of them before max_length)
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    out, _ = _check_against_oracle(dec, ref, ids, mask, T, eos, eos[0], monkeypatch)
    assert out.shape[1] <= 25
    with pytest.raises(ValueError):
        dec.generate(input_ids=ids.to(cuda_dev), attention_mask=mask.to(cuda_dev), max_length=12)


def test_falcon_generate(cuda_dev, monkeypatch):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.falcon import FalconDecoder
    from oracle import models as om
    V = 512
    cfg = synthetic.falcon_config("falcon-mini", vocab_size=V)               # 7 query heads x 64, one KV head
    sd = params.random_state_dict("falcon", cfg, seed=3)
    sd = {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}
    dec = FalconDecoder(cfg, sd, device=cuda_dev)
    ref = om.build_falcon(cfg, sd)
    ids, mask = _prompt(4, 12, V, seed=2)
    free, _ = _check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert free.shape == (4, 30)
    eos = sorted({int(free[0, 15]), int(free[1, 18]), int(free[2, 13]), int(free[3, 21])})
    _check_against_oracle(dec, ref, ids, mask, 30, eos, eos[0], monkeypatch)
