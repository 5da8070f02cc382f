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

from model_helpers import attach_lora, check_against_oracle, draw_lora_B, prompt, r16_2d, rel

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64


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
    assert rel(got.float(), want.float()) < 2e-3
    # arange positions == the training kernel (position = row % L)
    L = 10
    b2 = torch.randn(3 * L, heads * D, generator=g).to(bf16).to(cuda_dev)
    a = ops.rope_(b2.clone(), 0, heads, D, cos_t[:L].contiguous(), sin_t[:L].contiguous(), L)
    p = ops.rope_pos_(b2.clone(), 0, heads, D, cos_t, sin_t, torch.arange(L, device=cuda_dev).repeat(3))
    assert ((a.float() - p.float()).abs() <= a.float().abs() * 2 ** -7 + 1e-6).all() and rel(p.float(), a.float()) < 2e-3


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
    assert rel(out.float(), ref) < 5e-3                        # bf16 output rounding
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
    assert out.dtype == bf16 and rel(out.float(), ref) < 4e-3                 # bf16 output rounding
    out32 = ops.decode_gemm(a, w, out_dtype=f32)
    assert rel(out32, ref) < 1e-4                                             # fp32 tensor-core accumulate over up to 11 008 terms
    r32 = torch.randn(M, N, generator=g).to(cuda_dev)
    assert rel(ops.decode_gemm(a, w, out_dtype=f32, resid=r32), ref + r32) < 1e-4
    r16 = r32.to(bf16)
    assert rel(ops.decode_gemm(a, w, out_dtype=bf16, resid=r16).float(), ref + r16.float()) < 4e-3
    gelu = torch.nn.functional.gelu(ref)
    assert rel(ops.decode_gemm(a, w, out_dtype=f32, act=1), gelu) < 1e-4
    # the same numbers as the wgmma GEMM the rest of the engine uses (bf16 outputs agree to rounding)
    if M == 16:
        assert rel(ops.gemm(a, w).float(), out.float()) < 4e-3
    wide = torch.zeros(M, N + 16, dtype=f32, device=cuda_dev)                  # output into a column slice
    ops.decode_gemm(a, w, out=wide[:, 8:8 + N])
    assert rel(wide[:, 8:8 + N], ref) < 1e-4 and (wide[:, :8] == 0).all() and (wide[:, 8 + N:] == 0).all()
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
@pytest.mark.parametrize("name,lora,rows_gemm", [("llama-tiny", True, "1"), ("llama-hd128", False, "1"), ("llama-hd128", True, "0")])
def test_llama_generate(cuda_dev, monkeypatch, name, lora, rows_gemm):
    monkeypatch.setenv("DALM_B200_DECODE_GEMM", rows_gemm)                    # "0": decode-step GEMMs on the training tcgen05 kernel
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from oracle import models as om
    V = 512
    cfg = synthetic.llama_config(name, vocab_size=V)
    sd = r16_2d(params.random_state_dict("llama", cfg, seed=2))
    dec = LlamaDecoder(cfg, sd, device=cuda_dev, lora=lora)
    ref = om.build_llama(cfg, sd)
    if lora:
        draw_lora_B(dec, torch.Generator().manual_seed(9))
        attach_lora(ref, dec)
        dec.train()                                                          # generate must not apply adapter dropout
    ids, mask = prompt(4, 12, V, seed=1)
    T = 34
    free, _ = check_against_oracle(dec, ref, ids, mask, T, None, 0, monkeypatch)
    assert free.shape == (4, T)
    assert dec.training == bool(lora)
    # EOS ids taken from the free run so that rows finish at different steps (and all of them before max_length)
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    out, _ = check_against_oracle(dec, ref, ids, mask, T, eos, eos[0], monkeypatch)
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
    sd = r16_2d(params.random_state_dict("falcon", cfg, seed=3))
    dec = FalconDecoder(cfg, sd, device=cuda_dev)
    ref = om.build_falcon(cfg, sd)
    ids, mask = prompt(4, 12, V, seed=2)
    free, _ = check_against_oracle(dec, ref, ids, mask, 30, None, 0, monkeypatch)
    assert free.shape == (4, 30)
    eos = sorted({int(free[0, 15]), int(free[1, 18]), int(free[2, 13]), int(free[3, 21])})
    check_against_oracle(dec, ref, ids, mask, 30, eos, eos[0], monkeypatch)
