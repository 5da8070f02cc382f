"""Greedy autoregressive decoding with a KV cache — the generator half of `dalm eval-rag`.

The reference calls HF `model.generate(**inputs, max_length=max_length, early_stopping=True)` on the generator
(dalm/eval/eval_rag.py:126-140) and scores exact match on the decoded text (:268-277). This is that call's greedy-search
semantics (transformers GenerationMixin._sample with do_sample=False) as a launch sequence over the C-ABI kernels:

  prefill   the decoder's ordinary forward over the padded prompt with position ids cumsum(attention_mask) - 1
            (what HF generate feeds the model — NOT arange: left / right padded rows rotate differently), rotated K / V of
            every layer copied into a bf16 cache [B, max_length, kv width]; only the last column goes through the LM head
  step      one token per sequence: norm -> QKV GEMM -> RoPE at the token's position -> `attention_decode` (appends the
            token's K / V, attends over the cache) -> output projection -> MLP -> LM head -> `greedy_step` (argmax, pad
            after EOS, next position id, next column), all state on the device, so the launch sequence has the same
            arguments for every token and CAN be captured once as a CUDA graph and replayed (292 launches per token at
            Llama-2-7B). Capture has a fixed cost of 50-300 ms per `generate` call, so it is used for long generations only
            (GRAPH_MIN_STEPS; DALM_B200_DECODE_GRAPH = 1 / 0 forces it on / off); the host reads one "anyone still
            generating" counter every 8 tokens

A decoder takes part by providing `_prefill_last`, `_decode_step`, `kv_columns`, `_rope`, `lm_head`, `V`, `cfg`, `dev`.
"""
from __future__ import annotations

import logging
import os
from typing import Optional

import torch

from .. import ops

bf16 = torch.bfloat16
logger = logging.getLogger(__name__)
LAST_RUN = {"graph_replays": 0, "eager_steps": 0}          # how the decode steps of the most recent call were launched
MAX_CACHE_TOKENS = 8192                                     # dalm_b200_attention_decode: T <= 8192
GRAPH_MIN_STEPS = 192                                       # remaining tokens from which capturing the step pays for itself


_LEAN_POOL = None


def _capture_lean(graph: "torch.cuda.CUDAGraph", step) -> None:
    """CANDIDATE (DALM_B200_DECODE_GRAPH=2, not a default): capture without `torch.cuda.graph`'s entry work (gc.collect +
    empty_cache, measured at 50-300 ms per call) and into ONE memory pool shared by every capture of the process, so that
    later `generate` calls find their decode-step buffers already cached. Written after the round's GPU minutes were spent:
    its check (tests/test_generate_gpu.py, DALM_B200_EXPERIMENTAL=1) has not run yet."""
    global _LEAN_POOL
    if _LEAN_POOL is None:
        _LEAN_POOL = torch.cuda.graph_pool_handle()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        graph.capture_begin(pool=_LEAN_POOL)
        try:
            step()
        finally:
            graph.capture_end()
    torch.cuda.current_stream().wait_stream(side)


@torch.no_grad()
def greedy_generate(dec, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                    max_length: Optional[int] = None, max_new_tokens: Optional[int] = None, eos_token_id=None,
                    pad_token_id: Optional[int] = None, do_sample: bool = False, num_beams: int = 1, **unused) -> torch.Tensor:
    """Returns int64 [B, <= max_length] on the decoder's device, prompt included (HF layout). Position ids =
    cumsum(attention_mask) - 1; finished rows emit pad_token_id (default: the first EOS id); generation stops right after
    the step in which the last row emitted EOS, or at max_length TOTAL tokens. `early_stopping` (beam search only) and
    other HF flags are accepted and ignored; sampling / beam search (a checkpoint's generation_config may ask for them) are
    not built."""
    if do_sample or num_beams != 1:
        raise NotImplementedError("dalm_b200 generate: greedy search only (do_sample=False, num_beams=1)")
    if input_ids is None:
        raise ValueError("generate: input_ids is required")
    dev = dec.dev
    ids = input_ids.to(dev, torch.int64).contiguous()
    B, L0 = ids.shape
    mask = (torch.ones_like(ids) if attention_mask is None else attention_mask.to(dev, torch.int64)).contiguous()
    if max_new_tokens is not None:
        total = L0 + int(max_new_tokens)
    else:
        total = int(max_length) if max_length is not None else int(dec.cfg.get("max_length", 20))       # HF default: 20
    if L0 >= total:
        raise ValueError(f"Input length of input_ids is {L0}, but `max_length` is set to {total}. This can lead to unexpected "
                         "behavior. You should consider increasing `max_length` or, better yet, setting `max_new_tokens`.")
    if total > MAX_CACHE_TOKENS:
        raise NotImplementedError(f"generate: max_length {total} exceeds the decode attention kernel's cache limit of "
                                  f"{MAX_CACHE_TOKENS} tokens (its score row lives in shared memory)")
    eos = dec.cfg.get("eos_token_id") if eos_token_id is None else eos_token_id
    eos_list = [] if eos is None else ([int(e) for e in eos] if isinstance(eos, (list, tuple)) else [int(eos)])
    pad = pad_token_id if pad_token_id is not None else dec.cfg.get("pad_token_id")
    if pad is None:
        if not eos_list:
            raise ValueError("generate: need pad_token_id or eos_token_id to fill finished rows")
        pad = eos_list[0]                                                         # HF: "Setting pad_token_id to eos_token_id"
    eos_t = torch.tensor(eos_list, dtype=torch.int64, device=dev) if eos_list else None
    was_training = dec.training
    dec.eval()                                                                    # no adapter-input dropout while decoding
    try:
        tokens = torch.full((B, total), int(pad), dtype=torch.int64, device=dev)
        tokens[:, :L0] = ids
        kmask = torch.zeros(B, total, dtype=torch.int64, device=dev)
        kmask[:, :L0] = mask
        pos_prompt = (mask.cumsum(-1) - 1).masked_fill_(mask == 0, 1).reshape(-1).contiguous()
        tables = dec._rope(total)
        k0, v0, width = dec.kv_columns()
        caches = [(torch.empty(B, total, width, dtype=bf16, device=dev), torch.empty(B, total, width, dtype=bf16, device=dev))
                  for _ in dec.layers]

        def sink(li: int, qkv: torch.Tensor) -> None:                            # rotated K | V of the prompt -> cache
            caches[li][0][:, :L0].copy_(qkv[:, k0:k0 + width].view(B, L0, width))
            caches[li][1][:, :L0].copy_(qkv[:, v0:v0 + width].view(B, L0, width))

        last = dec._prefill_last(ids, mask, pos_prompt, tables, sink)             # bf16 [B,H]
        logits = ops.gemm_rows(last, dec.lm_head)                                 # bf16 [B, Vp]
        unfinished = torch.ones(B, dtype=torch.int32, device=dev)
        next_ids = torch.zeros(B, dtype=torch.int64, device=dev)
        pos = (mask.sum(-1) - 1).contiguous()                                     # position id of the last prompt token
        alive = torch.zeros(total, dtype=torch.int32, device=dev)
        col = L0
        ops.greedy_step_(logits, dec.V, eos_t, pad, unfinished, tokens, kmask, col, next_ids, pos, alive)
        col += 1
        # every remaining step is the same launch sequence: in device-column mode (cur_row holds each row's current column,
        # advanced by greedy_step) its arguments never change, so it is captured ONCE as a CUDA graph and replayed
        cur_row = torch.full((B,), L0, dtype=torch.int32, device=dev)           # column of the token in next_ids

        def step() -> None:
            lg = dec._decode_step(next_ids, pos, caches, kmask, cur_row, tables)
            ops.greedy_step_(lg, dec.V, eos_t, pad, unfinished, tokens, kmask, cur_row, next_ids, pos, alive)

        graph, replays, eager = None, 0, 0
        # A `torch.cuda.graph` capture is expensive per call (its entry runs gc.collect + empty_cache, the private pool is
        # allocated afresh) and a replayed step saves only launch overhead while the step is GPU-bound (decode attention), so
        # by default only long generations are captured. DALM_B200_DECODE_GRAPH=1 / 0 forces it.
        mode = os.environ.get("DALM_B200_DECODE_GRAPH", "auto")
        lean_capture = mode == "2"                                                # candidate, see _capture_lean
        use_graph = dev.type == "cuda" and ((mode in ("1", "2") and total - col >= 4) or (mode == "auto" and total - col >= GRAPH_MIN_STEPS))
        while col < total:
            if eos_list and (col - L0) % 8 == 0 and int(alive[col - 1].item()) == 0:    # one host read every 8 tokens
                break
            if use_graph and graph is None and col > L0 + 1:                     # one eager step first (lazy attributes, tensor maps)
                try:
                    graph = torch.cuda.CUDAGraph()
                    if lean_capture:
                        _capture_lean(graph, step)
                    else:
                        with torch.cuda.graph(graph):
                            step()
                except Exception as e:                                            # capture is an optimisation, never a requirement
                    logger.warning(f"CUDA-graph capture of the decode step failed ({type(e).__name__}: {e}); launching eagerly")
                    graph, use_graph = None, False
            if graph is not None:
                graph.replay()
                replays += 1
            else:
                step()
                eager += 1
            col += 1
        LAST_RUN.update(graph_replays=replays, eager_steps=eager)
        end = col
        if eos_list:                                                              # HF stops right after the step that finished the last row
            a = alive[L0:col].tolist()
            end = L0 + next((i + 1 for i, n in enumerate(a) if n == 0), len(a))
        return tokens[:, :end]
    finally:
        dec.train(was_training)
