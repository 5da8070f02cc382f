"""Autoregressive decoding with a KV cache — the generator half of `dalm eval-rag`.

The reference calls HF `model.generate(**inputs, max_length=max_length, early_stopping=True)` on the generator
(dalm/eval/eval_rag.py:126-140) and scores exact match on the decoded text (:268-277). `generate` below resolves what that
call does for the checkpoint the way HF does (generation_config.json, else config.json; call kwargs; global defaults):
greedy search (transformers GenerationMixin._sample with do_sample=False), or sampling with HF's temperature -> top-k ->
top-p warpers when the generation config asks for it (Llama-2's does: do_sample, temperature 0.6, top-p 0.9, top-k 50 by
default). Both run as one launch sequence over the C-ABI kernels:

  prefill   the decoder's ordinary forward over the padded prompt with position ids cumsum(attention_mask) - 1
            (what HF generate feeds the model — NOT arange: left / right padded rows rotate differently), rotated K / V of
            every layer copied into a bf16 cache [B, max_length, kv width]; only the last column goes through the LM head
  step      one token per sequence: norm -> QKV GEMM -> RoPE at the token's position -> `attention_decode` (appends the
            token's K / V, attends over the cache) -> output projection -> MLP -> LM head -> `greedy_step` (argmax) or
            `sample_step` (warpers + draw), each with the same bookkeeping (pad after EOS, next position id, next column),
            all state on the device, so the launch sequence has the same
            arguments for every token and CAN be captured once as a CUDA graph and replayed (292 launches per token at
            Llama-2-7B). Capture has a fixed cost of 50-300 ms per `generate` call, so it is used for long generations only
            (GRAPH_MIN_STEPS; DALM_B200_DECODE_GRAPH = 1 / 0 forces it on / off); the host reads one "anyone still
            generating" counter every 8 tokens

A decoder takes part by providing `_prefill_last`, `_decode_step`, `kv_columns`, `_rope`, `lm_head`, `V`, `cfg`, `dev`.
"""
from __future__ import annotations

import functools
import json
import logging
import math
import os
from typing import Optional

import torch

from .. import ops

bf16 = torch.bfloat16
logger = logging.getLogger(__name__)
LAST_RUN = {"graph_replays": 0, "eager_steps": 0}          # how the decode steps of the most recent call were launched
MAX_CACHE_TOKENS = 8192                                     # dalm_b200_attention_decode: T <= 8192
GRAPH_MIN_STEPS = 192                                       # remaining tokens from which capturing the step pays for itself


# ----------------------------------------------------------------------------------------------------------------
# generation config: what HF `generate` would do for the same checkpoint and call
# ----------------------------------------------------------------------------------------------------------------
GEN_FIELDS = ("do_sample", "num_beams", "temperature", "top_k", "top_p", "max_length", "eos_token_id", "pad_token_id")
GLOBAL_DEFAULTS = {"do_sample": False, "num_beams": 1, "temperature": 1.0, "top_k": 50, "top_p": 1.0, "max_length": 20}
# processors that would change the sampling distribution and are not built, with the value that leaves them off
NOT_BUILT = {"min_p": None, "typical_p": 1.0, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0, "top_h": None, "repetition_penalty": 1.0,
             "no_repeat_ngram_size": 0, "bad_words_ids": None, "suppress_tokens": None, "min_new_tokens": None,
             "renormalize_logits": False}


def load_generation_config(path: str) -> Optional[dict]:
    """<model dir>/generation_config.json, or None when the directory has none"""
    f = os.path.join(path, "generation_config.json")
    if not path or not os.path.isfile(f):
        return None
    with open(f) as fh:
        return json.load(fh)


def resolve_generation_config(cfg: dict, gen_cfg: Optional[dict], kwargs: dict) -> dict:
    """The effective settings of a `generate` call, resolved like HF's `_prepare_generation_config`: the checkpoint's
    generation_config.json when there is one, else the generation fields of config.json; then the call's kwargs; then
    transformers' global defaults for whatever is still unset. A kwarg passed as None counts as unset, as it always has for
    eos_token_id / pad_token_id here."""
    base = gen_cfg if gen_cfg is not None else cfg
    out = {k: base.get(k) for k in GEN_FIELDS + tuple(NOT_BUILT)}
    out.update({k: v for k, v in kwargs.items() if k in out and v is not None})
    for k, v in GLOBAL_DEFAULTS.items():
        if out[k] is None:
            out[k] = v
    if kwargs.get("max_new_tokens") is not None:
        out["max_new_tokens"] = kwargs["max_new_tokens"]
    return out


def _unbuilt_fields(res: dict) -> list:
    off = lambda k, v: v is None or v == NOT_BUILT[k] or (k in ("min_new_tokens", "renormalize_logits") and not v)
    return [k for k in NOT_BUILT if not off(k, res.get(k))]


def describe(res: dict) -> str:
    """one line naming the decoding a resolved config selects"""
    if not res["do_sample"]:
        return "greedy search (do_sample=False)"
    return f"sampling (temperature {res['temperature']}, top-k {res['top_k']}, top-p {res['top_p']})"


def decoding_mode(dec, **kwargs) -> str:
    """how `dec.generate(**kwargs)` decodes, as one line (eval-rag logs it)"""
    return describe(resolve_generation_config(dec.cfg, getattr(dec, "generation_config", None), kwargs))


def generate(dec, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
    """HF `generate` for a decoder: resolves the generation config (checkpoint file, call kwargs, global defaults) and
    dispatches to greedy search or sampling. Beam search and the sampling processors in NOT_BUILT raise."""
    gen_cfg = getattr(dec, "generation_config", None)
    res = resolve_generation_config(dec.cfg, gen_cfg, kw)
    if int(res["num_beams"]) > 1:
        raise NotImplementedError(f"dalm_b200 generate: beam search (num_beams={res['num_beams']}) is not built")
    rest = {k: v for k, v in kw.items() if k not in ("do_sample", "num_beams", "temperature", "top_k", "top_p")}
    if gen_cfg is not None:                        # the checkpoint's file decides what the call leaves open
        rest.update(eos_token_id=res["eos_token_id"], pad_token_id=res["pad_token_id"], max_length=res["max_length"])
    if not res["do_sample"]:
        return greedy_generate(dec, input_ids, attention_mask, **rest)
    bad = _unbuilt_fields(res)
    if bad:
        raise NotImplementedError(f"dalm_b200 generate: sampling with {', '.join(f'{k}={res[k]!r}' for k in bad)} is not built")
    return sample_generate(dec, input_ids, attention_mask, temperature=res["temperature"], top_k=res["top_k"],
                           top_p=res["top_p"], **rest)


@torch.no_grad()
def greedy_generate(dec, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                    max_length: Optional[int] = None, max_new_tokens: Optional[int] = None, eos_token_id=None,
                    pad_token_id: Optional[int] = None, do_sample: bool = False, num_beams: int = 1, **unused) -> torch.Tensor:
    """Returns int64 [B, <= max_length] on the decoder's device, prompt included (HF layout). Position ids =
    cumsum(attention_mask) - 1; finished rows emit pad_token_id (default: the first EOS id); generation stops right after
    the step in which the last row emitted EOS, or at max_length TOTAL tokens. `early_stopping` (beam search only) and
    other HF flags are accepted and ignored. Greedy search only: sampling is `sample_generate`, beam search is not built."""
    if do_sample or num_beams != 1:
        raise NotImplementedError("dalm_b200 generate: greedy search only (do_sample=False, num_beams=1)")
    return _decode(dec, ops.greedy_step_, input_ids, attention_mask, max_length, max_new_tokens, eos_token_id,
                   pad_token_id)


@torch.no_grad()
def sample_generate(dec, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                    max_length: Optional[int] = None, max_new_tokens: Optional[int] = None, eos_token_id=None,
                    pad_token_id: Optional[int] = None, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0,
                    **unused) -> torch.Tensor:
    """HF `_sample` with do_sample=True: every token is drawn from softmax(logits / temperature) restricted by top-k
    (0 = off) and then top-p (1 = off), in the order and with the tie rules of HF's warpers (`sample_step`). Everything
    else (prompt, stop rule, padding after EOS, output layout) is greedy_generate's.
    The call's seed is one 63-bit draw from torch's default CPU generator, so `torch.manual_seed(s)` makes a call
    reproducible, and eager launches and CUDA-graph replays emit the same tokens. The stream of tokens is NOT HF's for the
    same seed (a different generator draws the uniforms); the distribution each token is drawn from is the same."""
    temperature, top_k, top_p = float(temperature), int(top_k), float(top_p)
    if not (temperature > 0.0 and math.isfinite(temperature)):
        raise ValueError(f"`temperature` (={temperature}) has to be a strictly positive float")
    if top_k < 0:
        raise ValueError(f"`top_k` has to be a non-negative integer, but is {top_k}")
    if not 0.0 < top_p <= 1.0:
        raise ValueError(f"`top_p` has to be a float in (0, 1], but is {top_p}")
    seed = int(torch.randint(0, 2 ** 63 - 1, (1,)).item())
    step = functools.partial(ops.sample_step_, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed)
    return _decode(dec, step, input_ids, attention_mask, max_length, max_new_tokens, eos_token_id, pad_token_id)


def _decode(dec, token_step, input_ids, attention_mask, max_length, max_new_tokens, eos_token_id, pad_token_id) -> torch.Tensor:
    """the decode loop shared by greedy search and sampling: prefill, KV cache, per-token step (captured as a CUDA graph
    for long generations), stop rule. `token_step` chooses each token and keeps the bookkeeping (ops.greedy_step_'s
    signature)."""
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
        token_step(logits, dec.V, eos_t, pad, unfinished, tokens, kmask, col, next_ids, pos, alive)
        col += 1
        # every remaining step is the same launch sequence: in device-column mode (cur_row holds each row's current column,
        # advanced by the token step) its arguments never change, so it is captured ONCE as a CUDA graph and replayed
        cur_row = torch.full((B,), L0, dtype=torch.int32, device=dev)           # column of the token in next_ids

        def step() -> None:
            lg = dec._decode_step(next_ids, pos, caches, kmask, cur_row, tables)
            token_step(lg, dec.V, eos_t, pad, unfinished, tokens, kmask, cur_row, next_ids, pos, alive)

        graph, replays, eager = None, 0, 0
        # A `torch.cuda.graph` capture is expensive per call (its entry runs gc.collect + empty_cache, the private pool is
        # allocated afresh) and a replayed step saves only launch overhead while the step is GPU-bound (decode attention), so
        # by default only long generations are captured. DALM_B200_DECODE_GRAPH=1 / 0 forces it.
        mode = os.environ.get("DALM_B200_DECODE_GRAPH", "auto")
        use_graph = dev.type == "cuda" and ((mode == "1" and total - col >= 4) or (mode == "auto" and total - col >= GRAPH_MIN_STEPS))
        while col < total:
            if eos_list and (col - L0) % 8 == 0 and int(alive[col - 1].item()) == 0:    # one host read every 8 tokens
                break
            if use_graph and graph is None and col > L0 + 1:                     # one eager step first (lazy attributes, tensor maps)
                try:
                    graph = torch.cuda.CUDAGraph()
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
