"""Offline fixtures: synthetic (Abstract, Question, Answer) data, tokenizers and random-init model directories.

There is no network in the build / GPU environment, so pretrained checkpoints and tokenizers of bge-* / Llama-2 /
Falcon cannot be fetched. This module writes HF-layout directories (config.json + tokenizer files [+ safetensors])
with the PUBLIC architecture shapes (SURVEY §8 model table) so that the drop-in wrappers can be pointed at them exactly
like at a hub name. Weights are seeded random-init (std 0.02), as BASELINE.json's configs prescribe.
"""
from __future__ import annotations

import csv
import json
import os
from typing import Dict, List, Optional

import numpy as np

# ---------------------------------------------------------------------------------------------------------------
# architecture shapes
# ---------------------------------------------------------------------------------------------------------------
BERT_SHAPES: Dict[str, Dict] = {
    "bge-tiny": dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=2, intermediate_size=128),
    "bge-small-en": dict(hidden_size=384, num_hidden_layers=12, num_attention_heads=12, intermediate_size=1536),
    "bge-large-en": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096),
}
LLAMA_SHAPES: Dict[str, Dict] = {
    "llama-tiny": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=2,
                       intermediate_size=256),
    "llama-hd128": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=2,
                        intermediate_size=512),
    "llama-mini": dict(hidden_size=512, num_hidden_layers=4, num_attention_heads=4, num_key_value_heads=4,
                       intermediate_size=1408),
    "Llama-2-7b-hf": dict(hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=32,
                          intermediate_size=11008),
}


# Llama 3.x (model_type "llama", GQA, rope_theta 5e5, llama3 RoPE frequency scaling). The tiny shapes use an
# original_max_position_embeddings of 64 so that every band of the llama3 rule occurs at their head_dim: the short wavelengths
# (kept), the long ones (divided by factor) and the band between (blended)
LLAMA3_SHAPES: Dict[str, Dict] = {
    "llama3-tiny": dict(hidden_size=512, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=128,
                        intermediate_size=1024, tie_word_embeddings=False,                # 6 q|k heads x 128: RoPE in the QKV epilogue
                        rope_scaling=dict(factor=8.0, original_max_position_embeddings=64)),
    "llama3.2-tiny": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                          intermediate_size=512, tie_word_embeddings=True,                 # head_dim 64: the RoPE row kernel
                          rope_scaling=dict(factor=32.0, original_max_position_embeddings=64)),
    # published meta-llama config.json values (written from the model cards; not re-fetched offline)
    "llama-3.1-8b": dict(hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
                         intermediate_size=14336, tie_word_embeddings=False,
                         rope_scaling=dict(factor=8.0, original_max_position_embeddings=8192)),
    "llama-3.2-1b": dict(hidden_size=2048, num_hidden_layers=16, num_attention_heads=32, num_key_value_heads=8, head_dim=64,
                         intermediate_size=8192, tie_word_embeddings=True,
                         rope_scaling=dict(factor=32.0, original_max_position_embeddings=8192)),
    "llama-3.2-3b": dict(hidden_size=3072, num_hidden_layers=28, num_attention_heads=24, num_key_value_heads=8, head_dim=128,
                         intermediate_size=8192, tie_word_embeddings=True,
                         rope_scaling=dict(factor=32.0, original_max_position_embeddings=8192)),
    "llama-3.3-70b": dict(hidden_size=8192, num_hidden_layers=80, num_attention_heads=64, num_key_value_heads=8, head_dim=128,
                          intermediate_size=28672, tie_word_embeddings=False,
                          rope_scaling=dict(factor=8.0, original_max_position_embeddings=8192)),
}


QWEN2_SHAPES: Dict[str, Dict] = {
    "qwen2-tiny": dict(hidden_size=896, num_hidden_layers=2, num_attention_heads=14, num_key_value_heads=2,
                       intermediate_size=1152, tie_word_embeddings=True),                  # head_dim 64: un-fused RoPE
    "qwen2-hd128": dict(hidden_size=1536, num_hidden_layers=2, num_attention_heads=12, num_key_value_heads=2,
                        intermediate_size=2048, tie_word_embeddings=False),                # head_dim 128: RoPE in the QKV epilogue
    "qwen2.5-7b": dict(hidden_size=3584, num_hidden_layers=28, num_attention_heads=28, num_key_value_heads=4,
                       intermediate_size=18944, tie_word_embeddings=False),
}


# head_dim is 128 in every Qwen3 dense model and set explicitly; the q width nh * 128 need not equal hidden_size
QWEN3_SHAPES: Dict[str, Dict] = {
    "qwen3-tiny": dict(hidden_size=384, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=1,
                       intermediate_size=768, tie_word_embeddings=True),    # 5 q|k heads: q/k norm + RoPE in the row kernel
    "qwen3-hd128": dict(hidden_size=512, num_hidden_layers=2, num_attention_heads=6, num_key_value_heads=2,
                        intermediate_size=1024, tie_word_embeddings=False),  # 8 q|k heads: q/k norm + RoPE in the QKV epilogue
    # published Qwen/Qwen3-0.6B and Qwen/Qwen3-8B config.json values (written from the model cards; not re-fetched offline)
    "qwen3-0.6b": dict(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, num_key_value_heads=8,
                       intermediate_size=3072, tie_word_embeddings=True),
    "qwen3-8b": dict(hidden_size=4096, num_hidden_layers=36, num_attention_heads=32, num_key_value_heads=8,
                     intermediate_size=12288, tie_word_embeddings=False),
}

# Qwen3-MoE (HF Qwen3MoeForCausalLM): Qwen3 attention, routed SwiGLU experts on the sparse layers (params.moe_layers)
QWEN3_MOE_SHAPES: Dict[str, Dict] = {
    # layer 1 of 3 dense (mlp_only_layers); 5 q|k heads: q/k norm + RoPE in the row kernel
    "qwen3-moe-tiny": dict(hidden_size=384, num_hidden_layers=3, num_attention_heads=4, num_key_value_heads=1,
                           intermediate_size=768, num_experts=8, num_experts_per_tok=2, moe_intermediate_size=128,
                           mlp_only_layers=[1], norm_topk_prob=True, tie_word_embeddings=True),
    # 8 q|k heads: q/k norm + RoPE in the QKV epilogue; every layer sparse, weights not renormalised
    "qwen3-moe-hd128": dict(hidden_size=512, num_hidden_layers=2, num_attention_heads=6, num_key_value_heads=2,
                            intermediate_size=1024, num_experts=16, num_experts_per_tok=4, moe_intermediate_size=256,
                            mlp_only_layers=[], norm_topk_prob=False, tie_word_embeddings=False),
    # published Qwen/Qwen3-30B-A3B config.json values (written from the model card; not re-fetched offline)
    "qwen3-30b-a3b": dict(hidden_size=2048, num_hidden_layers=48, num_attention_heads=32, num_key_value_heads=4,
                          intermediate_size=6144, num_experts=128, num_experts_per_tok=8, moe_intermediate_size=768,
                          mlp_only_layers=[], norm_topk_prob=True, tie_word_embeddings=False),
}


# XLM-RoBERTa / RoBERTa encoders: BERT's layer, positions counted from pad_token_id + 1
ROBERTA_SHAPES: Dict[str, Dict] = {
    "xlmr-tiny": dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=2, intermediate_size=128),      # head_dim 32: mma.sync attention
    "xlmr-hd64": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256),     # head_dim 64: wgmma attention
    "roberta-tiny": dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=2, intermediate_size=128, model_type="roberta"),
    # published config.json values (written from the model cards; not re-fetched offline)
    "multilingual-e5-base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072),
    "xlm-roberta-base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072),
    "bge-m3": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
                   max_position_embeddings=8194),
}


# Mistral (model_type "mistral"): Llama's layer with GQA and sliding-window causal attention. The tiny shapes cover the fused
# RoPE epilogue (head_dim 128) and the RoPE row kernel (head_dim 64, an odd window below one 64-key tile), and a config
# without a window. The published shapes were written from memory of their config.json files and could not be re-checked
# offline. `headless`: saved as MistralModel (AutoModel: no `model.` prefix, no lm_head), like e5-mistral-7b-instruct and
# SFR-Embedding-Mistral.
MISTRAL_SHAPES: Dict[str, Dict] = {
    "mistral-tiny": dict(hidden_size=512, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=128,
                         intermediate_size=1024, sliding_window=48),            # 6 q|k heads x 128: RoPE in the QKV epilogue
    "mistral-hd64": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                         intermediate_size=512, sliding_window=37),
    "mistral-nowin": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                          intermediate_size=512, sliding_window=None),
    "Mistral-7B-v0.1": dict(hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
                            intermediate_size=14336, sliding_window=4096, rope_theta=10000.0, vocab_size=32000),
    "Mistral-7B-v0.3": dict(hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
                            intermediate_size=14336, sliding_window=None, rope_theta=1000000.0, vocab_size=32768),
    "e5-mistral-7b-instruct": dict(hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8,
                                   head_dim=128, intermediate_size=14336, sliding_window=4096, rope_theta=10000.0,
                                   vocab_size=32000, headless=True),
    "Mistral-Nemo-Base-2407": dict(hidden_size=5120, num_hidden_layers=40, num_attention_heads=32, num_key_value_heads=8,
                                   head_dim=128, intermediate_size=14336, sliding_window=None, rope_theta=1000000.0,
                                   vocab_size=131072, max_position_embeddings=1024000),
}
# ModernBERT encoders (model_type "modernbert"): pre-norm layers with RoPE, GeGLU and, on two layers of three, bidirectional
# sliding-window attention. The tiny shapes use local_attention 16 (query i sees keys |i - j| <= 8) so that several windows fit
# in short test rows, and 4 layers: layer 0 (global, no attn_norm), two local layers and a second global one. The published
# shapes were written from memory of their config.json files and could not be re-checked offline.
MODERNBERT_SHAPES: Dict[str, Dict] = {
    "modernbert-tiny": dict(hidden_size=64, num_hidden_layers=4, num_attention_heads=2, intermediate_size=96,
                            local_attention=16),                              # head_dim 32: mma.sync attention
    "modernbert-hd64": dict(hidden_size=128, num_hidden_layers=4, num_attention_heads=2, intermediate_size=160,
                            local_attention=16),                              # head_dim 64: wgmma attention
    "ModernBERT-base": dict(hidden_size=768, num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152),
    "gte-modernbert-base": dict(hidden_size=768, num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152),
    "modernbert-embed-base": dict(hidden_size=768, num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152),
    "ModernBERT-large": dict(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, intermediate_size=2624),
}
FALCON_SHAPES: Dict[str, Dict] = {
    "falcon-tiny": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=2),
    "falcon-mini": dict(hidden_size=448, num_hidden_layers=2, num_attention_heads=7),          # 7 q heads x 64, one KV head
    "falcon-7b": dict(hidden_size=4544, num_hidden_layers=32, num_attention_heads=71),
}


def falcon_config(name: str, vocab_size: int = 65024) -> Dict:
    s = FALCON_SHAPES[name]
    return dict(
        architectures=["FalconForCausalLM"], model_type="falcon", vocab_size=vocab_size, alibi=False,
        new_decoder_architecture=False, multi_query=True, parallel_attn=True, bias=False, layer_norm_epsilon=1e-5,
        rope_theta=10000.0, hidden_dropout=0.0, attention_dropout=0.0, initializer_range=0.02, bos_token_id=11,
        eos_token_id=11, tie_word_embeddings=True, ffn_hidden_size=4 * s["hidden_size"], **s,
    )


def bert_config(name: str, vocab_size: int = 30522) -> Dict:
    s = BERT_SHAPES[name]
    return dict(
        architectures=["BertModel"], model_type="bert", vocab_size=vocab_size, max_position_embeddings=512,
        type_vocab_size=2, hidden_act="gelu", layer_norm_eps=1e-12, hidden_dropout_prob=0.1,
        attention_probs_dropout_prob=0.1, initializer_range=0.02, pad_token_id=0, position_embedding_type="absolute", **s,
    )


def roberta_config(name: str, vocab_size: Optional[int] = None) -> Dict:
    """XLM-RoBERTa (HF XLMRobertaModel, model_type "xlm-roberta", vocab 250002) or, for `roberta-tiny`, RoBERTa (model_type
    "roberta", vocab 50265): BERT's layers with layer_norm_eps 1e-5, one token type, pad_token_id 1 and a position table of
    max_position_embeddings = usable length + 2 (514; bge-m3 8194), since positions start at pad_token_id + 1. The published
    shapes (multilingual-e5-base, xlm-roberta-base, bge-m3) were written from their config.json files and could not be re-checked
    offline. multilingual-e5-small is not among them: it is published as a `bert` config (Multilingual-MiniLM) with an
    XLM-R tokenizer, so it already runs as a BERT encoder."""
    s = dict(ROBERTA_SHAPES[name])
    mt = s.pop("model_type", "xlm-roberta")
    arch = "RobertaModel" if mt == "roberta" else "XLMRobertaModel"
    cfg = dict(
        architectures=[arch], model_type=mt, vocab_size=vocab_size or (50265 if mt == "roberta" else 250002),
        max_position_embeddings=514, type_vocab_size=1, hidden_act="gelu", layer_norm_eps=1e-5, hidden_dropout_prob=0.1,
        attention_probs_dropout_prob=0.1, initializer_range=0.02, pad_token_id=1, bos_token_id=0, eos_token_id=2,
        position_embedding_type="absolute", use_cache=True, classifier_dropout=None,
    )
    cfg.update(s)
    return cfg


MODERNBERT_SPECIAL = {"[UNK]": 50280, "[CLS]": 50281, "[SEP]": 50282, "[PAD]": 50283, "[MASK]": 50284}


def modernbert_config(name: str, vocab_size: int = 50368) -> Dict:
    """ModernBERT (HF ModernBertModel): vocab 50368 with [CLS] 50281 / [SEP] 50282 / [PAD] 50283, local_attention 128 (the
    tiny shapes: 16), a global layer every 3, RoPE theta 160000 (global) / 10000 (local) in the hub spelling, norm_eps 1e-5, no
    biases, zero dropout and 8192 positions"""
    cfg = dict(
        architectures=["ModernBertModel"], model_type="modernbert", vocab_size=vocab_size, max_position_embeddings=8192,
        hidden_activation="gelu", norm_eps=1e-5, norm_bias=False, attention_bias=False, mlp_bias=False, attention_dropout=0.0,
        mlp_dropout=0.0, embedding_dropout=0.0, local_attention=128, global_attn_every_n_layers=3, global_rope_theta=160000.0,
        local_rope_theta=10000.0, initializer_range=0.02, pad_token_id=MODERNBERT_SPECIAL["[PAD]"],
        bos_token_id=MODERNBERT_SPECIAL["[CLS]"], cls_token_id=MODERNBERT_SPECIAL["[CLS]"],
        eos_token_id=MODERNBERT_SPECIAL["[SEP]"], sep_token_id=MODERNBERT_SPECIAL["[SEP]"],
    )
    cfg.update(MODERNBERT_SHAPES[name])
    return cfg


def llama_config(name: str, vocab_size: int = 32000) -> Dict:
    s = LLAMA_SHAPES[name]
    return dict(
        architectures=["LlamaForCausalLM"], model_type="llama", vocab_size=vocab_size, max_position_embeddings=4096,
        hidden_act="silu", rms_norm_eps=1e-5, rope_theta=10000.0, initializer_range=0.02, bos_token_id=1, eos_token_id=2,
        tie_word_embeddings=False, attention_bias=False, mlp_bias=False, attention_dropout=0.0,
        head_dim=s["hidden_size"] // s["num_attention_heads"], **s,
    )


def llama3_config(name: str, vocab_size: int = 128256) -> Dict:
    """Llama 3.x (HF LlamaForCausalLM): Llama-2's layer with GQA, rope_theta 5e5 and the llama3 RoPE frequency scaling
    (low_freq_factor 1, high_freq_factor 4). Token ids follow the synthetic tokenizer (`build_llama3_tokenizer`:
    <|begin_of_text|> = 0, <|end_of_text|> = 1), not the published 128000 / 128001."""
    s = dict(LLAMA3_SHAPES[name])
    rs = dict(rope_type="llama3", low_freq_factor=1.0, high_freq_factor=4.0, **s.pop("rope_scaling"))
    return dict(
        architectures=["LlamaForCausalLM"], model_type="llama", vocab_size=vocab_size, max_position_embeddings=131072,
        hidden_act="silu", rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=rs, initializer_range=0.02, bos_token_id=0,
        eos_token_id=1, attention_bias=False, mlp_bias=False, attention_dropout=0.0, pretraining_tp=1, **s,
    )


def mistral_config(name: str, vocab_size: Optional[int] = None) -> Dict:
    """Mistral (HF MistralForCausalLM, or MistralModel for a headless shape): Llama-2's layer with GQA, rms_norm_eps 1e-5, no
    biases and a `sliding_window` (null = none). Token ids follow the Llama SentencePiece layout (<unk> = 0, <s> = 1,
    </s> = 2), which the published tokenizers share."""
    s = dict(MISTRAL_SHAPES[name])
    headless = s.pop("headless", False)
    cfg = dict(
        architectures=["MistralModel" if headless else "MistralForCausalLM"], model_type="mistral",
        vocab_size=s.pop("vocab_size", 32000), max_position_embeddings=32768, hidden_act="silu", rms_norm_eps=1e-5,
        rope_theta=s.pop("rope_theta", 10000.0), initializer_range=0.02, bos_token_id=1, eos_token_id=2,
        tie_word_embeddings=False, attention_dropout=0.0,
    )
    cfg.update(s)
    if vocab_size:
        cfg["vocab_size"] = vocab_size
    return cfg


def qwen2_config(name: str, vocab_size: int = 152064) -> Dict:
    """Qwen2 / Qwen2.5 (HF Qwen2ForCausalLM): Llama plus q/k/v biases, rope_theta 1e6, rms_norm_eps 1e-6; full attention on
    every layer (use_sliding_window false, as in the published checkpoints)"""
    s = QWEN2_SHAPES[name]
    return dict(
        architectures=["Qwen2ForCausalLM"], model_type="qwen2", vocab_size=vocab_size, max_position_embeddings=32768,
        hidden_act="silu", rms_norm_eps=1e-6, rope_theta=1000000.0, initializer_range=0.02, bos_token_id=0, eos_token_id=0,
        use_sliding_window=False, sliding_window=None, max_window_layers=s["num_hidden_layers"], attention_dropout=0.0, **s,
    )


def qwen3_config(name: str, vocab_size: int = 151936) -> Dict:
    """Qwen3 dense (HF Qwen3ForCausalLM): Llama plus a per-head RMSNorm of q and k before RoPE (q_norm / k_norm, weight [128]),
    head_dim 128, no attention biases, rope_theta 1e6, rms_norm_eps 1e-6, full attention on every layer. Token ids follow the
    synthetic ChatML tokenizer (<|endoftext|> = 0), not the published 151643 / 151645."""
    s = QWEN3_SHAPES[name]
    return dict(
        architectures=["Qwen3ForCausalLM"], model_type="qwen3", vocab_size=vocab_size, max_position_embeddings=40960,
        hidden_act="silu", rms_norm_eps=1e-6, rope_theta=1000000.0, rope_scaling=None, initializer_range=0.02, bos_token_id=0,
        eos_token_id=0, head_dim=128, attention_bias=False, attention_dropout=0.0, use_sliding_window=False, sliding_window=None,
        max_window_layers=s["num_hidden_layers"], **s,
    )


def qwen3_moe_config(name: str, vocab_size: int = 151936) -> Dict:
    """Qwen3-MoE (HF Qwen3MoeForCausalLM): qwen3_config's attention and norms; the sparse layers route each token to its top
    num_experts_per_tok of num_experts SwiGLU experts (moe_intermediate_size), decoder_sparse_step 1. No sliding window."""
    s = dict(QWEN3_MOE_SHAPES[name])
    return dict(
        architectures=["Qwen3MoeForCausalLM"], model_type="qwen3_moe", vocab_size=vocab_size, max_position_embeddings=40960,
        hidden_act="silu", rms_norm_eps=1e-6, rope_theta=1000000.0, rope_scaling=None, initializer_range=0.02, bos_token_id=0,
        eos_token_id=0, head_dim=128, attention_bias=False, attention_dropout=0.0, use_sliding_window=False, sliding_window=None,
        max_window_layers=s["num_hidden_layers"], decoder_sparse_step=1, output_router_logits=False,
        router_aux_loss_coef=0.001, **s,
    )


# ---------------------------------------------------------------------------------------------------------------
# synthetic text
# ---------------------------------------------------------------------------------------------------------------
_SYL = ["ka", "to", "mi", "ren", "sol", "va", "qu", "ex", "pli", "dor", "an", "be", "cu", "fi", "gra", "hy", "jo", "lu",
        "ne", "os", "pa", "ri", "su", "ty", "ul", "vo", "wi", "xa", "yo", "ze"]


def word_list(n: int = 20000, seed: int = 7) -> List[str]:
    rng = np.random.default_rng(seed)
    words, seen = [], set()
    while len(words) < n:
        k = int(rng.integers(1, 5))
        w = "".join(_SYL[int(i)] for i in rng.integers(0, len(_SYL), size=k))
        if w not in seen:
            seen.add(w)
            words.append(w)
    return words


def synthetic_rows(n_rows: int, seed: int = 1234, full: bool = False, words: Optional[List[str]] = None):
    """SURVEY §8d: Zipf(1.1) words; lengths passage~U[110,160], query~U[12,40], answer~U[3,25] words.
    full=True: passage>=200, query>=60, answer>=150 words so every tokenised sequence hits truncation (masks all ones)."""
    words = words or word_list()
    rng = np.random.default_rng(seed)
    nw = len(words)

    def sample(k: int) -> str:
        idx = np.minimum(rng.zipf(1.1, size=k) - 1, nw - 1)
        return " ".join(words[int(i)] for i in idx)

    for _ in range(n_rows):
        if full:
            lp, lq, la = int(rng.integers(200, 240)), int(rng.integers(60, 80)), int(rng.integers(150, 180))
        else:
            lp, lq, la = int(rng.integers(110, 161)), int(rng.integers(12, 41)), int(rng.integers(3, 26))
        yield {"Abstract": sample(lp), "Question": sample(lq), "Answer": sample(la)}


def write_csv(path: str, n_rows: int, seed: int = 1234, full: bool = False) -> str:
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for row in synthetic_rows(n_rows, seed=seed, full=full):
            w.writerow(row)
    return path


# ---------------------------------------------------------------------------------------------------------------
# tokenizers (trained offline on the synthetic word list with the `tokenizers` library)
# ---------------------------------------------------------------------------------------------------------------
def _corpus(n: int = 3000) -> List[str]:
    rows = list(synthetic_rows(n, seed=99))
    out = []
    for r in rows:
        out += [f"#query# {r['Question']}", f"#passage# {r['Abstract']}", f"#answer# {r['Answer']}"]
    return out


def build_bert_tokenizer(out_dir: str, vocab_size: int = 30522) -> str:
    """WordPiece vocabulary trained on the synthetic corpus, wrapped in transformers' BertTokenizer (lower-casing,
    [CLS]/[SEP], token_type_ids) like BAAI/bge-*'s tokenizer."""
    from tokenizers import Tokenizer, models, normalizers, pre_tokenizers, trainers
    from transformers import BertTokenizer

    tok = Tokenizer(models.WordPiece(unk_token="[UNK]"))
    tok.normalizer = normalizers.BertNormalizer(lowercase=True)
    tok.pre_tokenizer = pre_tokenizers.BertPreTokenizer()
    special = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    trainer = trainers.WordPieceTrainer(vocab_size=min(vocab_size, 8000), special_tokens=special, show_progress=False)
    tok.train_from_iterator(_corpus(), trainer)
    vocab = dict(tok.get_vocab())
    nxt = len(vocab)
    while nxt < vocab_size:          # pad up to the architecture's vocab size so ids span the real embedding table
        vocab[f"[unused{nxt}]"] = nxt
        nxt += 1
    bt = BertTokenizer(vocab=vocab, do_lower_case=True, model_max_length=512)
    os.makedirs(out_dir, exist_ok=True)
    bt.save_pretrained(out_dir)
    return out_dir


ROBERTA_SPECIAL = ["<s>", "<pad>", "</s>", "<unk>"]          # ids 0-3 as in XLM-R and RoBERTa; <mask> is the last id


def build_xlmr_tokenizer(out_dir: str, vocab_size: int = 250002, model_max_length: int = 512) -> str:
    """XLM-R-style Unigram (Metaspace) trained on the synthetic corpus, wrapped in transformers' XLMRobertaTokenizerFast:
    <s> / <pad> / </s> / <unk> = 0-3, <mask> last, `<s> $A </s>` framing, no token_type_ids"""
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import XLMRobertaTokenizerFast

    tok = Tokenizer(models.Unigram())
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
    trainer = trainers.UnigramTrainer(vocab_size=min(vocab_size - 1, 8000), special_tokens=ROBERTA_SPECIAL, unk_token="<unk>",
                                      show_progress=False)
    tok.train_from_iterator(_corpus(), trainer)
    pieces = [tuple(v) for v in json.loads(tok.to_str())["model"]["vocab"]]
    pieces += [(f"<extra_{i}>", -1e4) for i in range(len(pieces), vocab_size - 1)]   # ids span the real embedding table
    pieces.append(("<mask>", 0.0))
    xt = XLMRobertaTokenizerFast(vocab=pieces, model_max_length=model_max_length)
    os.makedirs(out_dir, exist_ok=True)
    xt.save_pretrained(out_dir)
    return out_dir


def build_roberta_tokenizer(out_dir: str, vocab_size: int = 50265, model_max_length: int = 512) -> str:
    """RoBERTa-style byte-level BPE trained on the synthetic corpus, wrapped in transformers' RobertaTokenizer (the fast,
    tokenizers-backed class): the same special ids and framing as build_xlmr_tokenizer"""
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import RobertaTokenizer

    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    trainer = trainers.BpeTrainer(vocab_size=min(vocab_size - 1, 6000), special_tokens=ROBERTA_SPECIAL, show_progress=False,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(), trainer)
    vocab = tok.get_vocab()
    model_json = json.loads(tok.to_str())["model"]
    merges = [tuple(m) if isinstance(m, list) else tuple(m.split(" ")) for m in model_json["merges"]]
    nxt = len(vocab)
    while nxt < vocab_size - 1:
        vocab[f"<extra_{nxt}>"] = nxt
        nxt += 1
    vocab["<mask>"] = nxt
    rt = RobertaTokenizer(vocab=vocab, merges=merges, model_max_length=model_max_length)
    os.makedirs(out_dir, exist_ok=True)
    rt.save_pretrained(out_dir)
    return out_dir


def build_modernbert_tokenizer(out_dir: str, vocab_size: int = 50368) -> str:
    """ModernBERT-style byte-level BPE trained on the synthetic corpus, saved as a `PreTrainedTokenizerFast` like the published
    one: [UNK] / [CLS] / [SEP] / [PAD] / [MASK] at 50280-50284, `[CLS] $A [SEP]` framing, right padding, and only input_ids /
    attention_mask as model inputs (no token_type_ids)"""
    from tokenizers import AddedToken, Tokenizer, decoders, models, pre_tokenizers, processors, trainers
    from transformers import PreTrainedTokenizerFast

    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=6000, show_progress=False, initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(), trainer)
    first = min(MODERNBERT_SPECIAL.values())
    tok.add_tokens([f"<|extra_{i}|>" for i in range(tok.get_vocab_size(), first)])       # ids span the real embedding table
    tok.add_special_tokens([AddedToken(t, special=True) for t in sorted(MODERNBERT_SPECIAL, key=MODERNBERT_SPECIAL.get)])
    tok.add_tokens([f"[unused{i}]" for i in range(tok.get_vocab_size(), vocab_size)])
    cls, sep = MODERNBERT_SPECIAL["[CLS]"], MODERNBERT_SPECIAL["[SEP]"]
    tok.post_processor = processors.TemplateProcessing(single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1",
                                                       special_tokens=[("[CLS]", cls), ("[SEP]", sep)])
    ft = PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="[UNK]", cls_token="[CLS]", sep_token="[SEP]",
                                 pad_token="[PAD]", mask_token="[MASK]", padding_side="right", model_max_length=8192,
                                 model_input_names=["input_ids", "attention_mask"])
    os.makedirs(out_dir, exist_ok=True)
    ft.save_pretrained(out_dir)
    return out_dir


def build_llama_tokenizer(out_dir: str, vocab_size: int = 32000) -> str:
    """Llama-style BPE (metaspace, byte fallback, <unk>/<s>/</s> = 0/1/2) wrapped in transformers' LlamaTokenizer so that
    `add_eos_token = True` (reference train_rage2e.py:304) behaves as it does for the real Llama-2 tokenizer."""
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import LlamaTokenizer

    tok = Tokenizer(models.BPE(unk_token="<unk>", fuse_unk=True, byte_fallback=True))
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="first", split=False)
    byte_tokens = [f"<0x{i:02X}>" for i in range(256)]
    trainer = trainers.BpeTrainer(vocab_size=min(vocab_size, 6000), special_tokens=["<unk>", "<s>", "</s>"] + byte_tokens, show_progress=False)
    tok.train_from_iterator(_corpus(), trainer)
    vocab = tok.get_vocab()
    model_json = json.loads(tok.to_str())["model"]
    merges = [tuple(m) if isinstance(m, list) else tuple(m.split(" ")) for m in model_json["merges"]]
    nxt = len(vocab)
    while nxt < vocab_size:
        vocab[f"<extra_{nxt}>"] = nxt
        nxt += 1
    lt = LlamaTokenizer(vocab=vocab, merges=merges)
    lt.add_bos_token = True           # Llama-2 prepends <s>; baked into the saved post-processor
    os.makedirs(out_dir, exist_ok=True)
    lt.save_pretrained(out_dir)
    return out_dir


LLAMA3_SPECIAL = ["<|begin_of_text|>", "<|end_of_text|>", "<|eot_id|>", "<|eom_id|>"]
# Llama 3's pre-tokenizer split (published tokenizer.json), ahead of the byte-level mapping
LLAMA3_SPLIT = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|"
                r"\s+(?!\S)|\s+")


def build_llama3_tokenizer(out_dir: str, vocab_size: int = 128256) -> str:
    """Llama-3-style byte-level BPE trained on the synthetic corpus, saved as a `PreTrainedTokenizerFast` like the published
    one: the specials <|begin_of_text|> / <|end_of_text|> / <|eot_id|> / <|eom_id|> are ids 0-3, BOS is prepended by a
    TemplateProcessing post-processor, and tokenizer_config.json carries no add_bos_token / add_eos_token. So setting
    `add_eos_token = True` (the trainer does, as the reference does) rebuilds the post-processor from those flags, exactly as
    it does for a real Llama 3 tokenizer under the installed transformers."""
    from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, processors, trainers
    from transformers import PreTrainedTokenizerFast

    tok = Tokenizer(models.BPE(ignore_merges=True))
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(LLAMA3_SPLIT), behavior="isolated"),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=min(vocab_size, 6000), special_tokens=LLAMA3_SPECIAL, show_progress=False,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(), trainer)
    nxt = tok.get_vocab_size()
    tok.add_special_tokens([f"<|reserved_special_token_{i}|>" for i in range(vocab_size - nxt)])   # fill the embedding table
    bos = LLAMA3_SPECIAL[0]
    tok.post_processor = processors.TemplateProcessing(single=f"{bos} $A", pair=f"{bos} $A {bos}:1 $B:1", special_tokens=[(bos, 0)])
    ft = PreTrainedTokenizerFast(tokenizer_object=tok, bos_token=bos, eos_token=LLAMA3_SPECIAL[1], model_max_length=131072)
    os.makedirs(out_dir, exist_ok=True)
    ft.save_pretrained(out_dir)
    path = os.path.join(out_dir, "tokenizer_config.json")
    with open(path) as f:
        tc = json.load(f)
    for k in ("add_bos_token", "add_eos_token"):
        tc.pop(k, None)
    tc["tokenizer_class"] = "PreTrainedTokenizerFast"
    with open(path, "w") as f:
        json.dump(tc, f, indent=1)
    return out_dir


QWEN2_SPECIAL = ["<|endoftext|>", "<|im_start|>", "<|im_end|>"]


def build_qwen2_tokenizer(out_dir: str, vocab_size: int = 152064) -> str:
    """Qwen2-style byte-level BPE (GPT-2 byte alphabet, no BOS) trained on the synthetic corpus and wrapped in transformers'
    Qwen2Tokenizer; the ChatML specials <|endoftext|> / <|im_start|> / <|im_end|> are ids 0-2, <|endoftext|> is pad and eos"""
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import Qwen2Tokenizer

    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    trainer = trainers.BpeTrainer(vocab_size=min(vocab_size, 6000), special_tokens=QWEN2_SPECIAL, show_progress=False,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(), trainer)
    vocab = tok.get_vocab()
    model_json = json.loads(tok.to_str())["model"]
    merges = [tuple(m) if isinstance(m, list) else tuple(m.split(" ")) for m in model_json["merges"]]
    nxt = len(vocab)
    while nxt < vocab_size:
        vocab[f"<|extra_{nxt}|>"] = nxt
        nxt += 1
    qt = Qwen2Tokenizer(vocab=vocab, merges=merges, unk_token=None, eos_token="<|endoftext|>", pad_token="<|endoftext|>",
                        additional_special_tokens=["<|im_start|>", "<|im_end|>"], model_max_length=32768)
    os.makedirs(out_dir, exist_ok=True)
    qt.save_pretrained(out_dir)
    return out_dir


# base Qwen2.5 checkpoints decode greedily; the Instruct ones sample with a repetition penalty (their generation_config.json)
QWEN2_GENERATION = {
    "base": dict(bos_token_id=0, eos_token_id=0, do_sample=False, max_new_tokens=2048),
    "instruct": dict(bos_token_id=0, eos_token_id=[2, 0], pad_token_id=0, do_sample=True, repetition_penalty=1.05,
                     temperature=0.7, top_p=0.8, top_k=20),
}


# Llama 3.x base and Instruct checkpoints both sample (temperature 0.6, top-p 0.9); the Instruct ones stop at <|end_of_text|>,
# <|eom_id|> or <|eot_id|>. Ids mapped onto the synthetic tokenizer.
LLAMA3_GENERATION = {
    "base": dict(bos_token_id=0, eos_token_id=1, do_sample=True, temperature=0.6, top_p=0.9),
    "instruct": dict(bos_token_id=0, eos_token_id=[1, 3, 2], do_sample=True, temperature=0.6, top_p=0.9),
}


# Qwen3 base checkpoints decode greedily; the hybrid-thinking / Instruct ones sample (temperature 0.6, top-k 20, top-p 0.95)
# and stop at <|im_end|> or <|endoftext|>. Ids mapped onto the synthetic tokenizer.
QWEN3_GENERATION = {
    "base": dict(bos_token_id=0, eos_token_id=0, do_sample=False, max_new_tokens=2048),
    "instruct": dict(bos_token_id=0, eos_token_id=[2, 0], pad_token_id=0, do_sample=True, temperature=0.6, top_k=20, top_p=0.95),
}


# ---------------------------------------------------------------------------------------------------------------
# model directories
# ---------------------------------------------------------------------------------------------------------------
def write_model_dir(out_dir: str, kind: str, name: str, vocab_size: Optional[int] = None, with_weights: bool = True,
                    seed: int = 0, generation_config: Optional[Dict] = None, bias_std: Optional[float] = None,
                    qk_norm_std: Optional[float] = None, headless: Optional[bool] = None,
                    router_std: Optional[float] = None) -> str:
    """kind: 'bert' | 'roberta' | 'modernbert' | 'llama' | 'qwen2' | 'qwen3' | 'mistral' | 'falcon' ('roberta' takes a ROBERTA_SHAPES name: XLM-R
    shapes get the XLM-R tokenizer, roberta-tiny the byte-level one; a Llama 3.x shape of LLAMA3_SHAPES takes kind 'llama' and
    gets the Llama 3 tokenizer; 'mistral' gets the Llama SentencePiece tokenizer). headless (mistral; default: the shape's own
    setting): a MistralModel directory, weights without the `model.` prefix and without lm_head. Writes config.json, tokenizer files and (optionally) seeded random-init
    safetensors in HF parameter naming so both transformers (oracle) and dalm_b200 (product) can load the same directory.
    generation_config: written as generation_config.json when given (e.g. QWEN2_GENERATION["base"]). bias_std: std of the
    random attention biases, qk_norm_std the spread of Qwen3's q / k norm weights around 1, router_std the std of Qwen3-MoE's
    router weights (engine/params.random_state_dict). 'qwen3_moe' takes a QWEN3_MOE_SHAPES name and Qwen2's tokenizer."""
    os.makedirs(out_dir, exist_ok=True)
    if kind == "bert":
        cfg = bert_config(name, vocab_size or 30522)
        build_bert_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "roberta":
        cfg = roberta_config(name, vocab_size)
        from .engine.params import roberta_max_len

        build = build_roberta_tokenizer if cfg["model_type"] == "roberta" else build_xlmr_tokenizer
        build(out_dir, cfg["vocab_size"], model_max_length=roberta_max_len(cfg))
    elif kind == "llama" and name in LLAMA3_SHAPES:
        cfg = llama3_config(name, vocab_size or 128256)
        build_llama3_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "llama":
        cfg = llama_config(name, vocab_size or 32000)
        build_llama_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "qwen2":
        cfg = qwen2_config(name, vocab_size or 152064)
        build_qwen2_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "qwen3":
        cfg = qwen3_config(name, vocab_size or 151936)
        build_qwen2_tokenizer(out_dir, cfg["vocab_size"])          # Qwen3 keeps Qwen2's byte-level BPE and Qwen2Tokenizer
    elif kind == "qwen3_moe":
        cfg = qwen3_moe_config(name, vocab_size or 151936)
        build_qwen2_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "mistral":
        cfg = mistral_config(name, vocab_size)
        if headless is not None:
            cfg["architectures"] = ["MistralModel" if headless else "MistralForCausalLM"]
        build_llama_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "modernbert":
        cfg = modernbert_config(name, vocab_size or 50368)
        build_modernbert_tokenizer(out_dir, cfg["vocab_size"])
    elif kind == "falcon":
        cfg = falcon_config(name, vocab_size or 65024)
        build_llama_tokenizer(out_dir, cfg["vocab_size"])       # any causal-LM tokenizer works for the synthetic fixture
    else:
        raise ValueError(kind)
    with open(os.path.join(out_dir, "config.json"), "w") as f:
        json.dump(cfg, f, indent=1)
    if generation_config is not None:
        with open(os.path.join(out_dir, "generation_config.json"), "w") as f:
            json.dump(generation_config, f, indent=1)
    if not with_weights:
        with open(os.path.join(out_dir, "dalm_b200_random_init.json"), "w") as f:      # engine/params.py: random init at load time
            json.dump({"seed": seed}, f)
    if with_weights:
        import torch
        from safetensors.torch import save_file

        from .engine.params import random_state_dict

        sd = random_state_dict(kind, cfg, seed=seed, dtype=torch.float32, device="cpu", bias_std=bias_std, qk_norm_std=qk_norm_std,
                               router_std=router_std)
        if cfg.get("architectures") == ["MistralModel"]:
            sd = headless_state_dict(sd)
        save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(out_dir, "model.safetensors"))
    return out_dir


def headless_state_dict(sd: Dict) -> Dict:
    """a CausalLM state dict as its base model saves it (AutoModel / MistralModel): `model.` stripped, lm_head dropped"""
    return {k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}
