"""H100-native `AutoModelForRagE2E` — same constructor, attributes and methods as the reference wrapper
(dalm/models/rag_e2e_base_model.py:16-160), with the HF/PEFT modules behind it replaced by the dalm_b200 engine
(hand-written sm_90a kernels through the C ABI). There is no CPU or eager-PyTorch fallback.
"""
from __future__ import annotations

import logging
import os
from enum import Enum
from typing import Dict, Optional

import torch

from .. import ops
from ..engine import params
from ..engine.bert import BertEncoder
from ..engine.bridge import EncodeFn, GenerateFn, PoolFn
from ..engine.decoding import load_generation_config
from ..engine.falcon import FalconDecoder
from ..engine.llama import LlamaDecoder
from ..engine.modernbert import LORA_REFUSAL as MODERNBERT_LORA_REFUSAL
from ..engine.modernbert import ModernBertEncoder

logger = logging.getLogger(__name__)


class Mode(str, Enum):                       # reference :16-19
    GENERATOR = "generator"
    RETRIEVER = "retriever"
    BOTH = "both"


_INFERENCE_ONLY = False


class inference_only:
    """context manager for evaluation code: wrappers built inside it keep sub-models WITHOUT adapters frozen (bf16 weights
    only) instead of allocating the fp32 master / gradient banks of full fine-tuning. The reference has no such switch — it
    builds the same modules and simply never calls backward in dalm/eval/*."""

    def __enter__(self):
        global _INFERENCE_ONLY
        self.prev, _INFERENCE_ONLY = _INFERENCE_ONLY, True
        return self

    def __exit__(self, *exc):
        global _INFERENCE_ONLY
        _INFERENCE_ONLY = self.prev
        return False


def _want_full(lora: bool) -> bool:
    return (not lora) and not _INFERENCE_ONLY


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("dalm_b200 needs a CUDA (sm_90a) device: there is no CPU path for the training step")
    return torch.device("cuda", int(os.environ.get("LOCAL_RANK", torch.cuda.current_device())))


def load_tokenizer(name_or_path: str):
    from transformers import AutoTokenizer

    return AutoTokenizer.from_pretrained(name_or_path)


def build_encoder(name_or_path: str, lora: bool, device: torch.device, state_dict: Optional[Dict] = None,
                  cfg: Optional[Dict] = None, autoregressive: bool = False, full: bool = False, bnb: bool = False):
    """BERT-family encoder (bge-*), (XLM-)RoBERTa encoder (multilingual-e5, bge-m3, xlm-roberta-*), ModernBERT encoder
    (gte-modernbert, modernbert-embed; frozen or fully fine-tuned), or — `retriever_is_autoregressive` — a Llama / Qwen2 / Qwen3 /
    Mistral decoder (e5-mistral-7b-instruct, SFR-Embedding-Mistral) used as an encoder
    (last hidden state, eos pooling; LoRA targets q_proj / v_proj: reference rag_e2e_base_model.py:66-70,84-90)"""
    cfg = cfg or params.load_config(name_or_path)
    kind = params.model_kind(cfg)
    if kind == "modernbert":
        _check_modernbert_mode(lora, autoregressive, bnb)
        sd = state_dict if state_dict is not None else params.load_state_dict(name_or_path)
        return _named(ModernBertEncoder(cfg, sd, device=device, full=full), name_or_path)
    sd = state_dict if state_dict is not None else params.load_state_dict(name_or_path)
    nf4 = _nf4_storage(bnb, full, kind)
    if not nf4:
        sd = _maybe_bnb(sd, bnb, full, device)
    if autoregressive:
        if kind not in ("llama", "qwen2", "qwen3", "mistral"):
            raise NotImplementedError("autoregressive retrievers are built for Llama, Qwen2 and Qwen3 models only; Mistral "
                                      "runs as Llama with a sliding window")
        return _named(LlamaDecoder(cfg, sd, device=device, lora=lora, lora_seed=0, full=full, nf4_storage=nf4), name_or_path)
    if kind not in ("bert", "roberta"):
        raise NotImplementedError("non-autoregressive retrievers must be BERT (bge-*) or (XLM-)RoBERTa (multilingual-e5, bge-m3) "
                                  "encoders, or ModernBERT ones; pass retriever_is_autoregressive=True for a causal LM")
    return _named(BertEncoder(cfg, sd, device=device, lora=lora, full=full, nf4_storage=nf4), name_or_path)


def _check_modernbert_mode(lora: bool, autoregressive: bool, bnb: bool) -> None:
    """ModernBERT retrievers run frozen or fully fine-tuned; every other mode is refused, naming why"""
    from ..engine.nf4store import storage_enabled
    if autoregressive:
        raise NotImplementedError("retriever_is_autoregressive=True: ModernBERT is a bidirectional encoder (mean-pooled), "
                                  "not a causal LM")
    if lora:
        raise NotImplementedError(MODERNBERT_LORA_REFUSAL)
    if bnb and storage_enabled():
        raise NotImplementedError("DALM_B200_NF4_STORAGE=1: 4-bit storage is not built for ModernBERT retrievers (it serves "
                                  "LoRA-carrying BERT / (XLM-)RoBERTa encoders and Llama decoders)")
    if bnb:
        raise NotImplementedError("use_bnb on a ModernBERT retriever: the reference's 4-bit retriever needs LoRA on the same "
                                  "sub-model, and LoRA is not built for ModernBERT; drop use_bnb for the retriever")


def _named(engine_model, name_or_path: str):
    """remember where the base weights came from: written as `base_model_name_or_path` into adapter_config.json"""
    engine_model.name_or_path = name_or_path or None
    return engine_model


def _check_qwen3_moe_mode(full: bool, bnb: bool) -> None:
    """Qwen3-MoE generators run frozen or with LoRA on q_proj / v_proj; every other mode is refused, naming why"""
    if full:
        raise NotImplementedError("full fine-tuning of a qwen3_moe generator is not built: grouped expert weight gradients are "
                                  "not built, and at ~18 bytes per parameter (fp32 master, gradient, Adam moments, bf16 copy) "
                                  "Qwen3-30B-A3B would need ~550 GB; use LoRA (use_peft) on the generator")
    if bnb:
        raise NotImplementedError("use_bnb on a qwen3_moe generator is not built: the 4-bit treatment of the fused 3-D expert "
                                  "weights differs across transformers versions, so no single reference exists to match")


def _nf4_storage(bnb: bool, full: bool, kind: str) -> bool:
    """use_bnb + DALM_B200_NF4_STORAGE=1: keep the sub-model's Linear weights as packed NF4 codes and expand them per use
    (engine/nf4store.py) instead of the dequantised-resident default. BERT / (XLM-)RoBERTa encoders and Llama decoders."""
    from ..engine.nf4store import storage_enabled
    if not bnb or not storage_enabled():
        return False
    if full:
        _maybe_bnb({}, True, True, None)                      # raises: 4-bit base weights cannot be fully fine-tuned
    if kind not in ("bert", "roberta", "llama"):
        raise NotImplementedError(f"DALM_B200_NF4_STORAGE=1: 4-bit storage is built for BERT / (XLM-)RoBERTa encoders and Llama "
                                  f"decoders, not {kind!r}")
    return True


def _maybe_bnb(sd: Dict, bnb: bool, full: bool, device) -> Dict:
    """use_bnb: replace the checkpoint values by what the reference's NF4-loaded model computes with (engine/params.py)"""
    if not bnb:
        return sd
    if full:
        raise NotImplementedError("use_bnb without PEFT on the same sub-model: 4-bit base weights cannot be fully fine-tuned "
                                  "(the reference's Linear4bit weights do not receive gradients either) — add it to use_peft")
    return params.bnb_nf4_state_dict(sd, device)


def pooling_mask(attention_mask: torch.Tensor, autoregressive: bool) -> torch.Tensor:
    """mask used by mean_pooling: the attention mask, or for autoregressive retrievers `eos_mask(attention_mask)` (one-hot
    at the last column, reference dalm/utils.py:22-35 default padding='left') so the pool picks the final token"""
    if not autoregressive:
        return attention_mask
    from ..utils import eos_mask
    return eos_mask(attention_mask)


def build_decoder(name_or_path: str, lora: bool, device: torch.device, state_dict: Optional[Dict] = None,
                  cfg: Optional[Dict] = None, full: bool = False, bnb: bool = False) -> LlamaDecoder:
    cfg = cfg or params.load_config(name_or_path)
    kind = params.model_kind(cfg)                # raises for unsupported families
    if kind == "qwen3_moe":
        _check_qwen3_moe_mode(full, bnb)
    sd = state_dict if state_dict is not None else params.load_state_dict(name_or_path)
    nf4 = _nf4_storage(bnb, full, kind)
    if not nf4:
        sd = _maybe_bnb(sd, bnb, full, device)
    if kind == "falcon":
        dec = FalconDecoder(cfg, sd, device=device, lora=lora, full=full)      # raises for lora=True, like peft would
    elif kind not in ("llama", "qwen2", "qwen3", "mistral", "qwen3_moe"):
        raise NotImplementedError(f"generator of kind {kind!r} is not a causal decoder")
    else:
        dec = LlamaDecoder(cfg, sd, device=device, lora=lora, full=full, nf4_storage=nf4)
    dec.generation_config = load_generation_config(name_or_path)              # what `generate` starts from, like HF
    return _named(dec, name_or_path)


class AutoModelForRagE2E(torch.nn.Module):
    def __init__(
        self,
        retriever_name: str,
        generator_name: str,
        normalize: bool = True,
        get_peft: Optional[Mode] = None,
        use_bnb: Optional[Mode] = None,
        retriever_is_autoregressive: bool = False,
        *,
        _retriever: Optional[BertEncoder] = None,
        _generator: Optional[LlamaDecoder] = None,
        _load_tokenizers: bool = True,
    ) -> None:
        super().__init__()
        get_peft = Mode(get_peft) if get_peft is not None else None
        use_bnb = Mode(use_bnb) if use_bnb is not None else None
        bnb_r, bnb_g = use_bnb in (Mode.RETRIEVER, Mode.BOTH), use_bnb in (Mode.GENERATOR, Mode.BOTH)
        dev = _device()
        lora_r = get_peft in (Mode.RETRIEVER, Mode.BOTH)
        lora_g = get_peft in (Mode.GENERATOR, Mode.BOTH)
        # a sub-model without adapters is FULLY fine-tuned, as in the reference (no get_peft_model => every parameter keeps
        # requires_grad=True and Adam is built over rag_model.parameters(), train_rage2e.py:336)
        self.retriever_model = (_retriever if _retriever is not None else
                                build_encoder(retriever_name, lora_r, dev, autoregressive=retriever_is_autoregressive,
                                              full=_want_full(lora_r), bnb=bnb_r))
        self.generator_model = (_generator if _generator is not None else
                                build_decoder(generator_name, lora_g, dev, full=_want_full(lora_g), bnb=bnb_g))
        self.retriever_tokenizer = load_tokenizer(retriever_name) if _load_tokenizers else None
        if retriever_is_autoregressive and self.retriever_tokenizer is not None:                   # reference :41-44
            self.retriever_tokenizer.add_eos_token = True
            self.retriever_tokenizer.pad_token = self.retriever_tokenizer.eos_token
        self.generator_tokenizer = load_tokenizer(generator_name) if _load_tokenizers else None
        self.normalize = normalize
        self.retriever_is_autoregressive = retriever_is_autoregressive

    # ---- reference :83-99 -------------------------------------------------------------------------------------
    def retrieval_forward(self, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        enc = self.retriever_model
        ids = input_ids.to(enc.dev, torch.int64).contiguous()
        mask = attention_mask.to(enc.dev, torch.int64).contiguous()
        pm = pooling_mask(mask, self.retriever_is_autoregressive).contiguous()
        if enc.trainable and torch.is_grad_enabled():
            return EncodeFn.apply(enc.anchor, enc, ids, mask, self.normalize, pm)
        hid, _ = enc.forward_hidden(ids, mask, save=False)
        emb, _ = ops.pool_norm_fwd(hid, pm, self.normalize)
        return emb

    # ---- reference :101-106 -----------------------------------------------------------------------------------
    def forward(self, task: str, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        if task == "retrieval":
            return self.retrieval_forward(input_ids, attention_mask)
        dec = self.generator_model
        ids = input_ids.to(dec.dev, torch.int64).contiguous()
        mask = attention_mask.to(dec.dev, torch.int64).contiguous()
        if dec.trainable and torch.is_grad_enabled():
            return GenerateFn.apply(dec.anchor, dec, ids, mask)
        logits, _ = dec.forward_logits(ids, mask, save=False)
        return logits

    # ---- reference :108-111 -----------------------------------------------------------------------------------
    def mean_pooling(self, model_output: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        return PoolFn.apply(model_output, attention_mask.to(model_output.device, torch.int64).contiguous())

    # ---- reference :113-134 -----------------------------------------------------------------------------------
    def attach_pre_trained_peft_layers(self, peft_retriever_path: Optional[str], peft_generator_path: Optional[str],
                                       device: str) -> None:
        from ..training.utils.train_utils import load_adapter_dir

        if peft_retriever_path is not None:
            load_adapter_dir(self.retriever_model, peft_retriever_path)
        if peft_generator_path is not None:
            load_adapter_dir(self.generator_model, peft_generator_path)

    # ---- optimizer-facing helpers -----------------------------------------------------------------------------
    def trainable_banks(self):
        """LoRA banks / dense parameter banks of both sub-models (each has a flat `.grad`)"""
        return [b for m in (self.retriever_model, self.generator_model) for b in m.banks()]

    def repack(self) -> None:
        """refresh the bf16 LoRA blocks inside the fused weights after an optimizer step"""
        self.retriever_model.repack_lora()
        self.generator_model.repack_lora()
