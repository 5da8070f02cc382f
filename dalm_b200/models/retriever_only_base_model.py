"""H100-native `AutoModelForSentenceEmbedding` (reference dalm/models/retriever_only_base_model.py:10-110)."""
from __future__ import annotations

import logging
from typing import Any, Optional

import torch

from .. import ops
from ..engine.bert import BertEncoder
from ..engine.bridge import EncodeFn, PoolFn
from .rag_e2e_base_model import _device, _want_full, build_encoder, load_tokenizer, pooling_mask

logger = logging.getLogger(__name__)


class AutoModelForSentenceEmbedding(torch.nn.Module):
    def __init__(self, model_name: str, normalize: bool = True, use_bnb: bool = True, get_peft: bool = True,
                 is_autoregressive: bool = False, *, _model: Optional[BertEncoder] = None,
                 _load_tokenizer: bool = True) -> None:
        super().__init__()
        # use_bnb (the reference's default, :15): the Linear weights take the values of the NF4 quantise/dequantise round trip
        # the reference's 4-bit model computes with (csrc/nf4.cu); they stay resident as bf16 — see DESIGN.md
        # get_peft=False: every parameter is trained (reference :28-33 skips get_peft_model, Adam covers model.parameters())
        self.model = _model if _model is not None else build_encoder(model_name, bool(get_peft), _device(),
                                                                     autoregressive=is_autoregressive, full=_want_full(bool(get_peft)),
                                                                     bnb=bool(use_bnb))
        self.tokenizer = load_tokenizer(model_name) if _load_tokenizer else None
        if is_autoregressive and self.tokenizer is not None:                                          # reference :36-38
            self.tokenizer.add_eos_token = True
            self.tokenizer.pad_token = self.tokenizer.eos_token
        self.normalize = normalize
        self.is_autoregressive = is_autoregressive

    def forward(self, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:      # reference :48-64
        enc = self.model
        ids = input_ids.to(enc.dev, torch.int64).contiguous()
        mask = attention_mask.to(enc.dev, torch.int64).contiguous()
        pm = pooling_mask(mask, self.is_autoregressive).contiguous()
        if enc.trainable and torch.is_grad_enabled():
            return EncodeFn.apply(enc.anchor, enc, ids, mask, self.normalize, pm)
        hid, _ = enc.forward_hidden(ids, mask, save=False)
        emb, _ = ops.pool_norm_fwd(hid, pm, self.normalize)
        return emb

    def mean_pooling(self, model_output: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:  # :66-68
        return PoolFn.apply(model_output, attention_mask.to(model_output.device, torch.int64).contiguous())

    def __getattr__(self, name: str) -> Any:                                                          # :70-75
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self.model, name)

    def print_trainable_parameters(self) -> None:
        """what `model.print_trainable_parameters()` (PEFT) prints through the reference's __getattr__ fall-through
        (train_retriever_only.py:260)"""
        trainable = sum(b.numel() for b in self.model.banks())
        if self.model.full is not None:
            total = trainable
        else:
            total = trainable + sum(t.numel() for W in self.model.layers for k, t in W.items()
                                    if isinstance(t, torch.Tensor) and not k.endswith("T") and not k.endswith("T_aug")
                                    and k not in ("A_stack", "Bblk"))
        print(f"trainable params: {trainable:,d} || all params: {total:,d} || trainable%: {100 * trainable / max(total, 1):.4f}")

    def attach_pre_trained_peft_layers(self, peft_retriever_path: str, device: str) -> None:          # :77-83
        from ..training.utils.train_utils import load_adapter_dir

        load_adapter_dir(self.model, peft_retriever_path)
