"""CPU fp32 model oracle: HF transformers modeling code (the reference's third-party dependency for K1/K5) plus a
restatement of PEFT LoRA.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

`peft` is not installed offline and is unpinned in the reference (pyproject.toml:16-33): the LoRA layer below restates
the published definition with the reference's hyper-parameters (rag_e2e_base_model.py:144-160: r=8, alpha=16,
dropout=0.05, bias none; PEFT default init A~kaiming_uniform(a=sqrt5), B=0) — "parity unpinned" for this piece.
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional

import torch
from torch import nn

from . import losses, pooling


class LoraLinear(nn.Module):
    """y = W x + b + (alpha/r) * B(A(dropout(x)))"""

    def __init__(self, base: nn.Linear, A: torch.Tensor, B: torch.Tensor, alpha: int = 16, dropout: float = 0.0):
        super().__init__()
        self.base = base
        for p in self.base.parameters():
            p.requires_grad_(False)
        self.lora_A = nn.Parameter(A.clone().float())
        self.lora_B = nn.Parameter(B.clone().float())
        self.scale = alpha / A.shape[0]
        self.drop = nn.Dropout(dropout) if dropout > 0 else nn.Identity()

    def forward(self, x):
        return self.base(x) + (self.drop(x) @ self.lora_A.t() @ self.lora_B.t()) * self.scale


def _set_module(root: nn.Module, dotted: str, new: nn.Module) -> None:
    parts = dotted.split(".")
    m = root
    for p in parts[:-1]:
        m = getattr(m, p)
    setattr(m, parts[-1], new)


def _get_module(root: nn.Module, dotted: str) -> nn.Module:
    m = root
    for p in dotted.split("."):
        m = getattr(m, p)
    return m


def attach_lora(model: nn.Module, factors: Dict[str, Dict[str, torch.Tensor]], dropout: float = 0.0) -> None:
    """factors: {module_name: {"A": [r,in], "B": [out,r]}} with module names relative to `model`."""
    for p in model.parameters():
        p.requires_grad_(False)
    for name, f in factors.items():
        base = _get_module(model, name)
        _set_module(model, name, LoraLinear(base, f["A"], f["B"], dropout=dropout))


def build_bert(cfg: Dict, state_dict: Dict[str, torch.Tensor]) -> nn.Module:
    from transformers import BertConfig, BertModel

    c = BertConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    m = BertModel(c)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in state_dict.items()}, strict=False)
    assert not [k for k in missing if "position_ids" not in k], missing
    return m.float().eval()


def build_roberta(cfg: Dict, state_dict: Dict[str, torch.Tensor]) -> nn.Module:
    """transformers' XLMRobertaModel / RobertaModel (by model_type), eager attention"""
    import transformers

    prefix = "Roberta" if cfg["model_type"] == "roberta" else "XLMRoberta"
    c = getattr(transformers, prefix + "Config")(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")},
                                                  _attn_implementation="eager")
    m = getattr(transformers, prefix + "Model")(c)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in state_dict.items()}, strict=False)
    assert not [k for k in missing if "position_ids" not in k and "token_type_ids" not in k], missing
    assert not unexpected, unexpected
    return m.float().eval()


def build_modernbert(cfg: Dict, state_dict: Dict[str, torch.Tensor]) -> nn.Module:
    """transformers' ModernBertModel, eager attention"""
    from transformers import ModernBertConfig, ModernBertModel

    c = ModernBertConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")},
                         _attn_implementation="eager")
    m = ModernBertModel(c)
    missing, unexpected = m.load_state_dict(state_dict, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m.float().eval()


_CAUSAL_LM = {"llama": "Llama", "qwen2": "Qwen2", "qwen3": "Qwen3", "mistral": "Mistral"}


def build_causal_lm(cfg: Dict, state_dict: Dict[str, torch.Tensor], headless: bool = False,
                    attn_implementation: Optional[str] = None) -> nn.Module:
    """transformers' <Family>ForCausalLM, or <Family>Model when `headless`, for cfg["model_type"] in llama / qwen2 / qwen3 /
    mistral. attn_implementation None keeps transformers' default. A config with tie_word_embeddings may store no lm_head."""
    import transformers

    family = _CAUSAL_LM[cfg["model_type"]]
    c = getattr(transformers, family + "Config")(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    cls = getattr(transformers, family + ("Model" if headless else "ForCausalLM"))
    m = cls(c) if attn_implementation is None else cls._from_config(c, attn_implementation=attn_implementation)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in state_dict.items()}, strict=False)
    tied = {"lm_head.weight"} if cfg.get("tie_word_embeddings") else set()
    assert not unexpected and set(missing) <= tied, (missing, unexpected)
    return m.float().eval()


def build_llama(cfg: Dict, state_dict: Dict[str, torch.Tensor]) -> nn.Module:
    return build_causal_lm({**cfg, "model_type": "llama"}, state_dict)


def build_falcon(cfg: Dict, state_dict: Dict[str, torch.Tensor]) -> nn.Module:
    from transformers import FalconConfig, FalconForCausalLM

    c = FalconConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    m = FalconForCausalLM(c)
    sd = {k: v.float() for k, v in state_dict.items()}
    sd.setdefault("lm_head.weight", sd["transformer.word_embeddings.weight"])          # tied
    m.load_state_dict(sd, strict=True)
    return m.float().eval()


def retrieval_forward(bert: nn.Module, ids: torch.Tensor, mask: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """reference rag_e2e_base_model.py:83-99 (non-autoregressive branch): positional call => token_type_ids = 0"""
    tok = bert(ids, mask)[0]
    emb = pooling.mean_pooling(tok, mask)
    return pooling.normalize(emb) if normalize else emb


def retrieval_forward_autoregressive(llama_lm: nn.Module, ids: torch.Tensor, mask: torch.Tensor, normalize: bool = True):
    """reference rag_e2e_base_model.py:84-90 (autoregressive branch): last hidden state of the base model, `eos_mask`
    (one-hot at the last column, padding='left' default) as the pooling mask"""
    base = llama_lm.model if hasattr(llama_lm, "model") else llama_lm
    tok = base(ids, attention_mask=mask, output_hidden_states=True, return_dict=True).hidden_states[-1]
    emb = pooling.mean_pooling(tok, pooling.eos_mask(mask))
    return pooling.normalize(emb) if normalize else emb


def rag_step(bert: nn.Module, llama: nn.Module, batch: Dict[str, torch.Tensor], logit_scale: float = 100.0) -> Dict:
    """One forward+backward of the loop body, reference train_rage2e.py:431-471, in fp32 on CPU."""
    for m in (bert, llama):
        m.zero_grad(set_to_none=True)
    q = retrieval_forward(bert, batch["retriever_query_input_ids"], batch["retriever_query_attention_mask"])
    p = retrieval_forward(bert, batch["retriever_passage_input_ids"], batch["retriever_passage_attention_mask"])
    S = losses.get_cosine_sim(q, p, logit_scale)
    Lc = losses.contrastive_loss(S)
    logits = llama(input_ids=batch["generator_input_input_ids"], attention_mask=batch["generator_input_attention_mask"]).logits
    Lm = losses.marginalized_loss_loopform(logits, batch["generator_input_input_ids"],
                                           batch["generator_input_attention_mask"], S, batch["query_passage_input_len"])
    loss = Lc + Lm
    loss.backward()
    grads = {n: p_.grad.detach().clone() for m, pre in ((bert, "retriever."), (llama, "generator."))
             for n, p_ in ((pre + n, p_) for n, p_ in m.named_parameters()) if p_.grad is not None}
    return {"loss": loss.detach(), "Lc": Lc.detach(), "Lm": Lm.detach(), "q": q.detach(), "p": p.detach(),
            "S": S.detach(), "logits": logits.detach(), "grads": grads}


def retriever_step(bert: nn.Module, batch: Dict[str, torch.Tensor], logit_scale: float = 100.0) -> Dict:
    """reference train_retriever_only.py:365-376"""
    bert.zero_grad(set_to_none=True)
    q = retrieval_forward(bert, batch["query_input_ids"], batch["query_attention_mask"])
    p = retrieval_forward(bert, batch["passage_input_ids"], batch["passage_attention_mask"])
    S = losses.get_cosine_sim(q, p, logit_scale)
    loss = losses.contrastive_loss(S)
    loss.backward()
    grads = {"retriever." + n: p_.grad.detach().clone() for n, p_ in bert.named_parameters() if p_.grad is not None}
    return {"loss": loss.detach(), "q": q.detach(), "p": p.detach(), "S": S.detach(), "grads": grads}


# ----------------------------------------------------------------------------------------------------------------
# timing support for bench.py's baselines (cpu_baseline / --impl reference on host cores, gpu_eager_baseline on the GPU):
# the SAME modules as above, built without the minutes-long HF random initialisation of a 7 B model
# ----------------------------------------------------------------------------------------------------------------
def build_for_timing(kind: str, cfg: Dict, device="cpu", seed: int = 0) -> nn.Module:
    """HF BertModel / LlamaForCausalLM of the given config on `device`, fp32, train() mode, parameters filled by tiling one
    4 Mi-element N(0, 0.02) block (norm gains 1, biases from the block too). Values only need to be non-degenerate: these
    models are TIMED, never compared. Construction skips HF's init (transformers.initialization.no_init_weights)."""
    from transformers.initialization import no_init_weights

    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type") and not k.startswith("_")}
    with no_init_weights(), torch.device(device):
        if kind == "bert":
            from transformers import BertConfig, BertModel
            m = BertModel(BertConfig(**keep))
        elif kind == "llama":
            from transformers import LlamaConfig, LlamaForCausalLM
            m = LlamaForCausalLM(LlamaConfig(**keep))
        else:
            raise ValueError(kind)
    g = torch.Generator(device=device).manual_seed(seed)
    block = torch.empty(1 << 22, dtype=torch.float32, device=device).normal_(0.0, 0.02, generator=g)
    with torch.no_grad():
        for name, p in m.named_parameters():
            flat = p.data.view(-1)
            if p.dim() == 1 and ("norm" in name.lower() and name.endswith("weight")):
                flat.fill_(1.0)
                continue
            for lo in range(0, flat.numel(), block.numel()):
                n = min(block.numel(), flat.numel() - lo)
                flat[lo:lo + n].copy_(block[:n])
    return m.float().train()


def timing_lora_factors(kind: str, cfg: Dict, device="cpu", seed: int = 3) -> Dict[str, Dict[str, torch.Tensor]]:
    """LoRA factors for the reference's targets (rag_e2e_base_model.py:66-68,76-77), A ~ small normal, B = 0 (PEFT init)"""
    g = torch.Generator().manual_seed(seed)
    H, nl = cfg["hidden_size"], cfg["num_hidden_layers"]
    if kind == "bert":
        names = [f"encoder.layer.{i}.attention.self.{n}" for i in range(nl) for n in ("query", "key", "value")]
    else:
        names = [f"model.layers.{i}.self_attn.{n}" for i in range(nl) for n in ("q_proj", "v_proj")]
    return {n: {"A": (torch.randn(8, H, generator=g) / H ** 0.5).to(device), "B": torch.zeros(H, 8, device=device)} for n in names}


def loop_body_step(bert: nn.Module, llama: nn.Module, batch: Dict[str, torch.Tensor], optimizer, logit_scale: float = 100.0,
                   autocast: Optional[torch.dtype] = None) -> torch.Tensor:
    """The reference's loop body, train_rage2e.py:429-474, in eager PyTorch over the HF modules: two retrieval forwards,
    similarity, two-way contrastive loss, generator forward, marginalised loss, backward, optimizer.step, zero_grad.
    autocast = torch.bfloat16 reproduces `accelerate launch --mixed_precision bf16`; None is the reference's default (fp32)."""
    dev_type = next(llama.parameters()).device.type
    ctx = torch.autocast(dev_type, dtype=autocast) if autocast is not None else torch.autocast(dev_type, enabled=False)
    with ctx:
        q = retrieval_forward(bert, batch["retriever_query_input_ids"], batch["retriever_query_attention_mask"])
        p = retrieval_forward(bert, batch["retriever_passage_input_ids"], batch["retriever_passage_attention_mask"])
        S = losses.get_cosine_sim(q, p, logit_scale)
        Lc = losses.contrastive_loss(S)
        logits = llama(input_ids=batch["generator_input_input_ids"], attention_mask=batch["generator_input_attention_mask"]).logits
        Lm = losses.marginalized_loss_loopform(logits, batch["generator_input_input_ids"],
                                               batch["generator_input_attention_mask"], S, batch["query_passage_input_len"])
        loss = Lc + Lm
    loss.backward()
    optimizer.step()
    optimizer.zero_grad()
    return loss.detach()
