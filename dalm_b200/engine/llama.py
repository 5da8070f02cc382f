"""Llama / Qwen2 / Qwen3 / Mistral decoder (Llama-2-7B / Qwen2.5-7B / Qwen3-8B / Mistral-7B shape and smaller) forward + backward as a launch sequence over the C-ABI kernels.

Mirrors `self.generator_model(input_ids=..., attention_mask=...).logits` of the reference
(dalm/models/rag_e2e_base_model.py:104-106) through HF LlamaForCausalLM: embed -> N x [RMSNorm -> QKV(+LoRA on q,v)
-> RoPE -> causal+padding attention -> o_proj + residual -> RMSNorm -> SwiGLU MLP + residual] -> RMSNorm -> lm_head.

HBM layout per layer (bf16 unless noted):
  Wqkv_aug [Nq+2Nkv, H+Ra]  fused q|k|v rows, last Ra = 2r columns = (alpha/r)*B_q | (alpha/r)*B_v  (LoRA folded into K)
  WqkvT_aug [H, Nq+2Nkv+Ra] resident transpose for dgrad, last Ra columns = A_q^T | A_v^T
  A_stack [64,H], Bblk [64, Nq+2Nkv]   LoRA down / mid-gradient operands (see bert.py)
  Wo [H,Nq], WoT; Wgu [2F,H] (gate rows, then up rows), WguT [H,2F]; Wd [H,F], WdT [F,H]; RMSNorm gains fp32
  bqkv [Nq+2Nkv], bo [H] fp32: attention biases (Qwen2: q|k|v only; Llama / Qwen3 with attention_bias: both), added in the GEMM epilogues
  qn, kn [128] fp32: Qwen3's per-head q_norm / k_norm weights (RMSNorm of each q / k head before RoPE)
Residual stream and its gradient are fp32; every GEMM operand is bf16.
Qwen2 is this architecture plus q/k/v biases (HF Qwen2ForCausalLM); Qwen3 (HF Qwen3ForCausalLM) adds the per-head q/k RMSNorm,
fused into the QKV GEMM's RoPE epilogue (training shapes) or applied by the qk_norm_rope row kernel (decode, prefill, other
widths); the backward saves the pre-norm q|k columns and their rstd. Configs are checked by params.check_llama_family.
Llama 3.x is this architecture with GQA and frequency-scaled RoPE: params.rope_inv_freq builds the default, `linear` and
`llama3` frequencies, and every RoPE kernel reads the cos / sin tables `_rope` makes from them.
Mistral (HF MistralForCausalLM) is Llama with sliding-window causal attention: params.sliding_windows gives each layer's key
window (0 = none; also Qwen2 / Qwen3 with use_sliding_window), and every attention launch of that layer (training forward and
backward, prefill, decode) takes it. Headless checkpoints (HF MistralModel / LlamaModel saved by AutoModel, e.g.
e5-mistral-7b-instruct: `layers.*` with no `model.` prefix and no lm_head) load too; hf_state_dict writes their layout back.
Qwen3-MoE (HF Qwen3MoeForCausalLM) is Qwen3 whose sparse layers (params.moe_layers) run a routed mixture of SwiGLU experts
instead of the dense MLP: W["moe"] holds the router and the stacked expert weights, and engine/moe.py runs the layer in the
training forward and backward, the prefill and the decode step. Expert weights stay frozen (LoRA or inference only).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import ops
from . import moe
from .dense import DenseBank
from .lora import LoraBank
from .params import attention_biases, check_llama_family, moe_layers, rope_inv_freq, sliding_windows

bf16, f32 = torch.bfloat16, torch.float32


def _aug_buf(rows: int, cols: int, ra: int, device, zero: bool = False) -> torch.Tensor:
    """[rows, cols+ra] bf16 view whose row stride is padded to cols+64 when ra > 0, so that every row starts on a
    128-byte boundary (TMA 128B-swizzled boxes then touch aligned lines; measured +20 % on the K-augmented GEMMs)"""
    ld = cols + (64 if ra else 0)
    base = (torch.zeros if zero else torch.empty)(rows, ld, dtype=bf16, device=device)
    return base[:, :cols + ra]


class _Ctx:
    pass


def _with_prefix(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """a headless (AutoModel) state dict under LlamaForCausalLM names: every key gains `model.` (it has no lm_head)"""
    return {"model." + k: v for k, v in sd.items()}


class LlamaDecoder(torch.nn.Module):
    LORA_TARGETS = ("q_proj", "v_proj")               # reference rag_e2e_base_model.py:76-77

    def __init__(self, cfg: Dict, state_dict: Dict[str, torch.Tensor], device="cuda", lora: bool = False,
                 lora_seed: int = 1, full: bool = False, nf4_storage: bool = False):
        """lora: PEFT mode (frozen base + rank-8 adapters on q_proj / v_proj). full: every parameter trainable (reference
        behaviour without --use-peft): weights in a DenseBank (fp32 master + bf16 shadow), no transposed copies."""
        super().__init__()
        if lora and full:
            raise ValueError("lora and full fine-tuning are mutually exclusive for one model")
        if nf4_storage and full:
            raise ValueError("4-bit base weights cannot be fully fine-tuned")
        # use_bnb with 4-bit STORAGE (engine/nf4store.py): `state_dict` then holds the ORIGINAL checkpoint values; the layers'
        # Linear weights are kept as NF4 codes and expanded to bf16 per use, everything else takes transformers' fp16 cast
        self.nf4 = None
        if nf4_storage:
            from .nf4store import Nf4Store
            self.nf4 = Nf4Store(device)
        check_llama_family(cfg)
        self.cfg = cfg
        self.kind = cfg.get("model_type") if cfg.get("model_type") in ("qwen2", "qwen3", "mistral", "qwen3_moe") else "llama"
        self.qkv_bias, self.o_bias = attention_biases(self.kind, cfg)
        self.qk_norm = self.kind in ("qwen3", "qwen3_moe")
        self.H = H = cfg["hidden_size"]
        self.F = F = cfg.get("intermediate_size") or 0          # qwen3_moe without dense layers may leave it out
        # Qwen3-MoE: the layers that run the routed MLP (engine/moe.py) instead of the dense SwiGLU one
        self.sparse = moe_layers(cfg) if self.kind == "qwen3_moe" else [False] * cfg["num_hidden_layers"]
        if any(self.sparse) and (full or nf4_storage):
            raise NotImplementedError("qwen3_moe: " + ("full fine-tuning is not built (grouped expert weight gradients are not "
                                                       "built)" if full else "4-bit storage of the expert weights is not built"))
        self.nl = cfg["num_hidden_layers"]
        self.nh = cfg["num_attention_heads"]
        self.nkv = cfg.get("num_key_value_heads", self.nh)
        self.hd = cfg.get("head_dim") or H // self.nh
        self.V = cfg["vocab_size"]
        self.eps = float(cfg.get("rms_norm_eps", 1e-5))
        self.dev = torch.device(device)
        if self.hd not in (32, 64, 128):
            raise NotImplementedError(f"head_dim {self.hd} not supported by the attention kernels")
        self.inv_freq = rope_inv_freq(cfg, self.hd)           # default, linear or llama3 frequencies (fp32, CPU)
        self.windows = sliding_windows(cfg)                   # key window of each layer, 0 = full causal attention
        self.Nq, self.Nkv = self.nh * self.hd, self.nkv * self.hd
        self.Nqkv = self.Nq + 2 * self.Nkv
        self.r = 8
        self.Ra = 2 * self.r if lora else 0
        # headless checkpoints (AutoModel: embed_tokens.*, layers.*, norm.*) are read under the model.-prefixed names
        self.headless = not any(k.startswith("model.") for k in state_dict)
        sd = _with_prefix(state_dict) if self.headless else state_dict
        if self.nf4 is not None:
            g = lambda k, dt: sd[k].to(device=self.dev, dtype=torch.float16).to(dt).contiguous()
        else:
            g = lambda k, dt: sd[k].to(device=self.dev, dtype=dt).contiguous()
        self.Vp = (self.V + 7) // 8 * 8                       # GEMM N granularity; extra rows are zero and never scored
        self.full: Optional[DenseBank] = None
        self.layers: List[Dict[str, torch.Tensor]] = []
        # frozen-base modes keep the fused gate|up weight in the interleaved layout of the SwiGLU-epilogue GEMM (F % 128 == 0);
        # a fully fine-tuned model keeps HF's [gate; up] order inside its parameter bank (un-fused activation kernel)
        self.fuse_rope = self.hd == 128
        self.gu_il = 128 if (not full and F % 128 == 0) else 0
        if full:
            self._init_full(sd)
        else:
            self._init_frozen(sd, g, lora)
        self._rope_cache: Dict[int, tuple] = {}
        # Llama has no hidden / attention dropout (attention_dropout = 0); only peft's LoRA input dropout (0.05) applies
        self.p_lora = 0.05 if lora else 0.0
        self.drop_seed = 0x11A3AB200 + lora_seed
        self.drop_offset = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self._call = 0
        self.lora: Optional[LoraBank] = None
        if lora:
            outs = {"q_proj": self.Nq, "v_proj": self.Nkv}
            specs = [(f"model.layers.{l}.self_attn.{n}", H, outs[n]) for l in range(self.nl) for n in self.LORA_TARGETS]
            self.lora = LoraBank(specs, r=self.r, alpha=16, dropout=0.05, device=self.dev, seed=lora_seed)
            self.lora_flat = torch.nn.Parameter(self.lora.flat, requires_grad=True)
            self.lora_flat.grad = self.lora.grad
            self.lora.param = self.lora_flat
            self.repack_lora()
        self.eval()                                           # like from_pretrained(): dropout only after .train()

    # ---- what is trainable ---------------------------------------------------------------------------------------
    @property
    def trainable(self) -> bool:
        return self.lora is not None or self.full is not None

    @property
    def anchor(self) -> torch.nn.Parameter:
        return self.lora_flat if self.lora is not None else self.full_flat

    def grad_buffers(self) -> List[torch.Tensor]:
        return [b.grad for b in (self.lora, self.full) if b is not None]

    def banks(self) -> list:
        return [b for b in (self.lora, self.full) if b is not None]

    def zero_grad_buffers(self) -> None:
        if self.lora is not None:
            self.lora.zero_grad()
        if self.full is not None:
            self.full.zero_grad()

    def _param_map(self, has_head: bool):
        m = [("embed", "acc", ["model.embed_tokens.weight"]), ("norm_g", "acc", ["model.norm.weight"])]
        if has_head:
            m.append(("lm_head", "gemm", ["lm_head.weight"]))
        for l in range(self.nl):
            p = f"model.layers.{l}."
            if self.qkv_bias:                                    # biases: "acc" entries (column sums accumulated by atomics)
                m.append((f"L{l}.bqkv", "acc", [p + f"self_attn.{n}_proj.bias" for n in "qkv"]))
            if self.o_bias:
                m.append((f"L{l}.bo", "acc", [p + "self_attn.o_proj.bias"]))
            if self.qk_norm:                                     # q / k norm weights: "acc" entries (the backward kernel's atomics)
                m += [(f"L{l}.qn", "acc", [p + "self_attn.q_norm.weight"]), (f"L{l}.kn", "acc", [p + "self_attn.k_norm.weight"])]
            m += [(f"L{l}.Wqkv", "gemm", [p + f"self_attn.{n}_proj.weight" for n in "qkv"]),
                  (f"L{l}.Wo", "gemm", [p + "self_attn.o_proj.weight"]),
                  (f"L{l}.Wgu", "gemm", [p + "mlp.gate_proj.weight", p + "mlp.up_proj.weight"]),
                  (f"L{l}.Wd", "gemm", [p + "mlp.down_proj.weight"]),
                  (f"L{l}.g1", "acc", [p + "input_layernorm.weight"]), (f"L{l}.g2", "acc", [p + "post_attention_layernorm.weight"])]
        return m

    def _init_full(self, sd) -> None:
        has_head = "lm_head.weight" in sd
        if not has_head and self.Vp != self.V:
            raise NotImplementedError("full fine-tuning with tied embeddings needs vocab_size % 8 == 0")
        pm = self._param_map(has_head)
        self._rows = {key: [(n, int(sd[n].shape[0])) for n in names] for key, _, names in pm}
        specs = []
        for key, kind, names in pm:
            rows = sum(r for _, r in self._rows[key])
            if key == "lm_head":
                rows = self.Vp                                                   # zero rows up to the GEMM granularity
            specs.append((key, (rows,) + tuple(sd[names[0]].shape[1:]), kind))
        bank = DenseBank(specs, self.dev)
        for key, _, names in pm:
            dst, r = bank.w32(key), 0
            for n in names:
                t = sd[n]
                dst[r:r + t.shape[0]].copy_(t.to(self.dev, f32))
                r += t.shape[0]
        bank.sync_shadow()
        self.full = bank
        self.full_flat = torch.nn.Parameter(bank.p32, requires_grad=True)
        self.full_flat.grad = bank.g32
        self.full_flat._dalm_bank = bank
        self.embed, self.norm_g = bank.w16("embed"), bank.w32("norm_g")
        self.tied = not has_head
        self.lm_head = bank.w16("lm_head") if has_head else self.embed
        for l in range(self.nl):
            k = lambda n: f"L{l}.{n}"
            self.layers.append({"Wqkv_aug": bank.w16(k("Wqkv")), "Wo": bank.w16(k("Wo")), "Wgu": bank.w16(k("Wgu")),
                                "Wd": bank.w16(k("Wd")), "g1": bank.w32(k("g1")), "g2": bank.w32(k("g2")),
                                "bqkv": bank.w32(k("bqkv")) if self.qkv_bias else None,
                                "bo": bank.w32(k("bo")) if self.o_bias else None,
                                "qn": bank.w32(k("qn")) if self.qk_norm else None,
                                "kn": bank.w32(k("kn")) if self.qk_norm else None})

    def hf_state_dict(self) -> Dict[str, torch.Tensor]:
        """fp32 CPU tensors under HF LlamaForCausalLM names (save_pretrained of a fully fine-tuned decoder), or under the
        unprefixed names of a headless checkpoint when the decoder was loaded from one"""
        if self.full is None:
            raise RuntimeError("hf_state_dict: only fully fine-tuned models own their weights (PEFT mode saves adapters)")
        out = {}
        for key, parts in self._rows.items():
            w, r = self.full.w32(key), 0
            for name, rows in parts:
                out[name[len("model."):] if self.headless else name] = w[r:r + rows].detach().cpu().clone()
                r += rows
        return out

    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        if not any(k.startswith("model.") for k in sd):
            sd = _with_prefix(sd)
        for key, parts in self._rows.items():
            w, r = self.full.w32(key), 0
            for name, rows in parts:
                w[r:r + rows].copy_(sd[name].to(self.dev, f32))
                r += rows
        self.full.sync_shadow()

    def enable_lora(self, lora_seed: int = 1) -> None:
        """frozen (inference-built) decoder -> adapter-carrying one, see BertEncoder.enable_lora"""
        if self.lora is not None:
            return
        if self.full is not None:
            raise RuntimeError("enable_lora: this decoder is being fully fine-tuned; adapters attach to frozen bases only")
        H, r = self.H, self.r
        self.Ra = 2 * r
        for li, W in enumerate(self.layers):
            if self.nf4 is not None:                             # 4-bit storage: give the packed q|k|v weight its LoRA tail block
                packed, absmax, rows, cols = self.nf4.q[(li, "Wqkv_aug")]
                self.nf4.tails[(li, "Wqkv_aug")] = torch.zeros(rows, self.Ra, dtype=bf16, device=self.dev)
                if self.nf4.slots["Wqkv_aug"].shape[1] < cols + 64:
                    self.nf4.slots["Wqkv_aug"] = torch.empty(rows, cols + 64, dtype=bf16, device=self.dev)
                W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
                W["Bblk"] = torch.zeros(64, self.Nqkv, dtype=bf16, device=self.dev)
                continue
            old, oldT = W["Wqkv_aug"], W["WqkvT_aug"]
            W["Wqkv_aug"] = _aug_buf(self.Nqkv, H, self.Ra, self.dev, zero=True)
            W["Wqkv_aug"][:, :H] = old[:, :H]
            W["WqkvT_aug"] = _aug_buf(H, self.Nqkv, self.Ra, self.dev, zero=True)
            W["WqkvT_aug"][:, :self.Nqkv] = oldT[:, :self.Nqkv]
            W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
            W["Bblk"] = torch.zeros(64, self.Nqkv, dtype=bf16, device=self.dev)
        outs = {"q_proj": self.Nq, "v_proj": self.Nkv}
        specs = [(f"model.layers.{l}.self_attn.{n}", H, outs[n]) for l in range(self.nl) for n in self.LORA_TARGETS]
        self.lora = LoraBank(specs, r=r, alpha=16, dropout=0.05, device=self.dev, seed=lora_seed)
        self.lora_flat = torch.nn.Parameter(self.lora.flat, requires_grad=True)
        self.lora_flat.grad = self.lora.grad
        self.lora.param = self.lora_flat
        self.p_lora = 0.05
        self._pack_tab = None
        self.repack_lora()

    def _dgrad(self, dy: torch.Tensor, W: Dict[str, torch.Tensor], name: str) -> torch.Tensor:
        if self.full is not None or self.nf4 is not None:        # W[out,in] read MN-major: no transposed copy in these modes
            return ops.gemm(dy, W[name], layout=1)
        return ops.gemm(dy, W[name + "T"])

    def _init_frozen(self, sd, g, lora: bool) -> None:
        H = self.H
        self.embed = g("model.embed_tokens.weight", bf16)
        self.norm_g = g("model.norm.weight", f32)
        lm = g("lm_head.weight", bf16) if "lm_head.weight" in sd else self.embed      # tied / headless (AutoModel) checkpoints
        if self.Vp != self.V:
            lm = torch.cat([lm, torch.zeros(self.Vp - self.V, H, dtype=bf16, device=self.dev)], 0)
        self.lm_head = lm
        self.lm_headT = self.lm_head.t().contiguous()
        H_, Ra = H, self.Ra
        for l in range(self.nl):
            p = f"model.layers.{l}."
            if self.nf4 is not None:
                self.layers.append(self._init_layer_nf4(sd, l, g, lora))
                continue
            W = {}
            wqkv = torch.cat([g(p + "self_attn.q_proj.weight", bf16), g(p + "self_attn.k_proj.weight", bf16),
                              g(p + "self_attn.v_proj.weight", bf16)], 0)
            W["Wqkv_aug"] = _aug_buf(self.Nqkv, H_, Ra, self.dev, zero=True)
            W["Wqkv_aug"][:, :H_] = wqkv
            W["WqkvT_aug"] = _aug_buf(H_, self.Nqkv, Ra, self.dev, zero=True)
            W["WqkvT_aug"][:, :self.Nqkv] = wqkv.t()
            del wqkv
            if lora:
                W["A_stack"] = torch.zeros(64, H_, dtype=bf16, device=self.dev)
                W["Bblk"] = torch.zeros(64, self.Nqkv, dtype=bf16, device=self.dev)
            W["Wo"] = g(p + "self_attn.o_proj.weight", bf16)
            W["WoT"] = W["Wo"].t().contiguous()
            if self.sparse[l]:
                W["moe"] = self._moe_weights(sd, p)
            else:
                if self.gu_il:   # gate / up rows interleaved in 128-feature blocks: SiLU(gate)*up is fused into this GEMM's epilogue
                    W["Wgu"] = ops.interleave_gate_up(g(p + "mlp.gate_proj.weight", bf16), g(p + "mlp.up_proj.weight", bf16), self.gu_il)
                else:
                    W["Wgu"] = torch.cat([g(p + "mlp.gate_proj.weight", bf16), g(p + "mlp.up_proj.weight", bf16)], 0)
                W["WguT"] = W["Wgu"].t().contiguous()
                W["Wd"] = g(p + "mlp.down_proj.weight", bf16)
                W["WdT"] = W["Wd"].t().contiguous()
            W["g1"] = g(p + "input_layernorm.weight", f32)
            W["g2"] = g(p + "post_attention_layernorm.weight", f32)
            self._frozen_biases(W, p, g)
            self.layers.append(W)

    def _moe_weights(self, sd, p: str) -> moe.MoeWeights:
        """a sparse layer's router and experts, from the hub layout (mlp.experts.{e}.{gate,up,down}_proj.weight) or from
        transformers 5's fused one (mlp.experts.gate_up_proj [E, 2I, H]: gate rows then up rows; mlp.experts.down_proj
        [E, H, I])"""
        cfg = self.cfg
        E, I = int(cfg["num_experts"]), int(cfg["moe_intermediate_size"])
        if p + "mlp.experts.gate_up_proj" in sd:
            gu, down = sd[p + "mlp.experts.gate_up_proj"], sd[p + "mlp.experts.down_proj"]
            gate_proj, up_proj = gu[:, :I], gu[:, I:]
        else:
            ex = lambda e, n: sd[p + f"mlp.experts.{e}.{n}_proj.weight"]
            gate_proj = [ex(e, "gate") for e in range(E)]
            up_proj = [ex(e, "up") for e in range(E)]
            down = torch.stack([ex(e, "down").to(bf16) for e in range(E)])
        return moe.pack_experts(sd[p + "mlp.gate.weight"], gate_proj, up_proj, down, int(cfg["num_experts_per_tok"]),
                                bool(cfg.get("norm_topk_prob", False)), self.dev)

    def _init_layer_nf4(self, sd, l: int, g, lora: bool):
        """one layer in 4-bit storage: q|k|v, o, gate|up (interleaved like the resident mode), down as NF4 codes; blocks of 64
        run along the input features, so fusing / interleaving ROWS leaves every block (and its absmax) what bitsandbytes
        computes for the separate nn.Linear weights"""
        from .nf4store import QuantLayer
        p = f"model.layers.{l}."
        raw = lambda k: sd[k].to(device=self.dev, dtype=f32)
        W = QuantLayer(self.nf4, l)
        self.nf4.put(l, "Wqkv_aug", torch.cat([raw(p + f"self_attn.{n}_proj.weight") for n in "qkv"], 0), tail_cols=self.Ra)
        self.nf4.put(l, "Wo", raw(p + "self_attn.o_proj.weight"))
        gate, up = raw(p + "mlp.gate_proj.weight"), raw(p + "mlp.up_proj.weight")
        self.nf4.put(l, "Wgu", ops.interleave_gate_up(gate, up, self.gu_il) if self.gu_il else torch.cat([gate, up], 0))
        self.nf4.put(l, "Wd", raw(p + "mlp.down_proj.weight"))
        if lora:
            W["A_stack"] = torch.zeros(64, self.H, dtype=bf16, device=self.dev)
            W["Bblk"] = torch.zeros(64, self.Nqkv, dtype=bf16, device=self.dev)
        W["g1"] = g(p + "input_layernorm.weight", f32)
        W["g2"] = g(p + "post_attention_layernorm.weight", f32)
        self._frozen_biases(W, p, g)
        return W

    def _frozen_biases(self, W, p: str, g) -> None:
        """frozen / LoRA modes: the attention biases (and Qwen3's q / k norm weights) are forward-only fp32 vectors (under use_bnb they take the fp16 cast of every
        non-Linear-weight tensor, never the NF4 round trip)"""
        W["bqkv"] = torch.cat([g(p + f"self_attn.{n}_proj.bias", f32) for n in "qkv"]) if self.qkv_bias else None
        W["bo"] = g(p + "self_attn.o_proj.bias", f32) if self.o_bias else None
        # Qwen3's q / k norm weights: forward-only fp32 vectors here too (use_bnb: the fp16 cast, as every norm weight)
        W["qn"] = g(p + "self_attn.q_norm.weight", f32) if self.qk_norm else None
        W["kn"] = g(p + "self_attn.k_norm.weight", f32) if self.qk_norm else None

    def _drop(self, training: bool, call: int, layer: int):
        if not training or self.p_lora <= 0.0:
            return None
        return ops.Drop(self.p_lora, self.drop_seed, (call << 24) | (layer << 8) | 3, self.drop_offset)

    # column offset / width of each LoRA target inside the fused qkv output
    def _target_cols(self, n: str):
        return (0, self.Nq) if n == "q_proj" else (self.Nq + self.Nkv, self.Nkv)

    def _pack_entries(self):
        H, r, s = self.H, self.r, self.lora.scale
        for l, W in enumerate(self.layers):
            for j, n in enumerate(self.LORA_TARGETS):
                name = f"model.layers.{l}.self_attn.{n}"
                A, B = self.lora.A[name], self.lora.B[name]             # [r,H], [out,r]
                c0, w = self._target_cols(n)
                if self.nf4 is not None:                                 # 4-bit storage: the LoRA columns live in the layer's tail block
                    yield (B, r, 1, self.nf4.tail(l, "Wqkv_aug")[c0:c0 + w, j * r:], w, r, s)
                else:
                    yield (B, r, 1, W["Wqkv_aug"][c0:c0 + w, H + j * r:], w, r, s)
                    yield (A, 1, H, W["WqkvT_aug"][:, self.Nqkv + j * r:], H, r, 1.0)
                yield (A, H, 1, W["A_stack"][j * r:(j + 1) * r], r, H, 1.0)
                yield (B, 1, r, W["Bblk"][j * r:(j + 1) * r, c0:], r, w, s)

    def repack_lora(self) -> None:
        if self.lora is None:
            return
        if getattr(self, "_pack_tab", None) is None:
            self._pack_tab = ops.build_pack_table(list(self._pack_entries()), self.dev)
        ops.pack_table_(self._pack_tab)

    def _rope(self, L: int):
        """fp32 cos / sin tables [L, hd/2] at positions 0..L-1: what every RoPE kernel reads (the QKV epilogue, the row kernels,
        decode); the frequency scaling of the config lives in `inv_freq` only"""
        if L not in self._rope_cache:
            fr = torch.outer(torch.arange(L, dtype=torch.float32), self.inv_freq)                      # [L, hd/2]
            self._rope_cache[L] = (fr.cos().to(self.dev).contiguous(), fr.sin().to(self.dev).contiguous())
        return self._rope_cache[L]

    # ------------------------------------------------------------------------------------------------------------
    def forward_logits(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True):
        """ids, mask int64 [B,L] -> (logits bf16 [B,L,V], ctx)"""
        B, L = ids.shape
        ctx = self._forward_body(ids, mask, save)
        logits = ops.gemm(ctx.hf, self.lm_head)                                   # bf16 [M,Vp]
        return logits.view(B, L, self.Vp)[:, :, :self.V], ctx

    def forward_final(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True) -> _Ctx:
        """the decoder up to the final RMSNorm (ctx.hf bf16 [M,H]) — the fused step's forward: the lm_head runs inside
        `head_loss`, chunk by chunk, and no [B,L,V] logits tensor is ever written"""
        return self._forward_body(ids, mask, save)

    def head_loss(self, ctx: _Ctx, ids: torch.Tensor, mask: torch.Tensor, nsum: torch.Tensor, need_grad: bool = True,
                  grad_out: float = 1.0):
        """lm_head + marginalised-NLL token terms (+ the head's dgrad / wgrad) over row chunks (engine/head.py; reference
        train_utils.py:113-138 on `generator_model(...).logits`). -> (tok_lp fp32 [B,L], d(hf) bf16 [M,H] or None)"""
        from .head import chunked_head_loss
        need_grad = need_grad and self.trainable
        wgrad = None
        if need_grad and self.full is not None:
            ctx.acc = self.full.begin_backward()
            tgt = self.full.g("embed") if self.tied else self.full.g("lm_head")      # tied head: gradient lands in the embedding table
            acc0 = True if self.tied else ctx.acc
            wgrad = lambda dl, h, first: ops.wgrad_(dl, h, tgt, acc0 if first else True)
        tok_lp, dhf = chunked_head_loss(ctx.hf, self.lm_head, getattr(self, "lm_headT", None) if self.full is None else None, self.V,
                                        ids, mask, nsum, need_grad, grad_out, wgrad)
        if wgrad is not None and not self.tied:
            self.full.bucket_ready("lm_head")                                      # final: all-reduce it under the layers' backward
        return tok_lp, dhf

    def backward_final(self, ctx: _Ctx, dhf: torch.Tensor) -> None:
        """continues `head_loss`'s backward from d(final-norm output) down through the layers"""
        if self.trainable and dhf is not None:
            self._backward_body(ctx, dhf)

    def forward_hidden(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True):
        """last hidden state (after the final RMSNorm) as fp32 [B,L,H] — what `AutoModel(...)(..., output_hidden_states=True)
        .hidden_states[-1]` gives the reference's autoregressive-retriever branch (rag_e2e_base_model.py:84-90)"""
        B, L = ids.shape
        ctx = self._forward_body(ids, mask, save)
        return ctx.hf.float().view(B, L, self.H), ctx

    def backward_hidden(self, ctx: _Ctx, d_hidden: torch.Tensor) -> None:
        """gradient w.r.t. the last hidden state (fp32 [B,L,H]) -> parameter gradients"""
        if not self.trainable:
            return
        if self.full is not None:
            ctx.acc = self.full.begin_backward()
            if not ctx.acc and not self.tied:
                self.full.g("lm_head").zero_()                 # the head is not on this path: its fresh gradient is zero
        self._backward_body(ctx, ops.cast_f32_bf16(d_hidden.reshape(ctx.B * ctx.L, self.H).contiguous()))

    def _forward_body(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True, pos: Optional[torch.Tensor] = None,
                      rope_tables=None, kv_sink=None):
        """pos / rope_tables / kv_sink serve `generate`'s prefill: explicit position ids (int64 [B*L]) into cos / sin tables
        [T, hd/2], and a callback (layer, qkv) that copies the rotated K / V columns into the KV cache"""
        B, L = ids.shape
        M, H, F, Ra = B * L, self.H, self.F, self.Ra
        cos_t, sin_t = self._rope(L) if rope_tables is None else rope_tables
        ctx = _Ctx()
        ctx.B, ctx.L, ctx.mask, ctx.layers = B, L, mask.contiguous(), []
        ctx.ids = ids.contiguous()
        self._call += 1
        ctx.call, ctx.training = self._call, self.training
        x = ops.embed_gather(ids, self.embed)                                    # fp32 residual stream [M,H]
        for li, W in enumerate(self.layers):
            a = _Ctx()
            a.x_in = x
            a.h1_aug = _aug_buf(M, H, Ra, self.dev)
            _, a.rstd1 = ops.rmsnorm_fwd(x, W["g1"], self.eps, h=a.h1_aug[:, :H])
            if Ra:
                ops.skinny_gemm(a.h1_aug[:, :H], W["A_stack"], a.h1_aug[:, H:], K=H, R=Ra,   # u = dropout(h1) A^T [M,2r]
                                dropx=self._drop(ctx.training, ctx.call, li))
            rope_cols = (self.nh + self.nkv) * self.hd
            a.pre = a.qk_rstd = None
            if self.qk_norm and save and self.trainable:                         # what the q/k norm backward reads
                a.pre = torch.empty(M, rope_cols, dtype=bf16, device=self.dev)
                a.qk_rstd = torch.empty(M, self.nh + self.nkv, dtype=f32, device=self.dev)
            if pos is None and self.fuse_rope and rope_cols % 256 == 0:
                norm = dict(q_norm=W["qn"], k_norm=W["kn"], nq_heads=self.nh, eps=self.eps, pre_out=a.pre,
                            rstd_out=a.qk_rstd) if self.qk_norm else {}
                a.qkv = ops.gemm_rope(a.h1_aug, W["Wqkv_aug"], cos_t, sin_t, L, rope_cols,   # QKV (+LoRA, + bias) with (q/k norm
                                      bias=W["bqkv"], **norm)                                # and) RoPE in the epilogue
            else:
                a.qkv = ops.gemm(a.h1_aug, W["Wqkv_aug"], bias=W["bqkv"])        # [M, Nq+2Nkv]
                if self.qk_norm:
                    ops.qk_norm_rope_(a.qkv, self.nh + self.nkv, self.nh, W["qn"], W["kn"], self.eps, cos_t, sin_t,
                                      L=L if pos is None else 0, pos=pos, pre=a.pre, rstd=a.qk_rstd)
                elif pos is None:
                    ops.rope_(a.qkv, 0, self.nh + self.nkv, self.hd, cos_t, sin_t, L)    # q heads then k heads are adjacent
                else:
                    ops.rope_pos_(a.qkv, 0, self.nh + self.nkv, self.hd, cos_t, sin_t, pos)
            if kv_sink is not None:
                kv_sink(li, a.qkv)
            a.att, a.lse = ops.attention_auto_fwd(a.qkv[:, :self.Nq], a.qkv[:, self.Nq:self.Nq + self.Nkv],
                                                  a.qkv[:, self.Nq + self.Nkv:], ctx.mask, B, L, self.nh, self.nkv, self.hd, causal=True,
                                                  window=self.windows[li])
            a.x_mid = ops.gemm(a.att, W["Wo"], out_dtype=f32, resid=x, bias=W["bo"])
            a.h2, a.rstd2 = ops.rmsnorm_fwd(a.x_mid, W["g2"], self.eps)
            if "moe" in W:
                x, a.moe = moe.forward(a.h2, W["moe"], resid=a.x_mid)
                if save:
                    ctx.layers.append(a)
                continue
            if self.gu_il:
                a.gu, a.act = ops.gemm_swiglu(a.h2, W["Wgu"])                     # [M,2F] (interleaved) + silu(gate)*up [M,F]: one launch
            else:
                a.gu = ops.gemm(a.h2, W["Wgu"])                                   # [M,2F]
                a.act = ops.swiglu_fwd(a.gu, F)
            x = ops.gemm(a.act, W["Wd"], out_dtype=f32, resid=a.x_mid)
            if save:
                ctx.layers.append(a)
        ctx.x_final = x
        ctx.hf, ctx.rstdf = ops.rmsnorm_fwd(x, self.norm_g, self.eps)
        return ctx

    # ------------------------------------------------------------------------------------------------------------
    # greedy decoding with a KV cache (evaluation: reference dalm/eval/eval_rag.py:126-140 calls HF `model.generate`)
    # ------------------------------------------------------------------------------------------------------------
    def _decode_step(self, ids: torch.Tensor, pos: torch.Tensor, caches, kmask: torch.Tensor, cur, tables) -> torch.Tensor:
        """one token per sequence: ids / pos int64 [B] (device) -> logits bf16 [B, Vp]; appends K / V at cache column `cur` (int, or the int32 [B] device tensor of per-row columns: CUDA-graph mode)"""
        B = ids.shape[0]
        H, F, Ra = self.H, self.F, self.Ra
        cos_t, sin_t = tables
        x = ops.embed_gather(ids, self.embed)                                    # fp32 residual stream [B,H]
        for li, W in enumerate(self.layers):
            h1_aug = _aug_buf(B, H, Ra, self.dev)
            ops.rmsnorm_fwd(x, W["g1"], self.eps, h=h1_aug[:, :H])
            if Ra:
                ops.skinny_gemm(h1_aug[:, :H], W["A_stack"], h1_aug[:, H:], K=H, R=Ra)
            qkv = ops.gemm_rows(h1_aug, W["Wqkv_aug"], bias=W["bqkv"])                # [B, Nq+2Nkv]
            if self.qk_norm:
                ops.qk_norm_rope_(qkv, self.nh + self.nkv, self.nh, W["qn"], W["kn"], self.eps, cos_t, sin_t, pos=pos)
            else:
                ops.rope_pos_(qkv, 0, self.nh + self.nkv, self.hd, cos_t, sin_t, pos)
            att = ops.attention_decode(qkv, 0, self.Nq, self.Nq + self.Nkv, caches[li][0], caches[li][1], kmask, cur,
                                       self.nh, self.nkv, self.hd, window=self.windows[li])
            x_mid = ops.gemm_rows(att, W["Wo"], out_dtype=f32, resid=x, bias=W["bo"])
            h2, _ = ops.rmsnorm_fwd(x_mid, W["g2"], self.eps)
            if "moe" in W:
                x, _ = moe.forward(h2, W["moe"], resid=x_mid)
                continue
            act = ops.swiglu_fwd(ops.gemm_rows(h2, W["Wgu"]), F, interleave=self.gu_il)
            x = ops.gemm_rows(act, W["Wd"], out_dtype=f32, resid=x_mid)
        hf, _ = ops.rmsnorm_fwd(x, self.norm_g, self.eps)
        return ops.gemm_rows(hf, self.lm_head)

    def _prefill_last(self, ids, mask, pos, tables, sink) -> torch.Tensor:
        """prompt pass of `generate`: rotated K / V of every layer go to `sink`; returns the last column's final hidden
        state (bf16 [B,H]) — only that column is scored"""
        B, L0 = ids.shape
        ctx = self._forward_body(ids, mask, save=False, pos=pos, rope_tables=tables, kv_sink=sink)
        return ctx.hf.view(B, L0, self.H)[:, -1].contiguous()

    def kv_columns(self):
        """(first K column, first V column, width) of the rotated keys / values inside a layer's qkv buffer"""
        return self.Nq, self.Nq + self.Nkv, self.Nkv

    def generate(self, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
        """HF `generate`: greedy search or sampling, as the checkpoint's generation config and the call select; see
        engine/decoding.py"""
        from .decoding import generate
        return generate(self, input_ids, attention_mask, **kw)

    # ------------------------------------------------------------------------------------------------------------
    def backward_logits(self, ctx: _Ctx, dlogits: torch.Tensor) -> None:
        """dlogits bf16 [B,L,V]; accumulates LoRA gradients (PEFT mode) or all parameter gradients (full mode)."""
        if not self.trainable:
            return
        B, L = ctx.B, ctx.L
        M, H, F, Ra, r = B * L, self.H, self.F, self.Ra, self.r
        cos_t, sin_t = self._rope(L)
        if dlogits.stride(-1) != 1 or dlogits.stride(-2) != self.Vp:             # a caller-made copy: re-pad to the GEMM layout
            pad = torch.zeros(B, L, self.Vp, dtype=bf16, device=self.dev)
            pad[:, :, :self.V] = dlogits
            dlogits = pad
        dl2 = torch.as_strided(dlogits, (M, self.Vp), (self.Vp, 1), dlogits.storage_offset())
        if self.full is None:
            self._backward_body(ctx, ops.gemm(dl2, self.lm_headT))                 # dhf [M,H]
            return
        ctx.acc = self.full.begin_backward()
        if self.tied:                                                              # head gradient lands in the embedding table
            ops.wgrad_(dl2, ctx.hf, self.full.g("embed"), True)
        else:
            ops.wgrad_(dl2, ctx.hf, self.full.g("lm_head"), ctx.acc)
            self.full.bucket_ready("lm_head")                                      # final: all-reduce it under the layers' backward
        self._backward_body(ctx, ops.gemm(dl2, self.lm_head, layout=1))

    def _backward_body(self, ctx: _Ctx, dhf: torch.Tensor) -> None:
        """from the gradient of the final-norm output (bf16 [M,H]) down through the layers"""
        B, L = ctx.B, ctx.L
        M, H, F, Ra, r = B * L, self.H, self.F, self.Ra, self.r
        cos_t, sin_t = self._rope(L)
        bank = self.full
        acc = getattr(ctx, "acc", False)
        G = (lambda l, n: bank.g(f"L{l}.{n}")) if bank is not None else None
        if bank is not None:
            ops.col_reduce_(dy_bf16=dhf, z=ctx.x_final, rstd=ctx.rstdf, out_prod=bank.g("norm_g"))
        dx32, dx16 = ops.rmsnorm_bwd(ctx.x_final, self.norm_g, ctx.rstdf, dhf)
        for l in range(self.nl - 1, -1, -1):
            W, a = self.layers[l], ctx.layers[l]
            if "moe" in W:                                                         # experts and router frozen: input gradient only
                dh2 = ops.cast_f32_bf16(moe.backward(dx16, a.moe, W["moe"]))
            else:
                if bank is not None:
                    ops.wgrad_(dx16, a.act, G(l, "Wd"), acc)
                dact = self._dgrad(dx16, W, "Wd")                                  # [M,F]
                ops.swiglu_bwd_(a.gu, dact, F, interleave=self.gu_il)              # gu <- [dgate | dup] (same layout as gu)
                if bank is not None:
                    ops.wgrad_(a.gu, a.h2, G(l, "Wgu"), acc)
                dh2 = self._dgrad(a.gu, W, "Wgu")                                  # [M,H]
            if bank is not None:
                ops.col_reduce_(dy_bf16=dh2, z=a.x_mid, rstd=a.rstd2, out_prod=G(l, "g2"))
            dmid32, dmid16 = ops.rmsnorm_bwd(a.x_mid, W["g2"], a.rstd2, dh2, dres_in=dx32)
            if bank is not None:
                ops.wgrad_(dmid16, a.att, G(l, "Wo"), acc)
                if self.o_bias:                                                    # d bo = column sums of d(o_proj output)
                    ops.col_reduce_(dy_f32=dmid32, out_sum=G(l, "bo"))
            datt = self._dgrad(dmid16, W, "Wo")                                    # [M,Nq]
            dqkv = _aug_buf(M, self.Nqkv, Ra, self.dev)
            ops.attention_auto_bwd(a.qkv[:, :self.Nq], a.qkv[:, self.Nq:self.Nq + self.Nkv], a.qkv[:, self.Nq + self.Nkv:],
                     ctx.mask, a.att, a.lse, datt, B, L, self.nh, self.nkv, self.hd, causal=True,
                     dq=dqkv[:, :self.Nq], dk=dqkv[:, self.Nq:self.Nq + self.Nkv],
                     dv=dqkv[:, self.Nq + self.Nkv:self.Nqkv], window=self.windows[l])
            if self.qk_norm:                                                       # un-rotate, then the q/k RMSNorm backward
                ops.qk_norm_rope_bwd_(dqkv, self.nh + self.nkv, self.nh, W["qn"], W["kn"], cos_t, sin_t, L, a.pre, a.qk_rstd,
                                      dw_q=G(l, "qn") if bank is not None else None, dw_k=G(l, "kn") if bank is not None else None)
            else:
                ops.rope_(dqkv, 0, self.nh + self.nkv, self.hd, cos_t, sin_t, L, backward=True)
            if bank is not None:
                ops.wgrad_(dqkv, a.h1_aug[:, :H], G(l, "Wqkv"), acc)
                if self.qkv_bias:                                                  # d bqkv = column sums of d(pre-RoPE qkv)
                    ops.col_reduce_(dy_bf16=dqkv, out_sum=G(l, "bqkv"))
                dh1 = ops.gemm(dqkv, W["Wqkv_aug"], layout=1)
                ops.col_reduce_(dy_bf16=dh1, z=a.x_in, rstd=a.rstd1, out_prod=G(l, "g1"))
                dx32, dx16 = ops.rmsnorm_bwd(a.x_in, W["g1"], a.rstd1, dh1, dres_in=dmid32)
                bank.bucket_ready(f"L{l}.")                                        # this layer's four weight gradients are final
                continue
            names = [f"model.layers.{l}.self_attn.{n}" for n in self.LORA_TARGETS]
            for j, n in enumerate(self.LORA_TARGETS):
                c0, w = self._target_cols(n)
                ops.skinny_gemm(dqkv[:, c0:c0 + w], W["Bblk"][j * r:(j + 1) * r, c0:c0 + w], dqkv[:, self.Nqkv + j * r:], K=w, R=r)
            # dA_q, dA_v in one pass over h1 (the 16-row MMA tile is exactly the two rank-8 adapters)
            xdrop = self._drop(ctx.training, ctx.call, l)
            ops.lora_wgrad_(a.h1_aug[:, :H], dqkv[:, self.Nqkv:], self.lora.gA[names[0]], H, 1, H, 2 * r, 1.0,
                            out1=self.lora.gA[names[1]], dropx=xdrop)
            for j, n in enumerate(self.LORA_TARGETS):
                c0, w = self._target_cols(n)
                ops.lora_wgrad_(dqkv[:, c0:c0 + w], a.h1_aug[:, H + j * r:], self.lora.gB[names[j]], 1, r, w, r, self.lora.scale)
            if l == 0:
                break                                                              # embeddings frozen
            if self.nf4 is not None:                                               # base path against the expanded W[out,in] + (g A)
                dh1 = ops.gemm(dqkv[:, :self.Nqkv], W["Wqkv_aug"][:, :H], layout=1)
                ops.lora_dx_(dh1, dqkv[:, self.Nqkv:], W["A_stack"], K=H, R=Ra, drop=xdrop)
            elif xdrop is None:
                dh1 = ops.gemm(dqkv, W["WqkvT_aug"])                               # [M,H], LoRA's A-path folded into K
            else:
                dh1 = ops.gemm(dqkv[:, :self.Nqkv], W["WqkvT_aug"][:, :self.Nqkv])
                ops.lora_dx_(dh1, dqkv[:, self.Nqkv:], W["A_stack"], K=H, R=Ra, drop=xdrop)
            dx32, dx16 = ops.rmsnorm_bwd(a.x_in, W["g1"], a.rstd1, dh1, dres_in=dmid32)
        if bank is not None:
            ops.embed_scatter_add_(dx32, ctx.ids, bank.g("embed"))                # embed_tokens
            bank.end_backward()
