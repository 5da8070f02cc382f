"""BERT encoder (bge-small / bge-large shapes) forward + backward as a launch sequence over the C-ABI kernels. The same class
serves RoBERTa / XLM-RoBERTa encoders (multilingual-e5, bge-m3): identical layers and parameter names; their embeddings take
positions from the ids (pad + running count of non-pad tokens, HF create_position_ids_from_input_ids) instead of the column,
and the padding_idx rows of the word and position tables receive no gradient.

Mirrors what `self.retriever_model(input_ids, attention_mask)[0]` computes in the reference
(dalm/models/rag_e2e_base_model.py:93, dalm/models/retriever_only_base_model.py:58) through HF BertModel:
embeddings(word+pos+type0) -> LN -> N x [QKV(+LoRA) -> masked softmax attention -> out-proj + residual -> LN ->
FFN(GELU erf) + residual -> LN], eps 1e-12, token_type_ids = 0 (the reference calls the model positionally).

HBM layout (per layer, bf16 unless noted):
  Wqkv_aug [3H, H+Ra]   rows q|k|v of the fused projection; the last Ra=3r columns hold (alpha/r)*B_j so that LoRA's
                        up-projection is part of the same wgmma GEMM (A operand = [x | x A^T])
  WqkvT_aug [H, 3H+Ra]  resident transpose for dgrad; last Ra columns hold A_j^T
  A_stack [64, H]       LoRA down-projection operand (rows j*r..), zero padded to one 64-row TMA box
  Bblk [64, 3H]         block-diagonal (alpha/r)*B_j^T: g = dQKV . Bblk^T gives all LoRA mid-gradients in one GEMM
  Wo, WoT [H,H]; Wi [F,H], WiT [H,F]; Wo2 [H,F], Wo2T [F,H]; biases / LN params fp32
Activations: residual path fp32, GEMM operands bf16.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import ops
from . import params
from .dense import DenseBank
from .lora import LoraBank

bf16, f32 = torch.bfloat16, torch.float32


def _hf_names(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """checkpoint names relative to the encoder: the `bert.` / `roberta.` prefix of *ForMaskedLM-style checkpoints stripped,
    their masked-LM head (`lm_head.*`) left out"""
    out = {}
    for k, v in sd.items():
        for pre in ("bert.", "roberta."):
            if k.startswith(pre):
                k = k[len(pre):]
                break
        if not k.startswith("lm_head."):
            out[k] = v
    return out


def _aug_buf(rows: int, cols: int, ra: int, device, zero: bool = False) -> torch.Tensor:
    """[rows, cols+ra] bf16 view whose row stride is padded to cols+64 when ra > 0, so that every row starts on a
    128-byte boundary (TMA 128B-swizzled boxes then touch aligned lines; measured +20 % on the K-augmented GEMMs)"""
    ld = cols + (64 if ra else 0)
    base = (torch.zeros if zero else torch.empty)(rows, ld, dtype=bf16, device=device)
    return base[:, :cols + ra]


class _Ctx:
    """activations of one forward call kept for its backward"""
    pass


class BertEncoder(torch.nn.Module):
    LORA_TARGETS = ("query", "key", "value")          # reference rag_e2e_base_model.py:66-68

    def __init__(self, cfg: Dict, state_dict: Dict[str, torch.Tensor], device="cuda", lora: bool = False,
                 lora_seed: int = 0, full: bool = False, nf4_storage: bool = False):
        """lora: PEFT mode (base frozen, rank-8 adapters on query/key/value). full: every parameter trainable (the
        reference's behaviour without --use-peft): weights live in a DenseBank, no transposed copies are kept.
        nf4_storage: use_bnb with 4-bit storage (engine/nf4store.py) - `state_dict` holds the ORIGINAL checkpoint values."""
        super().__init__()
        if lora and full:
            raise ValueError("lora and full fine-tuning are mutually exclusive for one model")
        if nf4_storage and full:
            raise ValueError("4-bit base weights cannot be fully fine-tuned")
        self.nf4 = None
        if nf4_storage:
            from .nf4store import Nf4Store
            self.nf4 = Nf4Store(device)
        self.cfg = cfg
        self.H = H = cfg["hidden_size"]
        self.F = F = cfg["intermediate_size"]
        self.nl = cfg["num_hidden_layers"]
        self.nh = cfg["num_attention_heads"]
        self.hd = H // self.nh
        self.V = cfg["vocab_size"]
        self.eps = float(cfg.get("layer_norm_eps", 1e-12))
        self.dev = torch.device(device)
        self.roberta = cfg.get("model_type") in ("roberta", "xlm-roberta")
        if self.roberta:
            params.check_roberta(cfg)
            self.pad = int(cfg.get("pad_token_id", 1))
            self.max_len = params.roberta_max_len(cfg)
        if self.hd not in (32, 64, 128):
            raise NotImplementedError(f"head_dim {self.hd} not supported by the attention kernels")
        self.r = 8
        self.Ra = 3 * self.r if lora else 0
        sd = _hf_names(state_dict)
        if self.nf4 is not None:                              # everything that is not an nn.Linear weight: transformers' fp16 cast
            g = lambda k, dt: sd[k].to(device=self.dev, dtype=torch.float16).to(dt).contiguous()
        else:
            g = lambda k, dt: sd[k].to(device=self.dev, dtype=dt).contiguous()
        self.full: Optional[DenseBank] = None
        self.layers: List[Dict[str, torch.Tensor]] = []
        if full:
            self._init_full(sd)
        else:
            self._init_frozen(sd, g, lora)
        self.pooler = {k: v for k, v in sd.items() if k.startswith("pooler.")}   # carried for save_pretrained only
        # dropout (active only in train() mode, like the HF module the reference wraps; from_pretrained returns eval())
        self.p_hidden = float(cfg.get("hidden_dropout_prob", 0.1))
        self.p_attn = float(cfg.get("attention_probs_dropout_prob", 0.1))
        self.p_lora = 0.05 if lora else 0.0                   # reference rag_e2e_base_model.py:151 (lora_dropout)
        self.drop_seed = 0x5DA1B200 + lora_seed
        self.drop_offset = torch.zeros(1, dtype=torch.int64, device=self.dev)      # bumped once per (graphed) step
        self._call = 0
        self.lora: Optional[LoraBank] = None
        if lora:
            specs = [(f"encoder.layer.{l}.attention.self.{n}", H, H) for l in range(self.nl) for n in self.LORA_TARGETS]
            self.lora = LoraBank(specs, r=self.r, alpha=16, dropout=0.05, device=self.dev, seed=lora_seed)
            self.lora_flat = torch.nn.Parameter(self.lora.flat, requires_grad=True)
            self.lora_flat.grad = self.lora.grad
            self.lora.param = self.lora_flat
            self.repack_lora()
        self.eval()

    # ---- what is trainable ---------------------------------------------------------------------------------------
    @property
    def trainable(self) -> bool:
        return self.lora is not None or self.full is not None

    @property
    def anchor(self) -> torch.nn.Parameter:
        """the flat parameter that ties engine outputs to the autograd graph (bridge.py)"""
        return self.lora_flat if self.lora is not None else self.full_flat

    def grad_buffers(self) -> List[torch.Tensor]:
        """flat gradient buffers for the data-parallel all-reduce"""
        return [b.grad for b in (self.lora, self.full) if b is not None]

    def banks(self) -> list:
        return [b for b in (self.lora, self.full) if b is not None]

    def zero_grad_buffers(self) -> None:
        if self.lora is not None:
            self.lora.zero_grad()
        if self.full is not None:
            self.full.zero_grad()

    def _param_map(self):
        """engine tensor -> (gradient kind, HF state-dict names whose rows it concatenates)"""
        E = "embeddings."
        m = [("word", "acc", [E + "word_embeddings.weight"]), ("pos", "acc", [E + "position_embeddings.weight"]),
             ("type", "acc", [E + "token_type_embeddings.weight"]), ("emb_g", "acc", [E + "LayerNorm.weight"]),
             ("emb_b", "acc", [E + "LayerNorm.bias"])]
        for l in range(self.nl):
            p = f"encoder.layer.{l}."
            qkv = [p + f"attention.self.{n}" for n in self.LORA_TARGETS]
            m += [(f"L{l}.Wqkv", "gemm", [n + ".weight" for n in qkv]), (f"L{l}.bqkv", "acc", [n + ".bias" for n in qkv]),
                  (f"L{l}.Wo", "gemm", [p + "attention.output.dense.weight"]), (f"L{l}.bo", "acc", [p + "attention.output.dense.bias"]),
                  (f"L{l}.ln1_g", "acc", [p + "attention.output.LayerNorm.weight"]),
                  (f"L{l}.ln1_b", "acc", [p + "attention.output.LayerNorm.bias"]),
                  (f"L{l}.Wi", "gemm", [p + "intermediate.dense.weight"]), (f"L{l}.bi", "acc", [p + "intermediate.dense.bias"]),
                  (f"L{l}.Wo2", "gemm", [p + "output.dense.weight"]), (f"L{l}.bo2", "acc", [p + "output.dense.bias"]),
                  (f"L{l}.ln2_g", "acc", [p + "output.LayerNorm.weight"]), (f"L{l}.ln2_b", "acc", [p + "output.LayerNorm.bias"])]
        return m

    def _init_full(self, sd) -> None:
        pm = self._param_map()
        self._rows = {key: [(n, int(sd[n].shape[0])) for n in names] for key, _, names in pm}
        specs = [(key, (sum(r for _, r in self._rows[key]),) + tuple(sd[names[0]].shape[1:]), kind) for key, kind, names in pm]
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
        self.word, self.pos, self.type0 = bank.w16("word"), bank.w16("pos"), bank.w16("type")[0]
        self.emb_g, self.emb_b = bank.w32("emb_g"), bank.w32("emb_b")
        for l in range(self.nl):
            k = lambda n: f"L{l}.{n}"
            self.layers.append({"Wqkv_aug": bank.w16(k("Wqkv")), "bqkv": bank.w32(k("bqkv")), "Wo": bank.w16(k("Wo")),
                                "bo": bank.w32(k("bo")), "ln1_g": bank.w32(k("ln1_g")), "ln1_b": bank.w32(k("ln1_b")),
                                "Wi": bank.w16(k("Wi")), "bi": bank.w32(k("bi")), "Wo2": bank.w16(k("Wo2")),
                                "bo2": bank.w32(k("bo2")), "ln2_g": bank.w32(k("ln2_g")), "ln2_b": bank.w32(k("ln2_b"))})

    def hf_state_dict(self) -> Dict[str, torch.Tensor]:
        """fp32 CPU tensors under HF BertModel / XLMRobertaModel names (save_pretrained of a fully fine-tuned encoder); the pooler
        only when the checkpoint had one"""
        if self.full is None:
            raise RuntimeError("hf_state_dict: only fully fine-tuned models own their weights (PEFT mode saves adapters)")
        out = {}
        for key, parts in self._rows.items():
            w, r = self.full.w32(key), 0
            for name, rows in parts:
                out[name] = w[r:r + rows].detach().cpu().clone()
                r += rows
        out.update({k: v.detach().float().cpu() for k, v in self.pooler.items()})
        return out

    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        sd = _hf_names(sd)
        for key, parts in self._rows.items():
            w, r = self.full.w32(key), 0
            for name, rows in parts:
                w[r:r + rows].copy_(sd[name].to(self.dev, f32))
                r += rows
        self.full.sync_shadow()

    def enable_lora(self, lora_seed: int = 0) -> None:
        """turn a frozen (inference-built) encoder into an adapter-carrying one — what `PeftModel.from_pretrained(base, path)`
        does to the reference's wrapper in attach_pre_trained_peft_layers (rag_e2e_base_model.py:113-134). The fused
        projection weights are re-laid-out with the K-augmentation columns; adapter weights are then loaded into the bank."""
        if self.lora is not None:
            return
        if self.full is not None:
            raise RuntimeError("enable_lora: this encoder is being fully fine-tuned; adapters attach to frozen bases only")
        H, r = self.H, self.r
        self.Ra = 3 * r
        for li, W in enumerate(self.layers):
            if self.nf4 is not None:                             # 4-bit storage: give the packed q|k|v weight its LoRA tail block
                packed, absmax, rows, cols = self.nf4.q[(li, "Wqkv_aug")]
                self.nf4.tails[(li, "Wqkv_aug")] = torch.zeros(rows, self.Ra, dtype=bf16, device=self.dev)
                if self.nf4.slots["Wqkv_aug"].shape[1] < cols + 64:
                    self.nf4.slots["Wqkv_aug"] = torch.empty(rows, cols + 64, dtype=bf16, device=self.dev)
                W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
                W["Bblk"] = torch.zeros(64, 3 * H, dtype=bf16, device=self.dev)
                continue
            old, oldT = W["Wqkv_aug"], W["WqkvT_aug"]
            W["Wqkv_aug"] = _aug_buf(3 * H, H, self.Ra, self.dev, zero=True)
            W["Wqkv_aug"][:, :H] = old[:, :H]
            W["WqkvT_aug"] = _aug_buf(H, 3 * H, self.Ra, self.dev, zero=True)
            W["WqkvT_aug"][:, :3 * H] = oldT[:, :3 * H]
            W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
            W["Bblk"] = torch.zeros(64, 3 * H, dtype=bf16, device=self.dev)
        specs = [(f"encoder.layer.{l}.attention.self.{n}", H, H) for l in range(self.nl) for n in self.LORA_TARGETS]
        self.lora = LoraBank(specs, r=r, alpha=16, dropout=0.05, device=self.dev, seed=lora_seed)
        self.lora_flat = torch.nn.Parameter(self.lora.flat, requires_grad=True)
        self.lora_flat.grad = self.lora.grad
        self.lora.param = self.lora_flat
        self.p_lora = 0.05
        self._pack_tab = None
        self.repack_lora()

    def _dgrad(self, dy: torch.Tensor, W: Dict[str, torch.Tensor], name: str, gelu_pre: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dx = dy W: against the resident transposed copy (frozen base) or W[out,in] itself read MN-major (full mode).
        gelu_pre: the result is a gradient w.r.t. gelu(pre) - multiply by gelu'(pre) in the epilogue (-> gradient w.r.t. pre)"""
        kw = dict(act=2, resid=gelu_pre) if gelu_pre is not None else {}
        if self.full is not None or self.nf4 is not None:
            return ops.gemm(dy, W[name], layout=1, **kw)
        return ops.gemm(dy, W[name + "T"], **kw)

    def _init_frozen(self, sd, g, lora: bool) -> None:
        H = self.H
        self.word = g("embeddings.word_embeddings.weight", bf16)
        self.pos = g("embeddings.position_embeddings.weight", bf16)
        self.type0 = g("embeddings.token_type_embeddings.weight", bf16)[0].contiguous()
        self.emb_g = g("embeddings.LayerNorm.weight", f32)
        self.emb_b = g("embeddings.LayerNorm.bias", f32)
        for l in range(self.nl):
            p = f"encoder.layer.{l}."
            if self.nf4 is not None:
                self.layers.append(self._init_layer_nf4(sd, l, g, lora))
                continue
            W = {}
            wq, wk, wv = (g(p + f"attention.self.{n}.weight", bf16) for n in self.LORA_TARGETS)
            W["Wqkv_aug"] = _aug_buf(3 * H, H, self.Ra, self.dev, zero=True)
            W["Wqkv_aug"][:, :H] = torch.cat([wq, wk, wv], 0)
            W["WqkvT_aug"] = _aug_buf(H, 3 * H, self.Ra, self.dev, zero=True)
            W["WqkvT_aug"][:, :3 * H] = torch.cat([wq, wk, wv], 0).t()
            W["bqkv"] = torch.cat([g(p + f"attention.self.{n}.bias", f32) for n in self.LORA_TARGETS])
            if lora:
                W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
                W["Bblk"] = torch.zeros(64, 3 * H, dtype=bf16, device=self.dev)
            W["Wo"] = g(p + "attention.output.dense.weight", bf16)
            W["WoT"] = W["Wo"].t().contiguous()
            W["bo"] = g(p + "attention.output.dense.bias", f32)
            W["ln1_g"] = g(p + "attention.output.LayerNorm.weight", f32)
            W["ln1_b"] = g(p + "attention.output.LayerNorm.bias", f32)
            W["Wi"] = g(p + "intermediate.dense.weight", bf16)
            W["WiT"] = W["Wi"].t().contiguous()
            W["bi"] = g(p + "intermediate.dense.bias", f32)
            W["Wo2"] = g(p + "output.dense.weight", bf16)
            W["Wo2T"] = W["Wo2"].t().contiguous()
            W["bo2"] = g(p + "output.dense.bias", f32)
            W["ln2_g"] = g(p + "output.LayerNorm.weight", f32)
            W["ln2_b"] = g(p + "output.LayerNorm.bias", f32)
            self.layers.append(W)

    def _init_layer_nf4(self, sd, l: int, g, lora: bool):
        """one layer in 4-bit storage (q|k|v fused row-wise, attention.output.dense, intermediate.dense, output.dense as NF4
        codes; biases / LayerNorms through the fp16 cast)"""
        from .nf4store import QuantLayer
        p = f"encoder.layer.{l}."
        H = self.H
        raw = lambda k: sd[k].to(device=self.dev, dtype=f32)
        W = QuantLayer(self.nf4, l)
        self.nf4.put(l, "Wqkv_aug", torch.cat([raw(p + f"attention.self.{n}.weight") for n in self.LORA_TARGETS], 0), tail_cols=self.Ra)
        self.nf4.put(l, "Wo", raw(p + "attention.output.dense.weight"))
        self.nf4.put(l, "Wi", raw(p + "intermediate.dense.weight"))
        self.nf4.put(l, "Wo2", raw(p + "output.dense.weight"))
        W["bqkv"] = torch.cat([g(p + f"attention.self.{n}.bias", f32) for n in self.LORA_TARGETS])
        if lora:
            W["A_stack"] = torch.zeros(64, H, dtype=bf16, device=self.dev)
            W["Bblk"] = torch.zeros(64, 3 * H, dtype=bf16, device=self.dev)
        for k, n in (("bo", "attention.output.dense.bias"), ("ln1_g", "attention.output.LayerNorm.weight"),
                     ("ln1_b", "attention.output.LayerNorm.bias"), ("bi", "intermediate.dense.bias"), ("bo2", "output.dense.bias"),
                     ("ln2_g", "output.LayerNorm.weight"), ("ln2_b", "output.LayerNorm.bias")):
            W[k] = g(p + n, f32)
        return W

    def _drop(self, p: float, call: int, layer: int, site: int):
        """dropout descriptor of one site, or None when inactive (eval mode / p == 0)"""
        if not self.training or p <= 0.0:
            return None
        return ops.Drop(p, self.drop_seed, (call << 24) | (layer << 8) | site, self.drop_offset)

    # ------------------------------------------------------------------------------------------------------------
    def _pack_entries(self):
        H, r, s = self.H, self.r, self.lora.scale
        for l, W in enumerate(self.layers):
            for j, n in enumerate(self.LORA_TARGETS):
                name = f"encoder.layer.{l}.attention.self.{n}"
                A, B = self.lora.A[name], self.lora.B[name]             # [r,H], [H,r] fp32
                if self.nf4 is not None:                                 # 4-bit storage: LoRA columns live in the layer's tail block
                    yield (B, r, 1, self.nf4.tail(l, "Wqkv_aug")[j * H:(j + 1) * H, j * r:], H, r, s)
                else:
                    yield (B, r, 1, W["Wqkv_aug"][j * H:(j + 1) * H, H + j * r:], H, r, s)      # (alpha/r) * B
                    yield (A, 1, H, W["WqkvT_aug"][:, 3 * H + j * r:], H, r, 1.0)                # A^T
                yield (A, H, 1, W["A_stack"][j * r:(j + 1) * r], r, H, 1.0)                  # A
                yield (B, 1, r, W["Bblk"][j * r:(j + 1) * r, j * H:], r, H, s)               # (alpha/r) * B^T, block j

    def repack_lora(self) -> None:
        """refresh the bf16 LoRA blocks inside the augmented weights from the fp32 master copies: ONE launch over a
        device-resident table of (source, strides, destination) records built once (pointers never move)"""
        if self.lora is None:
            return
        if getattr(self, "_pack_tab", None) is None:
            self._pack_tab = ops.build_pack_table(list(self._pack_entries()), self.dev)
        ops.pack_table_(self._pack_tab)

    # ------------------------------------------------------------------------------------------------------------
    def forward_hidden(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True):
        """ids, mask: int64 [B,L] on device -> (hidden fp32 [B,L,H], ctx)"""
        hs, ctx = self.forward_segments([(ids, mask)], save=save)
        return hs[0], ctx

    def forward_segments(self, segments, save: bool = True):
        """Several (ids, mask) batches with different sequence lengths (the query batch and the passage batch of one
        step) through ONE pass over the weights: all linear layers / norms / activations run on the concatenated token
        rows (M = sum B_i L_i: bigger, better-filled tensor-core tiles, half the launches); only attention is launched
        per segment. Returns ([hidden_i fp32 [B_i,L_i,H]], ctx)."""
        H, F, Ra = self.H, self.F, self.Ra
        if self.roberta:
            for ids, _ in segments:
                if ids.shape[1] > self.max_len:
                    raise ValueError(f"sequence length {ids.shape[1]} exceeds the {self.max_len} positions this encoder's table "
                                     f"serves (max_position_embeddings {self.cfg['max_position_embeddings']} - pad_token_id "
                                     f"{self.pad} - 1)")
        ctx = _Ctx()
        ctx.segs = []
        r0 = 0
        for ids, mask in segments:
            B, L = ids.shape
            ctx.segs.append((B, L, mask.contiguous(), r0))
            r0 += B * L
        M = r0
        ctx.M, ctx.layers = M, []
        self._call += 1
        ctx.call = call = self._call
        ctx.training = self.training
        z = torch.empty(M, H, dtype=f32, device=self.dev)
        pos_ids = torch.empty(M, dtype=torch.int64, device=self.dev) if self.roberta else None
        for (ids, _), (B, L, _, s0) in zip(segments, ctx.segs):
            if self.roberta:
                ops.roberta_embed(ids, self.word, self.pos, self.type0, self.pad, out=z[s0:s0 + B * L],
                                  pos_ids=pos_ids[s0:s0 + B * L])
            else:
                ops.bert_embed(ids, self.word, self.pos, self.type0, out=z[s0:s0 + B * L])
        x_aug = _aug_buf(M, H, Ra, self.dev)
        x32, _, mean, rstd = ops.layernorm_fwd(z, self.emb_g, self.emb_b, self.eps, y16=x_aug[:, :H],
                                               drop=self._drop(self.p_hidden, call, 255, 0))
        if save and self.full is not None:                     # the embedding tables are trainable: keep their LN state
            ctx.z_emb, ctx.mean_e, ctx.rstd_e = z, mean, rstd
            ctx.ids = [ids.contiguous() for ids, _ in segments]
            ctx.pos_ids = pos_ids
        for li, W in enumerate(self.layers):
            a = _Ctx()
            a.x_aug = x_aug
            if Ra:
                ops.skinny_gemm(x_aug[:, :H], W["A_stack"], x_aug[:, H:], K=H, R=Ra,              # u = dropout(x) A^T [M,3r]
                                dropx=self._drop(self.p_lora, call, li, 3))
            qkv = ops.gemm(x_aug, W["Wqkv_aug"], bias=W["bqkv"])                                   # [M,3H] (+LoRA via K-aug)
            att = torch.empty(M, H, dtype=bf16, device=self.dev)
            lses = []
            for si, (B, L, mask, s0) in enumerate(ctx.segs):
                rows = slice(s0, s0 + B * L)
                _, lse = ops.attention_auto_fwd(qkv[rows, :H], qkv[rows, H:2 * H], qkv[rows, 2 * H:], mask, B, L, self.nh,
                                           self.nh, self.hd, causal=False, out=att[rows],
                                           drop=self._drop(self.p_attn, call, li, 8 + si))
                lses.append(lse)
            z1 = ops.gemm(att, W["Wo"], out_dtype=f32, bias=W["bo"], resid=x32,                    # dropout(dense) + residual
                          drop=self._drop(self.p_hidden, call, li, 1))
            h_aug = torch.empty(M, H, dtype=bf16, device=self.dev)
            h32, _, m1, r1 = ops.layernorm_fwd(z1, W["ln1_g"], W["ln1_b"], self.eps, y16=h_aug)
            if ops.fuse_gelu(H):
                pre, act = ops.gemm_gelu(h_aug, W["Wi"], bias=W["bi"])                             # [M,F] pre-activation AND gelu(pre): one launch
            else:
                pre = ops.gemm(h_aug, W["Wi"], bias=W["bi"])
                act = ops.gelu_fwd(pre)
            z2 = ops.gemm(act, W["Wo2"], out_dtype=f32, bias=W["bo2"], resid=h32, drop=self._drop(self.p_hidden, call, li, 2))
            x_aug = _aug_buf(M, H, Ra, self.dev)
            x32, _, m2, r2 = ops.layernorm_fwd(z2, W["ln2_g"], W["ln2_b"], self.eps, y16=x_aug[:, :H])
            if save:
                a.qkv, a.att, a.lse, a.z1, a.m1, a.r1, a.h_aug, a.pre, a.act, a.z2, a.m2, a.r2 = \
                    qkv, att, lses, z1, m1, r1, h_aug, pre, act, z2, m2, r2
                ctx.layers.append(a)
        return [x32[s0:s0 + B * L].view(B, L, H) for (B, L, _, s0) in ctx.segs], ctx

    # ------------------------------------------------------------------------------------------------------------
    def backward_hidden(self, ctx: _Ctx, d_hidden: torch.Tensor) -> None:
        """d_hidden fp32 [B,L,H]; accumulates LoRA gradients into self.lora.grad (base weights are frozen: PEFT mode)."""
        self.backward_segments(ctx, [d_hidden])

    def backward_segments(self, ctx: _Ctx, d_hiddens) -> None:
        if not self.trainable:
            return                                           # nothing trainable below the pooled output
        M, H = ctx.M, self.H
        d = d_hiddens[0].reshape(-1, H) if len(d_hiddens) == 1 else torch.cat([t.reshape(-1, H) for t in d_hiddens], 0)
        d = d.contiguous()
        last, Wl = ctx.layers[self.nl - 1], self.layers[self.nl - 1]
        if self.full is not None:
            ctx.acc = self.full.begin_backward()
            ops.col_reduce_(dy_f32=d, z=last.z2, mean=last.m2, rstd=last.r2, out_sum=self.full.g(f"L{self.nl - 1}.ln2_b"),
                            out_prod=self.full.g(f"L{self.nl - 1}.ln2_g"))
        last._pre = ops.layernorm_bwd(last.z2, Wl["ln2_g"], last.m2, last.r2, dy_f32=d,
                                      drop16=self._bdrop(ctx, self.p_hidden, self.nl - 1, 2))
        self._bwd_from_ln2(ctx, self.nl - 1)
        if self.full is not None:
            self.full.end_backward()

    def _bdrop(self, ctx, p: float, layer: int, site: int):
        """the forward call's dropout descriptor, regenerated for its backward"""
        if not ctx.training or p <= 0.0:
            return None
        return ops.Drop(p, self.drop_seed, (ctx.call << 24) | (layer << 8) | site, self.drop_offset)

    def _bwd_from_ln2(self, ctx: _Ctx, l_start: int) -> None:
        """continue the backward at layer l_start whose LN2 input gradient has already been computed (stashed in _pre)"""
        M, H, Ra, r = ctx.M, self.H, self.Ra, self.r
        bank = self.full
        acc = getattr(ctx, "acc", False)
        G = (lambda l, n: bank.g(f"L{l}.{n}")) if bank is not None else None
        for l in range(l_start, -1, -1):
            W, a = self.layers[l], ctx.layers[l]
            dz2_32, dz2_16 = a._pre
            del a._pre
            if bank is not None:                               # output.dense: dW = dz2^T act, db = colsum(dz2)
                ops.wgrad_(dz2_16, a.act, G(l, "Wo2"), acc)
                ops.col_reduce_(dy_bf16=dz2_16, out_sum=G(l, "bo2"))
            if ops.fuse_gelu(H):
                dact = self._dgrad(dz2_16, W, "Wo2", gelu_pre=a.pre)                               # d(pre): gelu' applied in the dgrad epilogue
            else:
                dact = self._dgrad(dz2_16, W, "Wo2")
                ops.gelu_bwd_(a.pre, dact)
            if bank is not None:                               # intermediate.dense
                ops.wgrad_(dact, a.h_aug, G(l, "Wi"), acc)
                ops.col_reduce_(dy_bf16=dact, out_sum=G(l, "bi"))
            dh_16 = self._dgrad(dact, W, "Wi")
            if bank is not None:                               # attention.output.LayerNorm
                ops.col_reduce_(dy_f32=dz2_32, dy_bf16=dh_16, z=a.z1, mean=a.m1, rstd=a.r1, out_sum=G(l, "ln1_b"),
                                out_prod=G(l, "ln1_g"))
            dz1_32, dz1_16 = ops.layernorm_bwd(a.z1, W["ln1_g"], a.m1, a.r1, dy_f32=dz2_32, dy_bf16=dh_16,
                                               drop16=self._bdrop(ctx, self.p_hidden, l, 1))
            if bank is not None:                               # attention.output.dense
                ops.wgrad_(dz1_16, a.att, G(l, "Wo"), acc)
                ops.col_reduce_(dy_bf16=dz1_16, out_sum=G(l, "bo"))
            datt = self._dgrad(dz1_16, W, "Wo")
            dqkv_aug = _aug_buf(M, 3 * H, Ra, self.dev)
            for si, ((B, L, mask, s0), lse) in enumerate(zip(ctx.segs, a.lse)):
                rows = slice(s0, s0 + B * L)
                ops.attention_auto_bwd(a.qkv[rows, :H], a.qkv[rows, H:2 * H], a.qkv[rows, 2 * H:], mask, a.att[rows], lse,
                                  datt[rows], B, L, self.nh, self.nh, self.hd, causal=False, dq=dqkv_aug[rows, :H],
                                  dk=dqkv_aug[rows, H:2 * H], dv=dqkv_aug[rows, 2 * H:3 * H],
                                  drop=self._bdrop(ctx, self.p_attn, l, 8 + si))
            if bank is not None:
                self._bwd_full_tail(ctx, l, dqkv_aug, dz1_32, acc)
                continue
            for j, n in enumerate(self.LORA_TARGETS):
                # g_j = dY_j (alpha/r) B_j : only the target's own column block is read
                ops.skinny_gemm(dqkv_aug[:, j * H:(j + 1) * H], W["Bblk"][j * r:(j + 1) * r, j * H:(j + 1) * H],
                                dqkv_aug[:, 3 * H + j * r:], K=H, R=r)
            names = [f"encoder.layer.{l}.attention.self.{n}" for n in self.LORA_TARGETS]
            # dA[rr,k] += sum_m g_j[m,rr] x[m,k]: q and k share one pass over x (16-row MMA tile), v takes a second
            xdrop = self._bdrop(ctx, self.p_lora, l, 3)                          # dA = g^T dropout(x)
            ops.lora_wgrad_(a.x_aug[:, :H], dqkv_aug[:, 3 * H:], self.lora.gA[names[0]], H, 1, H, 2 * r, 1.0,
                            out1=self.lora.gA[names[1]], dropx=xdrop)
            ops.lora_wgrad_(a.x_aug[:, :H], dqkv_aug[:, 3 * H + 2 * r:], self.lora.gA[names[2]], H, 1, H, r, 1.0, dropx=xdrop)
            for j, name in enumerate(names):
                # dB[n,rr] += (alpha/r) * sum_m dY_j[m,n] u_j[m,rr]
                ops.lora_wgrad_(dqkv_aug[:, j * H:(j + 1) * H], a.x_aug[:, H + j * r:], self.lora.gB[name], 1, r, H, r,
                                self.lora.scale)
            if l == 0:
                return
            if self.nf4 is not None:                                              # expanded W[out,in] read MN-major + (g A)
                dx_16 = ops.gemm(dqkv_aug[:, :3 * H], W["Wqkv_aug"][:, :H], layout=1)
                ops.lora_dx_(dx_16, dqkv_aug[:, 3 * H:], W["A_stack"], K=H, R=Ra, drop=xdrop)
            elif xdrop is None:
                dx_16 = ops.gemm(dqkv_aug, W["WqkvT_aug"])                        # LoRA's A-path folded into K
            else:
                dx_16 = ops.gemm(dqkv_aug[:, :3 * H], W["WqkvT_aug"][:, :3 * H])   # base path only ...
                ops.lora_dx_(dx_16, dqkv_aug[:, 3 * H:], W["A_stack"], K=H, R=Ra, drop=xdrop)   # ... + mask * (g A)
            p, Wp = ctx.layers[l - 1], self.layers[l - 1]
            p._pre = ops.layernorm_bwd(p.z2, Wp["ln2_g"], p.m2, p.r2, dy_f32=dz1_32, dy_bf16=dx_16,
                                       drop16=self._bdrop(ctx, self.p_hidden, l - 1, 2))

    def _bwd_full_tail(self, ctx: _Ctx, l: int, dqkv: torch.Tensor, dz1_32: torch.Tensor, acc: bool) -> None:
        """full fine-tuning: fused q|k|v projection gradients, then either the previous layer's output LayerNorm or (l == 0)
        the embedding block: dropout -> LayerNorm -> word / position / token-type tables"""
        bank, W, a, H = self.full, self.layers[l], ctx.layers[l], self.H
        ops.wgrad_(dqkv, a.x_aug[:, :H], bank.g(f"L{l}.Wqkv"), acc)
        ops.col_reduce_(dy_bf16=dqkv, out_sum=bank.g(f"L{l}.bqkv"))
        dx_16 = ops.gemm(dqkv, W["Wqkv_aug"], layout=1)
        bank.bucket_ready(f"L{l}.")                                    # this layer's four weight gradients are final
        if l > 0:
            p, Wp = ctx.layers[l - 1], self.layers[l - 1]
            ops.col_reduce_(dy_f32=dz1_32, dy_bf16=dx_16, z=p.z2, mean=p.m2, rstd=p.r2, out_sum=bank.g(f"L{l - 1}.ln2_b"),
                            out_prod=bank.g(f"L{l - 1}.ln2_g"))
            p._pre = ops.layernorm_bwd(p.z2, Wp["ln2_g"], p.m2, p.r2, dy_f32=dz1_32, dy_bf16=dx_16,
                                       drop16=self._bdrop(ctx, self.p_hidden, l - 1, 2))
            return
        g = ops.masked_add(dz1_32, dx_16, drop=self._bdrop(ctx, self.p_hidden, 255, 0), out=dz1_32)   # through the embedding dropout
        ops.col_reduce_(dy_f32=g, z=ctx.z_emb, mean=ctx.mean_e, rstd=ctx.rstd_e, out_sum=bank.g("emb_b"), out_prod=bank.g("emb_g"))
        dz, _ = ops.layernorm_bwd(ctx.z_emb, self.emb_g, ctx.mean_e, ctx.rstd_e, dy_f32=g, want_bf16=False)
        for ids, (B, L, _, s0) in zip(ctx.ids, ctx.segs):
            if self.roberta:                                              # positions of the forward; padding_idx rows get nothing
                ops.embed_scatter_add_(dz[s0:s0 + B * L], ids, bank.g("word"), bank.g("pos"), L,
                                       pos_ids=ctx.pos_ids[s0:s0 + B * L], pad_id=self.pad)
            else:
                ops.embed_scatter_add_(dz[s0:s0 + B * L], ids, bank.g("word"), bank.g("pos"), L)
        ops.col_reduce_(dy_f32=dz, out_sum=bank.g("type")[0])                 # token_type_ids are all zero (reference quirk 7)
