"""Falcon decoder (Falcon-7B architecture: parallel attention + MLP, multi-query attention, LayerNorm, GELU, rotary,
tied lm_head) — forward and (full fine-tuning) backward launch sequences over the C-ABI kernels.

Mirrors `self.generator_model(input_ids=..., attention_mask=...).logits` of the reference
(dalm/models/rag_e2e_base_model.py:104-106) through HF FalconForCausalLM (`trust_remote_code=True`, :54) for BASELINE
config 5. The reference's generator LoRA targets (`q_proj`, `v_proj`, rag_e2e_base_model.py:76-77) do not exist in
Falcon (its fused projection is `query_key_value`), so peft refuses `--use-peft generator|both`; with `--use-peft
retriever` or no PEFT the reference trains EVERY Falcon parameter (no get_peft_model => requires_grad stays True,
Adam over rag_model.parameters(), train_rage2e.py:336). Two modes here:

  frozen (lora=False, full=False)  forward only — evaluation, and the cheap reading of cfg-5 where only the retriever learns
  full   (full=True)               all parameters in a DenseBank (fp32 master + bf16 shadow + fp32 gradients); the backward
                                   RECOMPUTES each layer's forward from its saved input (one fp32 [M,H] tensor per layer):
                                   cfg-5's 36 864 tokens x 32 layers of full activations (~140 GB) do not fit next to the
                                   125 GB parameter bank, 21 GB of layer inputs do. Costs one extra forward (+33 % FLOPs).

Per layer (bf16 weights): Wqkv [(nh+2)*hd, H] fused q|k|v (one KV head), Wd [H,H], W1 [4H,H], W2 [H,4H]; LayerNorm
gain/bias fp32. Residual stream fp32; x_out = x + attn(LN(x)) + mlp(LN(x)) (one LayerNorm feeds both branches).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import ops
from .dense import DenseBank
from .params import rope_inv_freq

bf16, f32 = torch.bfloat16, torch.float32


class _Ctx:
    pass


class FalconDecoder(torch.nn.Module):
    LORA_TARGETS = ()

    def __init__(self, cfg: Dict, state_dict: Dict[str, torch.Tensor], device="cuda", lora: bool = False, lora_seed: int = 1,
                 full: bool = False):
        super().__init__()
        if lora:
            raise ValueError("Target modules ['q_proj', 'v_proj'] not found in the base model (Falcon fuses them into "
                             "`query_key_value`): the reference's generator LoRA config cannot apply to Falcon; use "
                             "use_peft='retriever'")
        if cfg.get("new_decoder_architecture", False) or cfg.get("alibi", False) or not cfg.get("parallel_attn", True) \
                or not cfg.get("multi_query", True) or cfg.get("bias", False):
            raise NotImplementedError("only the Falcon-7B architecture variant (parallel_attn, multi_query, rotary, no bias) is built")
        self.cfg = cfg
        self.H = H = cfg["hidden_size"]
        self.nl = cfg["num_hidden_layers"]
        self.nh = cfg["num_attention_heads"]
        self.hd = H // self.nh
        self.V = cfg["vocab_size"]
        self.F = cfg.get("ffn_hidden_size") or 4 * H
        self.eps = float(cfg.get("layer_norm_epsilon", 1e-5))
        self.inv_freq = rope_inv_freq(cfg, self.hd)           # default RoPE only: a scaled one is refused
        self.dev = torch.device(device)
        if self.hd not in (32, 64, 128):
            raise NotImplementedError(f"head_dim {self.hd} not supported by the attention kernels")
        self.Nq, self.Nkv = self.nh * self.hd, self.hd
        self.Vp = (self.V + 7) // 8 * 8
        self.lora = None
        self.full: Optional[DenseBank] = None
        self.layers: List[Dict[str, torch.Tensor]] = []
        sd = state_dict
        if full:
            self._init_full(sd)
        else:
            self._init_frozen(sd)
        self._rope_cache: Dict[int, tuple] = {}
        self.drop_offset = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.eval()

    # ---- parameters -----------------------------------------------------------------------------------------------
    def _init_frozen(self, sd) -> None:
        H = self.H
        g = lambda k, dt: sd[k].to(device=self.dev, dtype=dt).contiguous()
        self.embed = g("transformer.word_embeddings.weight", bf16)
        lm = g("lm_head.weight", bf16) if "lm_head.weight" in sd else self.embed          # tied
        if self.Vp != self.V:
            lm = torch.cat([lm, torch.zeros(self.Vp - self.V, H, dtype=bf16, device=self.dev)], 0)
        self.lm_head = lm
        self.lnf_g, self.lnf_b = g("transformer.ln_f.weight", f32), g("transformer.ln_f.bias", f32)
        for l in range(self.nl):
            p = f"transformer.h.{l}."
            self.layers.append({
                "ln_g": g(p + "input_layernorm.weight", f32), "ln_b": g(p + "input_layernorm.bias", f32),
                "Wqkv": g(p + "self_attention.query_key_value.weight", bf16),
                "Wd": g(p + "self_attention.dense.weight", bf16),
                "W1": g(p + "mlp.dense_h_to_4h.weight", bf16), "W2": g(p + "mlp.dense_4h_to_h.weight", bf16),
            })

    def _param_map(self, has_head: bool):
        m = [("embed", "acc", "transformer.word_embeddings.weight"), ("lnf_g", "acc", "transformer.ln_f.weight"),
             ("lnf_b", "acc", "transformer.ln_f.bias")]
        if has_head:
            m.append(("lm_head", "gemm", "lm_head.weight"))
        for l in range(self.nl):
            p = f"transformer.h.{l}."
            m += [(f"L{l}.ln_g", "acc", p + "input_layernorm.weight"), (f"L{l}.ln_b", "acc", p + "input_layernorm.bias"),
                  (f"L{l}.Wqkv", "gemm", p + "self_attention.query_key_value.weight"),
                  (f"L{l}.Wd", "gemm", p + "self_attention.dense.weight"),
                  (f"L{l}.W1", "gemm", p + "mlp.dense_h_to_4h.weight"), (f"L{l}.W2", "gemm", p + "mlp.dense_4h_to_h.weight")]
        return m

    def _init_full(self, sd) -> None:
        if self.Vp != self.V:
            raise NotImplementedError("full fine-tuning of Falcon needs vocab_size % 8 == 0 (Falcon-7B: 65024)")
        # HF ties lm_head to word_embeddings (tie_word_embeddings=True): a separate tensor only if the checkpoint says so
        has_head = "lm_head.weight" in sd and not self.cfg.get("tie_word_embeddings", True)
        self._names = self._param_map(has_head)
        bank = DenseBank([(key, tuple(sd[name].shape), kind) for key, kind, name in self._names], self.dev)
        for key, _, name in self._names:
            bank.w32(key).copy_(sd[name].to(self.dev, f32))
        bank.sync_shadow()
        self.full = bank
        self.full_flat = torch.nn.Parameter(bank.p32, requires_grad=True)
        self.full_flat.grad = bank.g32
        self.full_flat._dalm_bank = bank
        self.tied = not has_head
        self.embed = bank.w16("embed")
        self.lm_head = self.embed if self.tied else bank.w16("lm_head")
        self.lnf_g, self.lnf_b = bank.w32("lnf_g"), bank.w32("lnf_b")
        for l in range(self.nl):
            k = lambda n: f"L{l}.{n}"
            self.layers.append({"ln_g": bank.w32(k("ln_g")), "ln_b": bank.w32(k("ln_b")), "Wqkv": bank.w16(k("Wqkv")),
                                "Wd": bank.w16(k("Wd")), "W1": bank.w16(k("W1")), "W2": bank.w16(k("W2"))})

    def hf_state_dict(self) -> Dict[str, torch.Tensor]:
        if self.full is None:
            raise RuntimeError("hf_state_dict: only fully fine-tuned models own their weights")
        out = {name: self.full.w32(key).detach().cpu().clone() for key, _, name in self._names}
        if self.tied:
            out["lm_head.weight"] = out["transformer.word_embeddings.weight"]
        return out

    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        for key, _, name in self._names:
            self.full.w32(key).copy_(sd[name].to(self.dev, f32))
        self.full.sync_shadow()

    @property
    def trainable(self) -> bool:
        return self.full is not None

    @property
    def anchor(self) -> torch.nn.Parameter:
        return self.full_flat

    def repack_lora(self) -> None:
        pass

    def banks(self) -> list:
        return [self.full] if self.full is not None else []

    def grad_buffers(self) -> list:
        return [b.grad for b in self.banks()]

    def _rope(self, L: int):
        if L not in self._rope_cache:
            fr = torch.outer(torch.arange(L, dtype=torch.float32), self.inv_freq)
            self._rope_cache[L] = (fr.cos().to(self.dev).contiguous(), fr.sin().to(self.dev).contiguous())
        return self._rope_cache[L]

    # ---- one layer ------------------------------------------------------------------------------------------------
    def _layer_fwd(self, W, x, mask, B, L, cos_t, sin_t, keep: bool, pos=None, kv_sink=None):
        """x fp32 [M,H] -> x_out fp32; with keep=True also everything the layer's backward needs. pos / kv_sink: `generate`'s
        prefill (explicit position ids into the cos / sin tables; callback receiving the rotated qkv buffer)"""
        _, h, mean, rstd = ops.layernorm_fwd(x, W["ln_g"], W["ln_b"], self.eps, want_f32=False)   # one LN feeds both branches
        qkv = ops.gemm(h, W["Wqkv"])                                                  # [M, (nh+2)*hd]
        if pos is None:
            ops.rope_(qkv, 0, self.nh + 1, self.hd, cos_t, sin_t, L)                  # q heads then the single k head
        else:
            ops.rope_pos_(qkv, 0, self.nh + 1, self.hd, cos_t, sin_t, pos)
        if kv_sink is not None:
            kv_sink(qkv)
        att, lse = ops.attention_auto_fwd(qkv[:, :self.Nq], qkv[:, self.Nq:self.Nq + self.hd], qkv[:, self.Nq + self.hd:],
                                     mask, B, L, self.nh, 1, self.hd, causal=True)
        t = ops.gemm(att, W["Wd"], out_dtype=f32, resid=x)                            # x + attention branch
        if keep:
            if ops.fuse_gelu(self.H):
                pre, h4 = ops.gemm_gelu(h, W["W1"])                                   # GELU's input (needed by its backward) and output, one launch
            else:
                pre = ops.gemm(h, W["W1"])
                h4 = ops.gelu_fwd(pre)
        else:
            pre, h4 = None, ops.gemm(h, W["W1"], act=1)                               # GELU(erf) fused in the epilogue
        x_out = ops.gemm(h4, W["W2"], out_dtype=f32, resid=t)                         # + MLP branch
        if not keep:
            return x_out, None
        a = _Ctx()
        a.h, a.mean, a.rstd, a.qkv, a.att, a.lse, a.pre, a.h4 = h, mean, rstd, qkv, att, lse, pre, h4
        return x_out, a

    def _layer_bwd(self, l: int, W, x, a, dx32, dx16, mask, B, L, cos_t, sin_t, acc: bool):
        """dx (fp32 + its bf16 copy) w.r.t. the layer output -> (dx32, dx16) w.r.t. the layer input; parameter gradients into
        the bank. dx32 is updated in place."""
        bank, M, H, hd = self.full, B * L, self.H, self.hd
        G = lambda n: bank.g(f"L{l}.{n}")
        # MLP branch
        ops.wgrad_(dx16, a.h4, G("W2"), acc)
        if ops.fuse_gelu(self.H):
            dpre = ops.gemm(dx16, W["W2"], layout=1, act=2, resid=a.pre)              # [M,4H] = d h4 * gelu'(pre) = d pre
        else:
            dpre = ops.gemm(dx16, W["W2"], layout=1)                                  # [M,4H] = d h4
            ops.gelu_bwd_(a.pre, dpre)                                                # -> d pre
        ops.wgrad_(dpre, a.h, G("W1"), acc)
        dh = ops.gemm(dpre, W["W1"], layout=1)                                        # [M,H] MLP part of d LN-output
        # attention branch
        ops.wgrad_(dx16, a.att, G("Wd"), acc)
        datt = ops.gemm(dx16, W["Wd"], layout=1)                                      # [M,Nq]
        dqkv = torch.empty(M, self.Nq + 2 * hd, dtype=bf16, device=self.dev)
        ops.attention_auto_bwd(a.qkv[:, :self.Nq], a.qkv[:, self.Nq:self.Nq + hd], a.qkv[:, self.Nq + hd:], mask, a.att, a.lse, datt,
                          B, L, self.nh, 1, hd, causal=True, dq=dqkv[:, :self.Nq], dk=dqkv[:, self.Nq:self.Nq + hd],
                          dv=dqkv[:, self.Nq + hd:])                                  # dK / dV summed over the 71 query heads
        ops.rope_(dqkv, 0, self.nh + 1, hd, cos_t, sin_t, L, backward=True)
        ops.wgrad_(dqkv, a.h, G("Wqkv"), acc)
        dh = ops.gemm(dqkv, W["Wqkv"], layout=1, resid=dh, out=dh)                    # + attention part, accumulated in place
        # the shared LayerNorm, and the residual connection around the whole block
        ops.col_reduce_(dy_bf16=dh, z=x, mean=a.mean, rstd=a.rstd, out_sum=G("ln_b"), out_prod=G("ln_g"))
        return ops.layernorm_bwd_res(x, W["ln_g"], a.mean, a.rstd, dh, dres=dx32, dz32=dx32)

    # ---- whole model ----------------------------------------------------------------------------------------------
    def _forward_to_final(self, ids: torch.Tensor, mask: torch.Tensor, save: bool):
        """-> (hf bf16 [M,H] after ln_f, ctx or None). ctx (save=True on a trainable model) holds only each layer's fp32 input:
        the backward recomputes the rest."""
        B, L = ids.shape
        cos_t, sin_t = self._rope(L)
        mask = mask.contiguous()
        keep_inputs = save and self.full is not None
        ctx = _Ctx() if keep_inputs else None
        x = ops.embed_gather(ids, self.embed)                                         # fp32 residual stream [M,H]
        xs = []
        for W in self.layers:
            if keep_inputs:
                xs.append(x)
            x, _ = self._layer_fwd(W, x, mask, B, L, cos_t, sin_t, keep=False)
        _, hf, mean_f, rstd_f = ops.layernorm_fwd(x, self.lnf_g, self.lnf_b, self.eps, want_f32=False)
        if keep_inputs:
            ctx.B, ctx.L, ctx.mask, ctx.ids, ctx.xs, ctx.x_final, ctx.hf, ctx.mean_f, ctx.rstd_f = \
                B, L, mask, ids.contiguous(), xs, x, hf, mean_f, rstd_f
        return hf, ctx

    def forward_logits(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = False):
        """ids, mask int64 [B,L] -> (logits bf16 [B,L,V], ctx)"""
        B, L = ids.shape
        hf, ctx = self._forward_to_final(ids, mask, save)
        logits = ops.gemm(hf, self.lm_head)
        return logits.view(B, L, self.Vp)[:, :, :self.V], ctx

    def forward_final(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = False):
        """the fused step's forward: everything up to ln_f; the (tied) lm_head runs chunk by chunk inside `head_loss`, so the
        [B,L,65024] logits (4.8 GB in bf16 at cfg-5) are never written. -> handle for head_loss / backward_final"""
        hf, ctx = self._forward_to_final(ids, mask, save)
        h = _Ctx()
        h.hf, h.ctx = hf, ctx
        return h

    def head_loss(self, h, ids: torch.Tensor, mask: torch.Tensor, nsum: torch.Tensor, need_grad: bool = True, grad_out: float = 1.0):
        """-> (tok_lp fp32 [B,L], d(hf) bf16 [M,H] or None); see engine/head.py"""
        from .head import chunked_head_loss
        need_grad = need_grad and self.full is not None and h.ctx is not None
        wgrad = None
        if need_grad:
            bank = self.full
            h.acc = bank.begin_backward()
            tgt = bank.g("embed") if self.tied else bank.g("lm_head")                 # tied head: lands in the embedding gradient
            acc0 = True if self.tied else h.acc
            wgrad = lambda dl, x, first: ops.wgrad_(dl, x, tgt, acc0 if first else True)
        return chunked_head_loss(h.hf, self.lm_head, None, self.V, ids, mask, nsum, need_grad, grad_out, wgrad)

    def backward_final(self, h, dhf: torch.Tensor) -> None:
        if self.full is None or h.ctx is None or dhf is None:
            return
        self._backward_from_dhf(h.ctx, dhf, h.acc)

    # ---- greedy decoding with a KV cache (evaluation: reference dalm/eval/eval_rag.py:126-140) ----------------------
    def kv_columns(self):
        """(first K column, first V column, width) of the rotated key / value head inside a layer's qkv buffer"""
        return self.Nq, self.Nq + self.hd, self.hd

    def _prefill_last(self, ids, mask, pos, tables, sink) -> torch.Tensor:
        B, L0 = ids.shape
        cos_t, sin_t = tables
        mask = mask.contiguous()
        x = ops.embed_gather(ids, self.embed)
        for li, W in enumerate(self.layers):
            x, _ = self._layer_fwd(W, x, mask, B, L0, cos_t, sin_t, keep=False, pos=pos, kv_sink=lambda qkv, li=li: sink(li, qkv))
        x_last = x.view(B, L0, self.H)[:, -1].contiguous()                            # only the last column is scored
        _, hf, _, _ = ops.layernorm_fwd(x_last, self.lnf_g, self.lnf_b, self.eps, want_f32=False)
        return hf

    def _decode_step(self, ids, pos, caches, kmask, cur, tables) -> torch.Tensor:
        """one token per sequence: ids / pos int64 [B] -> logits bf16 [B, Vp]; appends K / V at cache column `cur` (int, or the int32 [B] device tensor of per-row columns: CUDA-graph mode)"""
        cos_t, sin_t = tables
        x = ops.embed_gather(ids, self.embed)
        for li, W in enumerate(self.layers):
            _, h, _, _ = ops.layernorm_fwd(x, W["ln_g"], W["ln_b"], self.eps, want_f32=False)
            qkv = ops.gemm_rows(h, W["Wqkv"])
            ops.rope_pos_(qkv, 0, self.nh + 1, self.hd, cos_t, sin_t, pos)
            att = ops.attention_decode(qkv, 0, self.Nq, self.Nq + self.hd, caches[li][0], caches[li][1], kmask, cur,
                                       self.nh, 1, self.hd)
            t = ops.gemm_rows(att, W["Wd"], out_dtype=f32, resid=x)
            x = ops.gemm_rows(ops.gemm_rows(h, W["W1"], act=1), W["W2"], out_dtype=f32, resid=t)
        _, hf, _, _ = ops.layernorm_fwd(x, self.lnf_g, self.lnf_b, self.eps, want_f32=False)
        return ops.gemm_rows(hf, self.lm_head)

    def generate(self, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
        """HF `generate`: greedy search or sampling, as the checkpoint's generation config and the call select; see
        engine/decoding.py"""
        from .decoding import generate
        return generate(self, input_ids, attention_mask, **kw)

    def backward_logits(self, ctx, dlogits: torch.Tensor) -> None:
        """dlogits bf16 [B,L,V] -> gradients of every parameter (full mode); nothing to do for a frozen decoder"""
        if self.full is None or ctx is None:
            return
        bank, B, L = self.full, ctx.B, ctx.L
        M, H = B * L, self.H
        cos_t, sin_t = self._rope(L)
        acc = bank.begin_backward()
        if dlogits.stride(-1) != 1 or dlogits.stride(-2) != self.Vp:
            dlogits = dlogits.contiguous()
        dl2 = torch.as_strided(dlogits, (M, self.Vp), (self.Vp, 1), dlogits.storage_offset())
        # tied head: its weight gradient lands in the embedding table's (accumulating) gradient
        ops.wgrad_(dl2, ctx.hf, bank.g("embed") if self.tied else bank.g("lm_head"), True if self.tied else acc)
        dhf = ops.gemm(dl2, self.lm_head, layout=1)                                   # [M,H]
        self._backward_from_dhf(ctx, dhf, acc)

    def _backward_from_dhf(self, ctx, dhf: torch.Tensor, acc: bool) -> None:
        """from the gradient of ln_f's output (bf16 [M,H]) down through the layers (per-layer recomputation)"""
        bank, B, L = self.full, ctx.B, ctx.L
        cos_t, sin_t = self._rope(L)
        ops.col_reduce_(dy_bf16=dhf, z=ctx.x_final, mean=ctx.mean_f, rstd=ctx.rstd_f, out_sum=bank.g("lnf_b"), out_prod=bank.g("lnf_g"))
        dx32, dx16 = ops.layernorm_bwd(ctx.x_final, self.lnf_g, ctx.mean_f, ctx.rstd_f, dy_bf16=dhf)
        for l in range(self.nl - 1, -1, -1):
            W, x = self.layers[l], ctx.xs[l]
            _, a = self._layer_fwd(W, x, ctx.mask, B, L, cos_t, sin_t, keep=True)      # recompute this layer's activations
            dx32, dx16 = self._layer_bwd(l, W, x, a, dx32, dx16, ctx.mask, B, L, cos_t, sin_t, acc)
            del a
            bank.bucket_ready(f"L{l}.")                                                # this layer's four weight gradients are final
        ops.embed_scatter_add_(dx32, ctx.ids, bank.g("embed"))
        bank.end_backward()
