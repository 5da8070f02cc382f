"""ModernBERT encoder (gte-modernbert-base, modernbert-embed-base / -large, ModernBERT-base / -large) forward + backward as a
launch sequence over the C-ABI kernels. It offers its callers the interface of BertEncoder, so EncodeFn, the trainers, the
data-parallel buckets and the CUDA-graph step serve it unchanged.

Mirrors what `self.model(input_ids, attention_mask)[0]` computes through HF ModernBertModel (transformers 5.5):
tok_embeddings -> LayerNorm -> N x [h += Wo(attn(attn_norm(h))) ; h += mlp.Wo(gelu(in) * gate), in|gate = mlp.Wi(mlp_norm(h))]
-> final_norm. Pre-norm, LayerNorms without bias, no position table: RoPE (rotate_half over the whole head, positions =
column index) on q and k with the layer type's theta, scale head_dim ** -0.5, non-causal attention over the key-padding mask,
and on local layers the bidirectional window |i - j| <= local_attention // 2. Layer 0 has no attn_norm.

Modes: frozen (bf16 weights only: eval-retriever, eval-rag) and full fine-tuning (every parameter in a DenseBank). LoRA is
refused, like peft refuses it: the reference's retriever targets (query / key / value) do not exist in ModernBERT.
Activations: residual stream fp32, GEMM operands bf16.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import ops
from . import params
from .dense import DenseBank

bf16, f32 = torch.bfloat16, torch.float32

LORA_REFUSAL = ("ModernBERT retrievers with LoRA are not built: the reference's retriever LoRA targets (query / key / value) do "
                "not exist in ModernBERT, so get_peft_model refuses them too. Fine-tune the retriever fully (--no-use-peft, or "
                "use_peft=generator)")


def _hf_names(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """checkpoint names relative to ModernBertModel: the `model.` prefix of ModernBertForMaskedLM checkpoints stripped, its
    masked-LM head (`head.*`, `decoder.*`) left out, as AutoModel leaves it out"""
    out = {}
    for k, v in sd.items():
        if k.startswith("model."):
            k = k[len("model."):]
        elif k.startswith(("head.", "decoder.")):
            continue
        out[k] = v
    return out


class _Ctx:
    """activations of one forward call kept for its backward"""
    pass


class ModernBertEncoder(torch.nn.Module):
    def __init__(self, cfg: Dict, state_dict: Dict[str, torch.Tensor], device="cuda", lora: bool = False, full: bool = False):
        """full: every parameter trainable (the reference's behaviour without --use-peft); otherwise frozen"""
        super().__init__()
        if lora:
            raise NotImplementedError(LORA_REFUSAL)
        params.check_modernbert(cfg)
        self.cfg = cfg
        self.H = H = cfg["hidden_size"]
        self.F = cfg["intermediate_size"]
        self.nl = cfg["num_hidden_layers"]
        self.nh = cfg["num_attention_heads"]
        self.hd = H // self.nh
        self.V = cfg["vocab_size"]
        self.eps = float(cfg.get("norm_eps", 1e-5))
        self.pad = int(cfg.get("pad_token_id", 50283))
        self.dev = torch.device(device)
        spec = params.modernbert_layers(cfg)
        self.windows = [w for w, _ in spec]
        self.inv_freq = [f for _, f in spec]
        self._rope_cache: Dict[tuple, tuple] = {}
        self.zero_b = torch.zeros(H, dtype=f32, device=self.dev)     # the LayerNorm kernels' bias operand (norm_bias=False)
        self.lora = None
        self.nf4 = None
        self.full: Optional[DenseBank] = None
        self.layers: List[Dict[str, torch.Tensor]] = []
        sd = _hf_names(state_dict)
        if full:
            self._init_full(sd)
        else:
            g = lambda k, dt: sd[k].to(device=self.dev, dtype=dt).contiguous()
            self.tok, self.emb_g, self.final_g = g("embeddings.tok_embeddings.weight", bf16), g("embeddings.norm.weight", f32), \
                g("final_norm.weight", f32)
            for l in range(self.nl):
                p = f"layers.{l}."
                self.layers.append({"attn_g": g(p + "attn_norm.weight", f32) if l > 0 else None,
                                    "Wqkv": g(p + "attn.Wqkv.weight", bf16), "Wo": g(p + "attn.Wo.weight", bf16),
                                    "mlp_g": g(p + "mlp_norm.weight", f32), "Wi": g(p + "mlp.Wi.weight", bf16),
                                    "Wo2": g(p + "mlp.Wo.weight", bf16)})
        self.drop_offset = torch.zeros(1, dtype=torch.int64, device=self.dev)   # no dropout; kept for the step's interface
        self.eval()

    # ---- what is trainable ---------------------------------------------------------------------------------------
    @property
    def trainable(self) -> bool:
        return self.full is not None

    @property
    def anchor(self) -> torch.nn.Parameter:
        """the flat parameter that ties engine outputs to the autograd graph (bridge.py)"""
        return self.full_flat

    def grad_buffers(self) -> List[torch.Tensor]:
        return [self.full.grad] if self.full is not None else []

    def banks(self) -> list:
        return [self.full] if self.full is not None else []

    def zero_grad_buffers(self) -> None:
        if self.full is not None:
            self.full.zero_grad()

    def repack_lora(self) -> None:
        pass

    def enable_lora(self, lora_seed: int = 0) -> None:
        raise NotImplementedError(LORA_REFUSAL)

    def _param_map(self):
        """engine tensor -> (gradient kind, HF ModernBertModel name)"""
        m = [("tok", "acc", "embeddings.tok_embeddings.weight"), ("emb_g", "acc", "embeddings.norm.weight"),
             ("final_g", "acc", "final_norm.weight")]
        for l in range(self.nl):
            p = f"layers.{l}."
            if l > 0:
                m.append((f"L{l}.attn_g", "acc", p + "attn_norm.weight"))
            m += [(f"L{l}.mlp_g", "acc", p + "mlp_norm.weight"), (f"L{l}.Wqkv", "gemm", p + "attn.Wqkv.weight"),
                  (f"L{l}.Wo", "gemm", p + "attn.Wo.weight"), (f"L{l}.Wi", "gemm", p + "mlp.Wi.weight"),
                  (f"L{l}.Wo2", "gemm", p + "mlp.Wo.weight")]
        return m

    def _init_full(self, sd) -> None:
        pm = self._param_map()
        bank = DenseBank([(key, tuple(sd[name].shape), kind) for key, kind, name in pm], self.dev)
        for key, _, name in pm:
            bank.w32(key).copy_(sd[name].to(self.dev, f32))
        bank.sync_shadow()
        self._names = {key: name for key, _, name in pm}
        self.full = bank
        self.full_flat = torch.nn.Parameter(bank.p32, requires_grad=True)
        self.full_flat.grad = bank.g32
        self.full_flat._dalm_bank = bank
        self.tok, self.emb_g, self.final_g = bank.w16("tok"), bank.w32("emb_g"), bank.w32("final_g")
        for l in range(self.nl):
            k = lambda n: f"L{l}.{n}"
            self.layers.append({"attn_g": bank.w32(k("attn_g")) if l > 0 else None, "Wqkv": bank.w16(k("Wqkv")),
                                "Wo": bank.w16(k("Wo")), "mlp_g": bank.w32(k("mlp_g")), "Wi": bank.w16(k("Wi")),
                                "Wo2": bank.w16(k("Wo2"))})

    def hf_state_dict(self) -> Dict[str, torch.Tensor]:
        """fp32 CPU tensors under HF ModernBertModel names (save_pretrained of a fully fine-tuned encoder)"""
        if self.full is None:
            raise RuntimeError("hf_state_dict: only fully fine-tuned models own their weights")
        return {name: self.full.w32(key).detach().cpu().clone() for key, name in self._names.items()}

    def load_hf_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        sd = _hf_names(sd)
        for key, name in self._names.items():
            self.full.w32(key).copy_(sd[name].to(self.dev, f32))
        self.full.sync_shadow()

    def _rope(self, l: int, L: int):
        """fp32 cos / sin tables [L, hd/2] of layer l's type (global and local layers differ in theta), cached per length"""
        key = (self.windows[l] > 0, L)
        if key not in self._rope_cache:
            fr = torch.outer(torch.arange(L, dtype=torch.float32), self.inv_freq[l])
            self._rope_cache[key] = (fr.cos().to(self.dev).contiguous(), fr.sin().to(self.dev).contiguous())
        return self._rope_cache[key]

    # ------------------------------------------------------------------------------------------------------------
    def forward_hidden(self, ids: torch.Tensor, mask: torch.Tensor, save: bool = True):
        """ids, mask: int64 [B,L] on device -> (hidden fp32 [B,L,H], ctx)"""
        hs, ctx = self.forward_segments([(ids, mask)], save=save)
        return hs[0], ctx

    def forward_segments(self, segments, save: bool = True):
        """Several (ids, mask) batches with different sequence lengths through one pass over the weights: the linear layers,
        norms and activations run on the concatenated token rows; RoPE and attention are launched per segment.
        Returns ([hidden_i fp32 [B_i,L_i,H]], ctx)."""
        H, F, nh, hd = self.H, self.F, self.nh, self.hd
        ctx = _Ctx()
        ctx.segs, r0 = [], 0
        for ids, mask in segments:
            B, L = ids.shape
            ctx.segs.append((B, L, mask.contiguous(), r0))
            r0 += B * L
        M = ctx.M = r0
        ctx.layers = []
        z = torch.empty(M, H, dtype=f32, device=self.dev)
        for (ids, _), (B, L, _, s0) in zip(segments, ctx.segs):
            ops.embed_gather(ids.contiguous(), self.tok, out=z[s0:s0 + B * L])
        h, x16, me, re = ops.layernorm_fwd(z, self.emb_g, self.zero_b, self.eps)
        if save:
            ctx.z_emb, ctx.mean_e, ctx.rstd_e = z, me, re
            ctx.ids = [ids.contiguous() for ids, _ in segments]
        for l, W in enumerate(self.layers):
            a = _Ctx()
            if l == 0:                                          # attn_norm = Identity: the embedding LN output itself
                hn16, m_a, r_a = x16, None, None
            else:
                _, hn16, m_a, r_a = ops.layernorm_fwd(h, W["attn_g"], self.zero_b, self.eps, want_f32=False)
            qkv = ops.gemm(hn16, W["Wqkv"])                                                     # [M, 3H] q | k | v
            att = torch.empty(M, H, dtype=bf16, device=self.dev)
            lses = []
            for B, L, mask, s0 in ctx.segs:
                rows = slice(s0, s0 + B * L)
                cos_t, sin_t = self._rope(l, L)
                ops.rope_(qkv[rows], 0, 2 * nh, hd, cos_t, sin_t, L)                            # q heads then k heads
                _, lse = ops.attention_auto_fwd(qkv[rows, :H], qkv[rows, H:2 * H], qkv[rows, 2 * H:], mask, B, L, nh, nh, hd,
                                                causal=False, out=att[rows], window=self.windows[l], bidirectional=True)
                lses.append(lse)
            h1 = ops.gemm(att, W["Wo"], out_dtype=f32, resid=h)
            _, mn16, m_m, r_m = ops.layernorm_fwd(h1, W["mlp_g"], self.zero_b, self.eps, want_f32=False)
            xg = ops.gemm(mn16, W["Wi"])                                                       # [M, 2F] input | gate
            act = ops.geglu_fwd(xg, F)
            h2 = ops.gemm(act, W["Wo2"], out_dtype=f32, resid=h1)
            if save:
                a.h, a.m_a, a.r_a, a.hn16, a.qkv, a.att, a.lse, a.h1, a.m_m, a.r_m, a.mn16, a.xg, a.act = \
                    h, m_a, r_a, hn16, qkv, att, lses, h1, m_m, r_m, mn16, xg, act
                ctx.layers.append(a)
            h = h2
        out, _, mf, rf = ops.layernorm_fwd(h, self.final_g, self.zero_b, self.eps)
        if save:
            ctx.h_last, ctx.mean_f, ctx.rstd_f = h, mf, rf
        return [out[s0:s0 + B * L].view(B, L, H) for (B, L, _, s0) in ctx.segs], ctx

    # ------------------------------------------------------------------------------------------------------------
    def backward_hidden(self, ctx: _Ctx, d_hidden: torch.Tensor) -> None:
        """d_hidden fp32 [B,L,H]; accumulates every parameter's gradient into the DenseBank (full fine-tuning)"""
        self.backward_segments(ctx, [d_hidden])

    def backward_segments(self, ctx: _Ctx, d_hiddens) -> None:
        if not self.trainable:
            return
        M, H, nh, hd = ctx.M, self.H, self.nh, self.hd
        bank = self.full
        G = lambda key: bank.g(key)
        d = d_hiddens[0].reshape(-1, H) if len(d_hiddens) == 1 else torch.cat([t.reshape(-1, H) for t in d_hiddens], 0)
        d = d.contiguous()
        acc = bank.begin_backward()
        ops.col_reduce_(dy_f32=d, z=ctx.h_last, mean=ctx.mean_f, rstd=ctx.rstd_f, out_prod=G("final_g"))
        dh32, dh16 = ops.layernorm_bwd(ctx.h_last, self.final_g, ctx.mean_f, ctx.rstd_f, dy_f32=d)   # d(residual stream)
        for l in range(self.nl - 1, -1, -1):
            W, a = self.layers[l], ctx.layers[l]
            # ---- h2 = h1 + mlp.Wo(gelu(in) * gate) ----
            ops.wgrad_(dh16, a.act, G(f"L{l}.Wo2"), acc)
            dact = ops.gemm(dh16, W["Wo2"], layout=1)
            ops.geglu_bwd_(a.xg, dact, self.F)                                                  # xg <- [d in | d gate]
            ops.wgrad_(a.xg, a.mn16, G(f"L{l}.Wi"), acc)
            dmn16 = ops.gemm(a.xg, W["Wi"], layout=1)
            ops.col_reduce_(dy_bf16=dmn16, z=a.h1, mean=a.m_m, rstd=a.r_m, out_prod=G(f"L{l}.mlp_g"))
            dh32, dh16 = ops.layernorm_bwd_res(a.h1, W["mlp_g"], a.m_m, a.r_m, dmn16, dh32, dz32=dh32)
            # ---- h1 = h + Wo(attn(rope(Wqkv(attn_norm(h))))) ----
            ops.wgrad_(dh16, a.att, G(f"L{l}.Wo"), acc)
            datt = ops.gemm(dh16, W["Wo"], layout=1)
            dqkv = torch.empty(M, 3 * H, dtype=bf16, device=self.dev)
            for (B, L, mask, s0), lse in zip(ctx.segs, a.lse):
                rows = slice(s0, s0 + B * L)
                ops.attention_auto_bwd(a.qkv[rows, :H], a.qkv[rows, H:2 * H], a.qkv[rows, 2 * H:], mask, a.att[rows], lse,
                                       datt[rows], B, L, nh, nh, hd, causal=False, dq=dqkv[rows, :H], dk=dqkv[rows, H:2 * H],
                                       dv=dqkv[rows, 2 * H:], window=self.windows[l], bidirectional=True)
                cos_t, sin_t = self._rope(l, L)
                ops.rope_(dqkv[rows], 0, 2 * nh, hd, cos_t, sin_t, L, backward=True)
            ops.wgrad_(dqkv, a.hn16, G(f"L{l}.Wqkv"), acc)
            dhn16 = ops.gemm(dqkv, W["Wqkv"], layout=1)
            bank.bucket_ready(f"L{l}.")                                    # this layer's four weight gradients are final
            if l > 0:
                ops.col_reduce_(dy_bf16=dhn16, z=a.h, mean=a.m_a, rstd=a.r_a, out_prod=G(f"L{l}.attn_g"))
                dh32, dh16 = ops.layernorm_bwd_res(a.h, W["attn_g"], a.m_a, a.r_a, dhn16, dh32, dz32=dh32)
            else:
                dh32 = ops.masked_add(dh32, dhn16, out=dh32)                 # Identity attn_norm: both paths reach the LN output
        ops.col_reduce_(dy_f32=dh32, z=ctx.z_emb, mean=ctx.mean_e, rstd=ctx.rstd_e, out_prod=G("emb_g"))
        dz, _ = ops.layernorm_bwd(ctx.z_emb, self.emb_g, ctx.mean_e, ctx.rstd_e, dy_f32=dh32, want_bf16=False)
        for ids, (B, L, _, s0) in zip(ctx.ids, ctx.segs):                   # the padding_idx row gets no gradient
            ops.embed_scatter_add_(dz[s0:s0 + B * L], ids, G("tok"), None, L, pad_id=self.pad)
        bank.end_backward()
