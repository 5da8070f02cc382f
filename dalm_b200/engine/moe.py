"""Qwen3-MoE's routed MLP (Qwen3MoeSparseMoeBlock) on the grouped wgmma GEMM.

A router (`mlp.gate`, fp32 logits) picks the top k of E experts per token; each expert is a SwiGLU MLP with intermediate
size I; a token's output is the routing-weighted sum of its k experts' outputs. Rows are permuted so that each expert's
(token, slot) pairs are contiguous and padded to the GEMM's 128-row tile (`ops.moe_permute`), so each projection is one
grouped launch over all experts, sized for the static bound of padded rows: nothing waits on the host, and the whole layer
can be captured in a CUDA graph.

Memory: the backward keeps the router logits [M, E], the routing, and the experts' gate|up [rows, 2I] and activation
[rows, I] rows. The per-pair expert outputs y [rows, H] are not kept: the routing-weight gradient is
dw = <dy, y> = <W_down^T dy, act>, and W_down^T dy is the down projection's dgrad, which the backward computes anyway.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from .. import ops


@dataclass
class MoeWeights:
    """frozen bf16 weights of one sparse layer: gate [E, H], gate_up [E, 2I, H] (gate / up rows interleaved in 128-feature
    blocks, `ops.interleave_gate_up` per expert), down [E, H, I]"""
    gate: torch.Tensor
    gate_up: torch.Tensor
    down: torch.Tensor
    top_k: int
    norm_topk: bool

    @property
    def num_experts(self) -> int:
        return self.gate.shape[0]

    @property
    def inter(self) -> int:
        return self.down.shape[2]


def pack_experts(gate: torch.Tensor, gate_proj: torch.Tensor, up_proj: torch.Tensor, down_proj: torch.Tensor, top_k: int,
                 norm_topk: bool, device) -> MoeWeights:
    """hub-layout tensors (gate [E, H], gate_proj / up_proj [E, I, H], down_proj [E, H, I]) -> bf16 device weights"""
    to = lambda t: t.to(device=device, dtype=torch.bfloat16).contiguous()
    gu = torch.stack([ops.interleave_gate_up(to(g), to(u)) for g, u in zip(gate_proj, up_proj)])
    return MoeWeights(to(gate), gu.contiguous(), to(down_proj), int(top_k), bool(norm_topk))


@dataclass
class MoeSaved:
    logits: torch.Tensor          # fp32 [M, E]
    ids: torch.Tensor             # int32 [M, k]
    w: torch.Tensor               # fp32 [M, k]
    routing: ops.MoeRouting
    gu: torch.Tensor              # bf16 [rows, 2I] interleaved gate|up; overwritten by its gradient in the backward
    act: torch.Tensor             # bf16 [rows, I]


def forward(x: torch.Tensor, mw: MoeWeights, resid: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
            routing: Optional[ops.MoeRouting] = None, max_ctas: int = 0):
    """out = resid + MoE(x). x: bf16 [M, H] (the post-attention RMSNorm output); resid / out: fp32 or bf16 [M, H], out may be
    resid. -> (out, MoeSaved)"""
    logits = ops.gemm(x, mw.gate, out_dtype=torch.float32)
    ids, w = ops.moe_router(logits, mw.top_k, mw.norm_topk)
    r = ops.moe_permute(ids, mw.num_experts, routing)
    xr = ops.moe_gather(x, r)
    gu, act = ops.gemm_grouped(xr, mw.gate_up, r.tile_expert, r.live, swiglu=True, max_ctas=max_ctas)
    y = ops.gemm_grouped(act, mw.down, r.tile_expert, r.live, out=xr, max_ctas=max_ctas)   # x rows are dead: reuse them
    out = ops.moe_combine(y, r, w, resid=resid, out=out)
    return out, MoeSaved(logits, ids, w, r, gu, act)


def backward(d_out: torch.Tensor, s: MoeSaved, mw: MoeWeights, dx: Optional[torch.Tensor] = None, max_ctas: int = 0) -> torch.Tensor:
    """gradient of the MoE output (fp32 or bf16 [M, H]) -> dx fp32 [M, H] (added into `dx` when given): the experts' input
    gradient plus the router's, dlogits @ W_gate. Expert and router weights are frozen: no weight gradients."""
    r = s.routing
    g = ops.moe_gather(d_out, r)                                                 # unweighted: dw needs W_down^T dy
    da = ops.gemm_grouped(g, mw.down, r.tile_expert, r.live, layout=1, max_ctas=max_ctas)
    dw, d_act = ops.moe_down_bwd(da, s.act, r, s.w, d_act=s.act)                 # act is read before it is overwritten
    ops.swiglu_bwd_(s.gu, d_act, mw.inter, interleave=128)
    dxr = ops.gemm_grouped(s.gu, mw.gate_up, r.tile_expert, r.live, out=g, layout=1, max_ctas=max_ctas)
    dlogits = ops.moe_router_bwd(s.logits, s.ids, s.w, dw, mw.norm_topk)
    dx = ops.gemm(dlogits, mw.gate, out=dx, out_dtype=torch.float32, resid=dx, layout=1)
    return ops.moe_combine(dxr, r, None, resid=dx, out=dx)
