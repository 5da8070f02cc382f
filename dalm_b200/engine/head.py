"""Chunked lm_head + vocabulary cross-entropy: the marginalised-NLL head of the fused step without a [B,L,V] tensor.

The reference materialises fp32 logits [B,L,V] and three more copies of them (train_utils.py:113-138: `log_softmax`, the
per-sample `cat`, the `stack`) — 590 MB each at cfg-3, 9.6 GB each at cfg-5. Here the token rows are processed in
chunks of whole 128-row GEMM tiles:

    logits_chunk = hf[r0:r1] @ W_head^T          wgmma GEMM into a scratch sized for the L2
    ce_rows(logits_chunk)                        log-softmax + gather + mask weights; d(logits) written IN PLACE
    dhf[r0:r1]   = dlogits_chunk @ W_head        head dgrad straight from the same scratch
    dW_head     += dlogits_chunk^T @ hf[r0:r1]   (full fine-tuning only)

so forward, loss and the head's backward are one sweep over the rows; what survives it is tok_lp [B,L] (fp32) and
dhf [M,H] (bf16). The scratch is re-used by every chunk and, in PEFT mode, sized to fit the H100's 50 MB L2 between the three
launches that touch it; whatever part of a chunk is evicted anyway costs one extra pass over the scratch, not the reference's
four [B,L,V] tensors. The gain is the memory and the absence of a V-sized tensor.
"""
from __future__ import annotations

import os
from typing import Callable, Optional, Tuple

import torch

from .. import ops

bf16, f32 = torch.bfloat16, torch.float32

# scratch budgets (bytes of bf16 logits per chunk): frozen head -> sized to sit in L2 next to the streaming weight panels
# (24 MB: about half of the H100's 50 MB L2; an estimate, not a measured optimum); trainable head -> larger chunks, because
# every chunk's wgrad re-reads and re-writes the fp32 [V,H] gradient
L2_BUDGET = int(os.environ.get("DALM_B200_HEAD_CHUNK_MB", "24")) << 20
FULL_BUDGET = int(os.environ.get("DALM_B200_HEAD_CHUNK_FULL_MB", "512")) << 20


def chunked_head_loss(hf: torch.Tensor, w_head: torch.Tensor, w_headT: Optional[torch.Tensor], V: int, ids: torch.Tensor,
                      mask: torch.Tensor, nsum: torch.Tensor, need_grad: bool, grad_out: float = 1.0,
                      wgrad: Optional[Callable[[torch.Tensor, torch.Tensor, bool], None]] = None,
                      budget: Optional[int] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """hf bf16 [M,H] (final-norm output), w_head bf16 [Vp,H] (rows >= V are zero), w_headT its resident transpose [H,Vp] or
    None (then the dgrad reads w_head MN-major); ids / mask int64 [B,L]; nsum fp32 [1] = sum(mask[:,1:]).
    wgrad(dl_chunk [n,Vp], hf_chunk [n,H], first) accumulates the head's weight gradient (full fine-tuning).
    -> (tok_lp fp32 [B,L], dhf bf16 [M,H] or None)"""
    B, L = ids.shape
    M, H = hf.shape
    Vp = w_head.shape[0]
    if M != B * L:
        raise ValueError(f"chunked_head_loss: {M} hidden rows for a {B} x {L} batch")
    ids, mask = ids.contiguous(), mask.contiguous()
    if budget is None:
        budget = FULL_BUDGET if wgrad is not None else L2_BUDGET
    rows = min(ops.head_chunk_rows(M, Vp, budget), (M + 127) // 128 * 128)
    scratch = torch.empty(min(rows, M), Vp, dtype=bf16, device=hf.device)
    tok_lp = torch.empty(B, L, dtype=f32, device=hf.device)
    dhf = torch.empty(M, H, dtype=bf16, device=hf.device) if need_grad else None
    for r0 in range(0, M, rows):
        n = min(rows, M - r0)
        lg = scratch[:n]
        ops.gemm(hf[r0:r0 + n], w_head, out=lg)                                   # logits of these rows (pad columns: zero rows of W)
        ops.ce_marginal_rows_(lg, ids, mask, nsum, tok_lp, r0, V, need_grad=need_grad, grad_out=grad_out)
        if not need_grad:
            continue
        if wgrad is not None:
            wgrad(lg, hf[r0:r0 + n], r0 == 0)
        if w_headT is not None:
            ops.gemm(lg, w_headT, out=dhf[r0:r0 + n])
        else:
            ops.gemm(lg, w_head, out=dhf[r0:r0 + n], layout=1)
    return tok_lp, dhf
