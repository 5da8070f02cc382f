"""4-bit weight storage for `use_bnb` sub-models (DALM_B200_NF4_STORAGE=1).

The reference's `use_bnb` (rag_e2e_base_model.py:136-142) keeps every nn.Linear weight of the sub-model as NF4 codes and
dequantises it inside each forward (`bnb.matmul_4bit`: dequantize_4bit -> matmul). The default here expands the codes once at
load time and keeps bf16 copies resident (an H100 has the HBM for 7B). This module is the other choice: the base weights stay packed
(0.5625 B per parameter; Llama-2-7B: 3.6 GB instead of 26.5 GB with the dgrad transposes) and one layer's worth of bf16
scratch is shared by all layers - a weight is expanded right before the GEMM that reads it, forward and backward. The values
the GEMMs see are bit-identical to the resident mode (csrc/nf4.cu). The backward reads W[out,in] itself as an MN-major operand
(GEMM layout 1), so no transposed copies exist in this mode.
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Tuple

import torch

from .. import ops

bf16, f32 = torch.bfloat16, torch.float32


def storage_enabled() -> bool:
    return os.environ.get("DALM_B200_NF4_STORAGE", "0") == "1"


class Nf4Store:
    """packed weights of one model + the shared scratch. `slot` names one scratch buffer (one per weight kind: every layer's
    `Wo` expands into the same [H, H] buffer; stream order keeps a layer's GEMM ahead of the next layer's expansion)."""

    def __init__(self, device):
        self.dev = torch.device(device)
        self.q: Dict[Tuple[int, str], Tuple[torch.Tensor, torch.Tensor, int, int]] = {}
        self.tails: Dict[Tuple[int, str], torch.Tensor] = {}
        self.slots: Dict[str, torch.Tensor] = {}

    def put(self, layer: int, name: str, w: torch.Tensor, tail_cols: int = 0) -> None:
        """w: [rows, cols] (any float dtype, ORIGINAL checkpoint values). tail_cols > 0 reserves a per-layer bf16 [rows, tail_cols]
        block (zero) that is appended behind each expanded row (K-augmented weights: the LoRA columns)"""
        w32 = w.to(device=self.dev, dtype=f32).contiguous()
        rows, cols = w32.shape
        if cols % 64:
            raise NotImplementedError(f"NF4 storage: {name} has {cols} input features; blocks of 64 must not straddle rows")
        packed, absmax = ops.nf4_quantize(w32)
        self.q[(layer, name)] = (packed, absmax, rows, cols)
        if tail_cols:
            self.tails[(layer, name)] = torch.zeros(rows, tail_cols, dtype=bf16, device=self.dev)
        ld = cols + (64 if tail_cols else 0)                 # same 128-byte row alignment as engine _aug_buf
        cur = self.slots.get(name)
        if cur is None or cur.shape[0] < rows or cur.shape[1] < ld:
            self.slots[name] = torch.empty(max(rows, 0 if cur is None else cur.shape[0]), max(ld, 0 if cur is None else cur.shape[1]),
                                           dtype=bf16, device=self.dev)

    def tail(self, layer: int, name: str) -> Optional[torch.Tensor]:
        return self.tails.get((layer, name))

    def has(self, layer: int, name: str) -> bool:
        return (layer, name) in self.q

    def get(self, layer: int, name: str) -> torch.Tensor:
        """expand (layer, name) into its slot on the current stream -> bf16 view [rows, cols (+ tail)]"""
        packed, absmax, rows, cols = self.q[(layer, name)]
        tail = self.tails.get((layer, name))
        out = self.slots[name][:rows]
        ops.nf4_dequant_(packed, absmax, rows, cols, out, tail)
        return out[:, :cols + (tail.shape[1] if tail is not None else 0)]

    def nbytes(self) -> int:
        n = sum(p.numel() + a.numel() * 4 for p, a, _, _ in self.q.values())
        n += sum(t.numel() * 2 for t in self.tails.values()) + sum(s.numel() * 2 for s in self.slots.values())
        return n


class QuantLayer(dict):
    """a layer's weight dict whose big matrices are fetched from the Nf4Store on access (everything else is a plain entry)"""

    def __init__(self, store: Nf4Store, layer: int):
        super().__init__()
        self.store, self.layer = store, layer

    def __getitem__(self, k):
        if self.store.has(self.layer, k):
            return self.store.get(self.layer, k)
        return dict.__getitem__(self, k)

    def __contains__(self, k):
        return self.store.has(self.layer, k) or dict.__contains__(self, k)
