"""Full fine-tuning parameter bank.

The reference's default (`use_peft=None`, dalm/training/rag_e2e/train_rage2e.py:229-260; `--no-use-peft`,
dalm/training/retriever_only/train_retriever_only.py:175-203) trains EVERY parameter of the wrapped HF model with
torch.optim.Adam (train_rage2e.py:336). Here all parameters of one model live in three flat device buffers with identical
element offsets:

  p32  fp32 master weights  (what Adam updates; biases / norm gains are read by the kernels straight from here)
  g32  fp32 gradients       (weight gradients are written by the wgrad GEMM epilogue, the rest accumulated by atomics)
  p16  bf16 shadow          (what the wgmma GEMMs / embedding gathers read; refreshed by the Adam kernel itself)

so the optimizer is one launch and the data-parallel all-reduce one contiguous range per model. Entries of kind "acc"
(bias, norm and embedding gradients: accumulated with atomics, so they must start from zero) are laid out first; entries of
kind "gemm" follow: a fresh gradient of those is WRITTEN by the first wgrad of a step (no 27 GB memset at 7B) and
accumulated into by later ones (second encoder call of the un-fused API path, gradient accumulation).
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import torch

f32, bf16 = torch.float32, torch.bfloat16
_ALIGN = 64                      # elements: 256 B in fp32, 128 B in bf16 (TMA base alignment is 16 B, rows 128 B)


class DenseBank:
    def __init__(self, specs: Sequence[Tuple[str, Tuple[int, ...], str]], device):
        """specs: (key, shape, kind) with kind in {"acc", "gemm"}"""
        self.device = torch.device(device)
        self.shape: Dict[str, Tuple[int, ...]] = {}
        self.off: Dict[str, int] = {}
        self.kind: Dict[str, str] = {}
        off = 0
        for want in ("acc", "gemm"):
            for key, shape, kind in specs:
                if kind != want:
                    continue
                if key in self.off:
                    raise ValueError(f"duplicate parameter key {key}")
                n = 1
                for s in shape:
                    n *= int(s)
                self.shape[key], self.off[key], self.kind[key] = tuple(int(s) for s in shape), off, kind
                off += (n + _ALIGN - 1) // _ALIGN * _ALIGN
            if want == "acc":
                self.n_acc = off
        self.total = off
        self.p32 = torch.zeros(off, dtype=f32, device=self.device)
        self.g32 = torch.zeros(off, dtype=f32, device=self.device)
        self.p16 = torch.zeros(off, dtype=bf16, device=self.device)
        self.fresh = True                   # no gradient has been written since the last zero_grad()
        self.force_accumulate = False       # gradient accumulation under a captured graph: always +=, zero everything
        # data-parallel overlap (accel.GradientSync): the engine announces, during backward, every contiguous range of g32
        # whose gradients are final ("bucket = layer", SURVEY 8e); the hook all-reduces it on a side stream while the
        # backward of the layers below is still running. Ranges not announced are reduced at the end of the step.
        self.bucket_hook = None
        self.reduced: List[Tuple[int, int]] = []

    def _view(self, buf: torch.Tensor, key: str) -> torch.Tensor:
        shape = self.shape[key]
        n = 1
        for s in shape:
            n *= s
        return buf[self.off[key]:self.off[key] + n].view(shape)

    def w32(self, key: str) -> torch.Tensor:
        return self._view(self.p32, key)

    def w16(self, key: str) -> torch.Tensor:
        return self._view(self.p16, key)

    def g(self, key: str) -> torch.Tensor:
        return self._view(self.g32, key)

    @property
    def grad(self) -> torch.Tensor:
        """flat gradient buffer (same attribute name as LoraBank: what the data-parallel all-reduce touches)"""
        return self.g32

    def keys(self) -> List[str]:
        return list(self.off)

    def numel(self) -> int:
        """parameters (without alignment padding)"""
        n = 0
        for shape in self.shape.values():
            k = 1
            for s in shape:
                k *= s
            n += k
        return n

    def sync_shadow(self) -> None:
        """bf16 shadow <- fp32 master (load time / after a checkpoint restore; the training step never needs it: the Adam
        kernel writes both)"""
        self.p16.copy_(self.p32)

    # ---- data-parallel buckets ------------------------------------------------------------------------------------
    def gemm_range(self, prefix: str) -> Tuple[int, int]:
        """[lo, hi) element range of the "gemm"-kind entries whose key starts with `prefix` (one layer's weight gradients:
        contiguous by construction, specs are laid out layer by layer)"""
        lo, hi = None, None
        for key, off in self.off.items():
            if self.kind[key] == "gemm" and key.startswith(prefix):
                n = 1
                for d in self.shape[key]:
                    n *= d
                lo = off if lo is None else min(lo, off)
                hi = off + n if hi is None else max(hi, off + n)
        if lo is None:
            raise KeyError(f"no weight-gradient entries under {prefix!r}")
        return lo, hi

    def bucket_ready(self, prefix: str) -> None:
        """called by the engine's backward once every gradient under `prefix` has been written"""
        if self.bucket_hook is not None:
            lo, hi = self.gemm_range(prefix)
            self.bucket_hook(self, lo, hi)

    def unreduced_ranges(self) -> List[Tuple[int, int]]:
        """complement of the announced (already reduced) ranges in [0, total)"""
        out, pos = [], 0
        for lo, hi in sorted(self.reduced):
            if lo > pos:
                out.append((pos, lo))
            pos = max(pos, hi)
        if pos < self.total:
            out.append((pos, self.total))
        return out

    # ---- gradient freshness protocol ----------------------------------------------------------------------------
    def zero_grad(self) -> None:
        if self.force_accumulate:
            self.g32.zero_()
        else:
            self.g32[: self.n_acc].zero_()
        self.fresh = True

    def begin_backward(self) -> bool:
        """-> True if the weight-gradient GEMMs of this backward call must accumulate (+=) instead of write"""
        return self.force_accumulate or not self.fresh

    def end_backward(self) -> None:
        self.fresh = False
