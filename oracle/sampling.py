"""fp64 restatement of HF's sampling warpers and of the draw `dalm_b200_sample_step` makes. TEST INFRASTRUCTURE ONLY (see
oracle/__init__.py).

transformers 5.5 `_get_logits_processor` (do_sample=True, num_beams=1) applies, in this order:
  TemperatureLogitsWarper  x = scores / temperature            (fp32, as HF divides the fp32 scores; skipped at T == 1)
  TopKLogitsWarper         remove x < the k-th largest x        (0 < top_k < V; ties at the k-th value are all kept)
  TopPLogitsWarper         ascending order, remove while the cumulative softmax share <= 1 - top_p, keep the last one
                                                               (top_p < 1)
HF sorts with an unstable `torch.sort`; here the order is (x, index) ascending, the library's rule for a tie group that
straddles the top-p cut. Shares are computed in fp64. The draw: the first kept index, ascending, whose inclusive prefix sum
of exp(x - max) exceeds u * Z.
"""
from __future__ import annotations

import numpy as np
import torch


def warp(logits, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0) -> np.ndarray:
    """logits [..., V] (any float dtype) -> fp64 warped scores, -inf where removed; kept values are the fp32 x exactly"""
    x32 = torch.as_tensor(logits).float()
    if temperature != 1.0:
        x32 = x32 / float(temperature)
    x = x32.double().numpy().copy()
    rows = x.reshape(-1, x.shape[-1])
    V = rows.shape[1]
    for r in rows:
        if 0 < top_k < V:
            kth = np.sort(r)[-top_k]
            r[r < kth] = -np.inf
        if top_p < 1.0:
            order = np.lexsort((np.arange(V), r))              # ascending by (x, index)
            s = r[order]
            fin = np.isfinite(s)
            p = np.zeros(V)
            p[fin] = np.exp(s[fin] - s[fin].max())
            cum = np.cumsum(p / p.sum())
            remove = cum <= 1.0 - top_p
            remove[-1] = False                                # min_tokens_to_keep = 1
            r[order[remove]] = -np.inf
    return x


def probs(warped: np.ndarray) -> np.ndarray:
    """softmax of the warped scores (fp64)"""
    w = np.where(np.isfinite(warped), np.exp(warped - warped.max(-1, keepdims=True)), 0.0)
    return w / w.sum(-1, keepdims=True)


def choose(warped_row: np.ndarray, u: float) -> int:
    """inverse-CDF choice in ascending index order: first kept index whose inclusive prefix mass exceeds u * Z"""
    kept = np.isfinite(warped_row)
    w = np.where(kept, np.exp(warped_row - warped_row[kept].max()), 0.0)
    c = np.cumsum(w)
    hit = np.nonzero(kept & (w > 0) & (c > u * c[-1]))[0]
    return int(hit[0]) if len(hit) else int(np.nonzero(kept)[0][-1])


def hf_warp(logits, temperature: float, top_k: int, top_p: float) -> torch.Tensor:
    """the installed transformers' own warper stack on fp32 scores, as `_get_logits_processor` builds it"""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.as_tensor(logits).float().reshape(-1, np.shape(logits)[-1])
    ids = torch.zeros(s.shape[0], 1, dtype=torch.long)
    if temperature != 1.0:
        s = TemperatureLogitsWarper(float(temperature))(ids, s)
    if top_k != 0:
        s = TopKLogitsWarper(top_k=int(top_k))(ids, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p=float(top_p))(ids, s)
    return s


def clear_of_cut(logits_row, temperature: float, top_k: int, top_p: float, margin: float = 1e-5, ties_ok: bool = False) -> bool:
    """True when HF's top-p decision on this row cannot depend on summation order: no cumulative share HF computes (the
    always-kept last one aside) lies within `margin` of 1 - top_p. Unless `ties_ok`, also no tie group straddles the cut
    (where HF's unstable sort decides which of the tied tokens go)"""
    if top_p >= 1.0:
        return True
    s = hf_warp(logits_row, temperature, top_k, 1.0)[0]
    cum = torch.sort(s).values.softmax(-1).cumsum(-1)[:-1].double()
    if (cum - (1.0 - top_p)).abs().min().item() <= margin:
        return False
    if ties_ok:
        return True
    w = warp(np.asarray(logits_row, dtype=np.float32), temperature, top_k, top_p).reshape(-1)
    survivors = np.isfinite(warp(np.asarray(logits_row, dtype=np.float32), temperature, top_k, 1.0).reshape(-1))
    x = (torch.as_tensor(logits_row).float() / float(temperature) if temperature != 1.0 else torch.as_tensor(logits_row).float())
    x = x.double().numpy().reshape(-1)
    cut = survivors & ~np.isfinite(w)
    return not np.isin(x[cut], x[np.isfinite(w)]).any()


def straddling_value(logits_row, temperature: float, top_k: int, top_p: float):
    """the x value of a tie group that the top-p cut splits, or None"""
    w = warp(np.asarray(logits_row, dtype=np.float32), temperature, top_k, top_p).reshape(-1)
    s = warp(np.asarray(logits_row, dtype=np.float32), temperature, top_k, 1.0).reshape(-1)
    cut = np.isfinite(s) & ~np.isfinite(w)
    both = np.intersect1d(s[cut], w[np.isfinite(w)])
    return float(both[0]) if len(both) else None


def prefix_mass(warped_row: np.ndarray):
    """(inclusive prefix sums of exp(x - max) over the kept tokens in index order, Z)"""
    kept = np.isfinite(warped_row)
    w = np.where(kept, np.exp(warped_row - warped_row[kept].max()), 0.0)
    c = np.cumsum(w)
    return c, float(c[-1])
