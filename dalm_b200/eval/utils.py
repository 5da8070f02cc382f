"""Retrieval evaluation helpers — same names, arguments and return values as the reference's dalm/eval/utils.py:18-295.

The one semantic change: the reference builds an APPROXIMATE hnswlib index (space "ip", M=100, ef_construction=200, ef=100,
dalm/eval/utils.py:18-55) on the host; here `construct_search_index` keeps the passage embeddings resident in HBM and
`get_nearest_neighbours` runs an EXACT inner-product top-k sweep over them (csrc/topk.cu: one pass over 200k x 1024 fp32 is
819 MB, about 0.25 ms at the H100's 3.35 TB/s data-sheet bandwidth). Exact search is the limit hnswlib approximates, so recall / precision / hit-rate computed
from it are >= the reference's for the same embeddings.
"""
from __future__ import annotations

import logging
from typing import Any, Callable, Dict, List, Tuple

import numpy as np
import torch
from torch.utils.data import DataLoader

from .. import ops
from .eval_results import EvalResults

logger = logging.getLogger(__name__)


class ExactIndex:
    """stands where hnswlib.Index stands in the reference: holds the passages, answers knn_query(queries, k)"""

    def __init__(self, dim: int, num_elements: int, device=None):
        from ..models.rag_e2e_base_model import _device

        self.dim, self.num_elements = int(dim), int(num_elements)
        self.device = device if device is not None else _device()
        self.data = torch.empty(self.num_elements, self.dim, dtype=torch.float32, device=self.device)
        self.count = 0
        self.ef = None

    def add_items(self, data, ids=None) -> None:
        t = torch.as_tensor(np.asarray(data), dtype=torch.float32)
        n = t.shape[0]
        if ids is not None and not np.array_equal(np.asarray(ids), np.arange(self.count, self.count + n)):
            raise ValueError("ExactIndex stores rows in insertion order: ids must be consecutive")
        if self.count + n > self.num_elements:
            raise RuntimeError("The number of elements exceeds the specified limit")          # hnswlib's message
        self.data[self.count:self.count + n].copy_(t)
        self.count += n

    def set_ef(self, ef: int) -> None:                       # accepted for API compatibility; the search is exact
        self.ef = ef

    def knn_query(self, queries, k: int = 1) -> Tuple[np.ndarray, np.ndarray]:
        """-> (labels [nq,k] int, distances [nq,k] float32 = 1 - inner product, ascending): hnswlib's 'ip' convention"""
        if k > self.count:
            raise RuntimeError("Cannot return the results in a contiguous 2D array. Probably ef or M is too small")
        q = torch.as_tensor(np.asarray(queries), dtype=torch.float32).to(self.device)
        if q.dim() == 1:
            q = q[None]
        scores, idx = ops.topk_ip(q, self.data[: self.count], k)
        return idx.cpu().numpy().astype(np.int64), (1.0 - scores).cpu().numpy()


def construct_search_index(dim: int, num_elements: int, data: np.ndarray) -> ExactIndex:
    """reference :18-42"""
    search_index = ExactIndex(dim, num_elements)
    search_index.add_items(data, np.arange(num_elements))
    return search_index


def get_nearest_neighbours(k: int, search_index: ExactIndex, query_embeddings: np.ndarray, ids_to_cat_dict: Dict[int, Any],
                           threshold: float = 0.7) -> List[List[Tuple[str, float]]]:
    """reference :45-66: per query the (item, similarity) pairs of its k nearest rows whose similarity 1 - distance reaches
    `threshold`, best first"""
    search_index.set_ef(100)
    labels, distances = search_index.knn_query(query_embeddings, k=k)
    sims = 1 - distances
    return [[(ids_to_cat_dict[int(row)], sim) for row, sim in zip(rows, row_sims, strict=True) if sim >= threshold]
            for rows, row_sims in zip(labels, sims)]


def calculate_precision_recall(retrieved_items: List, correct_items: List) -> Tuple[float, float]:
    """reference :69-81: set precision / recall (an empty retrieved set divides by zero there too)"""
    got, want = frozenset(retrieved_items), frozenset(correct_items)
    hits = len(got & want)
    return hits / len(got), hits / len(want)


def preprocess_function(examples, retriever_tokenizer, query_column_name: str = "query", passage_column_name: str = "passage",
                        max_length: int = 128) -> Dict[str, Any]:
    """reference :84-108"""
    q = retriever_tokenizer(examples[query_column_name], padding="max_length", max_length=max_length, truncation=True)
    p = retriever_tokenizer(examples[passage_column_name], padding="max_length", max_length=max_length, truncation=True)
    pre_batch = {}
    for k, v in q.items():
        pre_batch[f"retriever_query_{k}"] = v
    for k, v in p.items():
        pre_batch[f"retriever_passage_{k}"] = v
    return pre_batch


def preprocess_dataset(dataset, tokenizer, query_column_name: str, passage_column_name: str, max_length: int):
    """reference :111-130 (single process here: the tokenizer closure must not fork a CUDA context)"""
    return dataset.map(lambda ex: preprocess_function(ex, tokenizer, query_column_name=query_column_name,
                                                      passage_column_name=passage_column_name, max_length=max_length),
                       batched=True, desc="Running tokenizer on dataset")


def filter_unique_passages(dataset, passage_column_name: str):
    """reference :133-143: keeps the FIRST row of every distinct passage, in dataset order"""
    first_row: Dict[Any, int] = {}
    for row, passage in enumerate(dataset[passage_column_name]):
        first_row.setdefault(passage, row)
    return dataset.select(sorted(first_row.values()))


def mixed_collate_fn(batch: List[Dict[str, Any]]) -> Dict[str, Any]:
    """reference :146-162: text (or missing) columns stay python lists, everything else is stacked into a tensor"""
    head = batch[0]
    is_text = {key: isinstance(value, str) or value is None for key, value in head.items()}
    return {key: [sample[key] for sample in batch] if is_text[key] else torch.stack([torch.tensor(sample[key]) for sample in batch])
            for key in head}


def get_retriever_embeddings(forward_fn: Callable[[torch.Tensor, torch.Tensor], torch.Tensor], device: str,
                             retriever_input_ids: torch.Tensor, retriever_attention_masks: torch.Tensor) -> np.ndarray:
    """reference :165-181"""
    return forward_fn(retriever_input_ids.to(device), retriever_attention_masks.to(device)).detach().float().cpu().numpy()


def _int_collate(features: List[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
    keep = [k for k, v in features[0].items() if isinstance(v, (list, tuple)) and v and isinstance(v[0], int)]
    return {k: torch.tensor([f[k] for f in features], dtype=torch.int64) for k in keep}


def get_passage_embeddings(passage_dataset, passage_column_name: str, forward_fn, device: str, embed_dim: int,
                           torch_dtype: torch.dtype, batch_size: int):
    """reference :184-220. `torch_dtype` selected the autocast dtype there; dalm_b200's forward is bf16 GEMMs with fp32
    pooling whatever is passed (DESIGN.md)."""
    unique_passage_dataset = filter_unique_passages(passage_dataset, passage_column_name)
    loader = DataLoader(unique_passage_dataset, shuffle=False, collate_fn=_int_collate, batch_size=batch_size)
    num_passages = len(unique_passage_dataset)
    logger.info(f"Starting to generate passage embeddings (Number of passages: {num_passages})")
    out = np.zeros((num_passages, embed_dim))
    for step, batch in enumerate(loader):
        with torch.no_grad():
            embs = get_retriever_embeddings(forward_fn, device, batch["retriever_passage_input_ids"],
                                            batch["retriever_passage_attention_mask"])
        start = step * batch_size
        out[start:start + len(embs)] = embs
    return unique_passage_dataset, out


def evaluate_retriever_on_batch(batch, passage_column_name: str, forward_fn, search_index: ExactIndex, torch_dtype: torch.dtype,
                                device: str, top_k: int, id_to_passage: Dict[int, str]):
    """reference :223-271 -> (list[precision], list[recall], total_hit, list[top passage per query]); every query has exactly
    one correct passage: its own row's"""
    with torch.no_grad():
        query_embeddings = get_retriever_embeddings(forward_fn, device, batch["retriever_query_input_ids"],
                                                    batch["retriever_query_attention_mask"])
    neighbours = get_nearest_neighbours(top_k, search_index, query_embeddings, id_to_passage, threshold=0.0)
    precisions, recalls, top_passages, hits = [], [], [], 0
    for gold, found in zip(batch[passage_column_name], neighbours):
        passages = [passage for passage, _similarity in found]
        top_passages.append(passages[0])                        # closest match; an empty result raises IndexError as in the reference
        p, r = calculate_precision_recall(passages, [gold])
        precisions.append(p)
        recalls.append(r)
        hits += gold in passages
    return precisions, recalls, hits, top_passages


def calc_eval_results(total_examples: int, precisions: List[float], recalls: List[float], total_hit: int) -> EvalResults:
    """reference :274-285: means over ALL examples"""
    n = float(total_examples)
    return EvalResults(total_examples=total_examples, recall=sum(recalls) / n, precision=sum(precisions) / n, hit_rate=total_hit / n)


def print_eval_results(eval_results: EvalResults) -> None:
    """reference :288-295 (same log lines)"""
    for line in eval_results.log_lines():
        logger.info(line)
