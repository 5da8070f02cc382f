"""`dalm eval-retriever` — reference dalm/eval/eval_retriever_only.py:33-200 with the encoder forward on dalm_b200's kernels
and the hnswlib index replaced by the exact HBM-resident top-k (eval/utils.py)."""
from __future__ import annotations

import logging
from argparse import Namespace
from typing import Any, Final, Literal, Optional

import torch
from torch.utils.data import DataLoader

from ..models.rag_e2e_base_model import inference_only
from ..models.retriever_only_base_model import AutoModelForSentenceEmbedding
from ..utils import load_dataset
from .eval_results import EvalResults
from .utils import (calc_eval_results, construct_search_index, evaluate_retriever_on_batch, get_passage_embeddings,
                    mixed_collate_fn, preprocess_dataset, print_eval_results)

logger = logging.getLogger(__name__)


# script flags of the reference (:33-102): same names and defaults, one table
_FLAGS = [
    ("dataset_path", dict(type=str, default=None, required=True, help="csv file or datasets directory")),
    ("query_column_name", dict(type=str, default="query")),
    ("passage_column_name", dict(type=str, default="passage")),
    ("embed_dim", dict(type=int, default=1024, help="width of the retriever's embeddings")),
    ("max_length", dict(type=int, default=128, help="tokens per query / passage (truncated, padded)")),
    ("retriever_name_or_path", dict(type=str, required=True)),
    ("retriever_peft_model_path", dict(type=str, required=False, help="directory with trained retriever adapters")),
    ("test_batch_size", dict(type=int, default=8)),
    ("device", dict(type=str, default="cuda", help="must be a CUDA device: there is no CPU path")),
    ("torch_dtype", dict(type=str, default="float16", help="float16 | bfloat16 (signature parity; the forward is bf16 + fp32 pooling)")),
    ("top_k", dict(type=int, default=10)),
    ("is_autoregressive", dict(action="store_true", help="the retriever is a causal LM")),
]


def parse_args() -> Namespace:
    from ..training.utils.loop import build_parser
    return build_parser("Retriever evaluation: exact top-k search over the passage embeddings (H100-native)", _FLAGS).parse_args()


def evaluate_retriever(
    dataset_or_path: Any,
    retriever_name_or_path: str,
    retriever_peft_model_path: Optional[str],
    passage_column_name: str,
    query_column_name: str,
    embed_dim: int,
    max_length: int,
    test_batch_size: int = 8,
    device: str = "cuda",
    torch_dtype: Literal["float16", "bfloat16"] = "float16",
    top_k: int = 10,
    is_autoregressive: bool = False,
) -> EvalResults:
    """reference :105-178. `device` must be a CUDA device (no CPU path); `torch_dtype` is accepted for signature parity —
    the forward always runs bf16 GEMMs with fp32 pooling."""
    if not str(device).startswith("cuda"):
        raise RuntimeError("dalm_b200 evaluates on a CUDA (sm_90a) device only: there is no CPU path")
    test_dataset = load_dataset(dataset_or_path)
    selected_torch_dtype: Final[torch.dtype] = torch.float16 if torch_dtype == "float16" else torch.bfloat16
    with inference_only():
        retriever_model = AutoModelForSentenceEmbedding(retriever_name_or_path, get_peft=False, use_bnb=False,
                                                        is_autoregressive=is_autoregressive)
    retriever_model.eval()
    processed = preprocess_dataset(test_dataset, retriever_model.tokenizer, query_column_name, passage_column_name, max_length)
    if retriever_peft_model_path is not None:
        retriever_model.attach_pre_trained_peft_layers(retriever_peft_model_path, device)
    dev = str(retriever_model.model.dev)
    unique_passage_dataset, passage_embeddings = get_passage_embeddings(processed, passage_column_name, retriever_model.forward,
                                                                       dev, embed_dim, selected_torch_dtype, test_batch_size)
    id_to_passage = {i: p[passage_column_name] for i, p in enumerate(unique_passage_dataset)}
    logger.info("Construct passage index")
    index = construct_search_index(embed_dim, len(passage_embeddings), passage_embeddings)
    batch_precision, batch_recall, total_hit = [], [], 0
    logger.info("Evaluation start")
    loader = DataLoader(processed, batch_size=test_batch_size, shuffle=True, collate_fn=mixed_collate_fn)
    for batch in loader:
        p_, r_, h_, _ = evaluate_retriever_on_batch(batch, passage_column_name, retriever_model.forward, index,
                                                    selected_torch_dtype, dev, top_k, id_to_passage)
        batch_precision.extend(p_)
        batch_recall.extend(r_)
        total_hit += h_
    results = calc_eval_results(len(processed), batch_precision, batch_recall, total_hit)
    print_eval_results(results)
    return results


def main() -> None:
    a = parse_args()
    evaluate_retriever(dataset_or_path=a.dataset_path, retriever_name_or_path=a.retriever_name_or_path,
                       retriever_peft_model_path=a.retriever_peft_model_path, passage_column_name=a.passage_column_name,
                       query_column_name=a.query_column_name, embed_dim=a.embed_dim, max_length=a.max_length,
                       test_batch_size=a.test_batch_size, device=a.device, torch_dtype=a.torch_dtype, top_k=a.top_k,
                       is_autoregressive=a.is_autoregressive)


if __name__ == "__main__":
    main()
