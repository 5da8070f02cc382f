"""`dalm eval-rag` — reference dalm/eval/eval_rag.py:167-290. Retriever half: passage sweep, exact top-k, recall / precision /
hit-rate through `rag_model.retrieval_forward`. Generator half (`run_generator_on_prompts` :126-140, `eval_generator_on_batch`
:143-164, exact match :268-283): prompts `#query# q #passage# p #answer# ` are tokenised exactly as the reference does and
decoded by `generator_model.generate` with a KV cache over the C-ABI kernels (engine/decoding.py), HF `generate` semantics
for the reference's call: greedy search, or sampling (temperature -> top-k -> top-p) when the checkpoint's generation_config
asks for it, as Llama-2's does. The log line states which one runs."""
from __future__ import annotations

import logging
from argparse import Namespace
from typing import Any, Final, List, Literal, Optional

import torch
from torch.utils.data import DataLoader

from ..models.rag_e2e_base_model import AutoModelForRagE2E, inference_only
from ..utils import load_dataset
from .eval_results import EvalResults
from .utils import (calc_eval_results, construct_search_index, evaluate_retriever_on_batch, get_passage_embeddings,
                    mixed_collate_fn, preprocess_dataset, print_eval_results)

logger = logging.getLogger(__name__)


def run_generator_on_prompts(model: Any, tokenizer: Any, prompts: List[str], max_length: int = 256) -> List[str]:
    """Runs the generator model over the prompts (query + passage) — reference eval_rag.py:126-140. `model` is the
    wrapper's `generator_model` (LlamaDecoder / FalconDecoder); its `generate` takes the tokenizer's tensors as they are
    (host int64) and returns the padded prompt + continuation like HF does."""
    inputs = tokenizer(prompts, return_tensors="pt", padding=True, truncation=True, max_length=max_length)
    outputs = model.generate(**inputs, max_length=max_length, early_stopping=True)
    return tokenizer.batch_decode(outputs.cpu(), skip_special_tokens=True)


def eval_generator_on_batch(model: Any, tokenizer: Any, queries: List[str], passages: List[str], query_batch_size: int,
                            queries_for_gen_eval: List[str], max_length: int) -> tuple:
    """reference eval_rag.py:143-164: accumulate prompts, flush every `query_batch_size`"""
    generated_answers_for_eval: List[str] = []
    for _query, search_result_passage in zip(queries, passages, strict=True):
        queries_for_gen_eval.append(f"#query# {_query} #passage# {search_result_passage} #answer# ")     # no answer in the prompt
        if len(queries_for_gen_eval) >= query_batch_size:
            generated_answers_for_eval.extend(run_generator_on_prompts(model, tokenizer, queries_for_gen_eval, max_length=max_length))
            queries_for_gen_eval.clear()
    return queries_for_gen_eval, generated_answers_for_eval


def exact_match_hits(generated_answers: List[str], answers: List[str]) -> int:
    """reference eval_rag.py:268-277: the text after the first `#answer#`, stripped, must equal the gold answer"""
    hits = 0
    for generated_answer, answer in zip(generated_answers, answers, strict=True):
        parts = generated_answer.split("#answer#")
        if len(parts) < 2:
            continue
        if parts[1].strip() == answer:
            hits += 1
    return hits


def evaluate_rag(
    dataset_or_path: Any,
    retriever_name_or_path: str,
    generator_name_or_path: str,
    retriever_peft_model_path: Optional[str],
    generator_peft_model_path: Optional[str],
    passage_column_name: str,
    query_column_name: str,
    answer_column_name: str,
    embed_dim: int,
    max_length: int,
    test_batch_size: int = 8,
    query_batch_size: int = 16,
    device: str = "cuda",
    torch_dtype: Literal["float16", "bfloat16"] = "float16",
    top_k: int = 10,
    evaluate_generator: bool = True,
    retriever_is_autoregressive: bool = False,
) -> EvalResults:
    if not str(device).startswith("cuda"):
        raise RuntimeError("dalm_b200 evaluates on a CUDA (sm_90a) device only: there is no CPU path")
    test_dataset = load_dataset(dataset_or_path)
    selected_torch_dtype: Final[torch.dtype] = torch.float16 if torch_dtype == "float16" else torch.bfloat16
    with inference_only():
        rag_model = AutoModelForRagE2E(retriever_name_or_path, generator_name_or_path,
                                       retriever_is_autoregressive=retriever_is_autoregressive)
    rag_model.eval()
    processed = preprocess_dataset(test_dataset, rag_model.retriever_tokenizer, query_column_name, passage_column_name, max_length)
    rag_model.attach_pre_trained_peft_layers(retriever_peft_model_path, generator_peft_model_path, device)
    dev = str(rag_model.retriever_model.dev)
    unique_passage_dataset, passage_embeddings = get_passage_embeddings(processed, passage_column_name, rag_model.retrieval_forward,
                                                                       dev, embed_dim, selected_torch_dtype, test_batch_size)
    id_to_passage = {i: p[passage_column_name] for i, p in enumerate(unique_passage_dataset)}
    index = construct_search_index(embed_dim, len(passage_embeddings), passage_embeddings)
    batch_precision, batch_recall, total_hit = [], [], 0
    queries_for_gen_eval: List[str] = []
    generated_answers_for_eval: List[str] = []
    model, tokenizer = rag_model.generator_model, rag_model.generator_tokenizer
    if evaluate_generator:
        tokenizer.pad_token = tokenizer.eos_token                                 # reference :240
        from ..engine.decoding import decoding_mode
        logger.info(f"generator evaluation decodes by {decoding_mode(model, max_length=max_length, early_stopping=True)}")
    loader = DataLoader(processed, batch_size=test_batch_size, shuffle=True, collate_fn=mixed_collate_fn)
    for batch in loader:
        p_, r_, h_, top_passages = evaluate_retriever_on_batch(batch, passage_column_name, rag_model.retrieval_forward, index,
                                                               selected_torch_dtype, dev, top_k, id_to_passage)
        batch_precision.extend(p_)
        batch_recall.extend(r_)
        total_hit += h_
        if not evaluate_generator:
            continue
        queries_for_gen_eval, batch_answers = eval_generator_on_batch(model, tokenizer, batch[query_column_name], top_passages,
                                                                      query_batch_size, queries_for_gen_eval, max_length)
        generated_answers_for_eval.extend(batch_answers)
    results = calc_eval_results(len(processed), batch_precision, batch_recall, total_hit)
    if not evaluate_generator:
        print_eval_results(results)
        return results
    if len(queries_for_gen_eval) > 0:                                             # leftover prompts (reference :258-261)
        generated_answers_for_eval.extend(run_generator_on_prompts(model, tokenizer, queries_for_gen_eval, max_length=max_length))
        queries_for_gen_eval.clear()
    # like the reference (:263-266) the gold answers are read in DATASET order while the generated ones come in the shuffled
    # loader's order; kept as is — it is the number the reference prints
    total_em_hit = exact_match_hits(generated_answers_for_eval, list(processed[answer_column_name]))
    print_eval_results(results)
    print("Generator evaluation:")
    print("Exact match:", total_em_hit / len(processed))
    return results


# script entry point of the reference (:27-123, :293-313): same flags and defaults, one table
_FLAGS = [
    ("dataset_path", dict(type=str, default=None, required=True, help="csv file or datasets directory")),
    ("query_column_name", dict(type=str, default="query")),
    ("passage_column_name", dict(type=str, default="passage")),
    ("answer_column_name", dict(type=str, default="answer")),
    ("embed_dim", dict(type=int, default=1024, help="width of the retriever's embeddings")),
    ("max_length", dict(type=int, default=256, help="tokens per query / passage, and TOTAL tokens of a generated answer")),
    ("retriever_name_or_path", dict(type=str, required=True)),
    ("generator_name_or_path", dict(type=str, required=True)),
    ("retriever_peft_model_path", dict(type=str, required=False)),
    ("generator_peft_model_path", dict(type=str, required=False)),
    ("test_batch_size", dict(type=int, default=8)),
    ("query_batch_size", dict(type=int, default=16, help="prompts per generate() call")),
    ("device", dict(type=str, default="cuda", help="must be a CUDA device: there is no CPU path")),
    ("torch_dtype", dict(type=str, default="float16")),
    ("top_k", dict(type=int, default=10)),
    ("evaluate_generator", dict(action="store_true", help="also generate answers and score exact match")),
    ("is_retriever_autoregressive", dict(action="store_true")),
]


def parse_args() -> Namespace:
    from ..training.utils.loop import build_parser
    return build_parser("RAG evaluation: retrieval metrics + generation / exact match (H100-native)", _FLAGS).parse_args()


def main() -> None:
    a = parse_args()
    evaluate_rag(dataset_or_path=a.dataset_path, retriever_name_or_path=a.retriever_name_or_path,
                 generator_name_or_path=a.generator_name_or_path, retriever_peft_model_path=a.retriever_peft_model_path,
                 generator_peft_model_path=a.generator_peft_model_path, passage_column_name=a.passage_column_name,
                 query_column_name=a.query_column_name, answer_column_name=a.answer_column_name, embed_dim=a.embed_dim,
                 max_length=a.max_length, test_batch_size=a.test_batch_size, query_batch_size=a.query_batch_size, device=a.device,
                 torch_dtype=a.torch_dtype, top_k=a.top_k, evaluate_generator=a.evaluate_generator,
                 retriever_is_autoregressive=a.is_retriever_autoregressive)


if __name__ == "__main__":
    main()
