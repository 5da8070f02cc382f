"""`train_e2e` — drop-in for the reference's dalm/training/rag_e2e/train_rage2e.py (signature :229-260, script flags
:54-226, loop :420-500), running the loop body as dalm_b200's fused CUDA launch sequence.

    python -m dalm_b200.training.rag_e2e.train_rage2e --dataset_path data.csv \
        --retriever_name_or_path <dir> --generator_name_or_path <dir> --use_peft both
"""
from __future__ import annotations

import os
from argparse import Namespace
from typing import Any, Optional, Union

from transformers import SchedulerType

from ...models.rag_e2e_base_model import AutoModelForRagE2E, Mode
from ..utils.loop import Recipe, build_parser, run_training
from ..utils.rag_e2e_dataloader_utils import preprocess_dataset
from ..utils.train_utils import fused_rag_step, save_adapter_dir

_FLAGS = [
    ("dataset_path", dict(type=str, default=None, help="csv file or datasets directory")),
    ("passage_column_name", dict(type=str, default="Abstract")),
    ("query_column_name", dict(type=str, default="Question")),
    ("answer_column_name", dict(type=str, default="Answer")),
    ("query_max_len", dict(type=int, default=50)),
    ("passage_max_len", dict(type=int, default=160)),            # argparse default differs from the function's 128
    ("generator_max_len", dict(type=int, default=256)),
    ("retriever_name_or_path", dict(type=str, required=True)),
    ("generator_name_or_path", dict(type=str, required=True)),
    ("per_device_train_batch_size", dict(type=int, default=32)),
    ("learning_rate", dict(type=float, default=1e-4)),
    ("logit_scale", dict(type=int, default=100)),
    ("weight_decay", dict(type=float, default=0.0)),
    ("num_train_epochs", dict(type=int, default=1)),
    ("max_train_steps", dict(type=int, default=None)),
    ("gradient_accumulation_steps", dict(type=int, default=1)),
    ("lr_scheduler_type", dict(type=SchedulerType, default=SchedulerType.LINEAR,
                               choices=[s for s in SchedulerType])),
    ("num_warmup_steps", dict(type=int, default=100)),
    ("output_dir", dict(type=str, default=None)),
    ("seed", dict(type=int, default=None)),
    ("hub_model_id", dict(type=str, default=None)),
    ("hub_token", dict(type=str, default=None)),
    ("checkpointing_steps", dict(type=str, default=None)),
    ("resume_from_checkpoint", dict(type=str, default=None)),
    ("with_tracking", dict(action="store_true")),
    ("report_to", dict(type=str, default="all")),
    ("sanity_test", dict(action="store_true")),
    ("use_peft", dict(type=Mode, default=None, choices=[m for m in Mode])),
    ("use_bnb", dict(type=Mode, default=None, choices=[m for m in Mode])),
    ("retriever_is_autoregressive", dict(action="store_true")),
]


def parse_args() -> Namespace:
    return build_parser("RAG end-to-end training (H100-native)", _FLAGS).parse_args()


def _save_final(tokenizers):
    def save(model: AutoModelForRagE2E, output_dir: str) -> None:
        r_dir, g_dir = os.path.join(output_dir, "retriever"), os.path.join(output_dir, "generator")
        save_adapter_dir(model.retriever_model, r_dir, "FEATURE_EXTRACTION")
        save_adapter_dir(model.generator_model, g_dir, "CAUSAL_LM")
        if model.retriever_tokenizer is not None:
            model.retriever_tokenizer.save_pretrained(r_dir)
        if model.generator_tokenizer is not None:
            model.generator_tokenizer.save_pretrained(g_dir)
    return save


def train_e2e(
    dataset_or_path: Any,
    retriever_name_or_path: str,
    generator_name_or_path: str,
    passage_column_name: str = "Abstract",
    query_column_name: str = "Question",
    answer_column_name: str = "Answer",
    query_max_len: int = 50,
    passage_max_len: int = 128,
    generator_max_len: int = 256,
    per_device_train_batch_size: int = 32,
    learning_rate: float = 1e-4,
    logit_scale: int = 100,
    weight_decay: float = 0.0,
    num_train_epochs: int = 1,
    max_train_steps: Optional[int] = None,
    gradient_accumulation_steps: int = 1,
    lr_scheduler_type: SchedulerType = SchedulerType.LINEAR,
    num_warmup_steps: int = 100,
    output_dir: Optional[str] = None,
    seed: int = 42,
    hub_model_id: Optional[str] = None,
    hub_token: Optional[str] = None,
    checkpointing_steps: Optional[Union[int, str]] = None,
    resume_from_checkpoint: Optional[str] = None,
    with_tracking: bool = True,
    report_to: str = "all",
    sanity_test: bool = True,
    use_peft: Optional[Mode] = None,
    use_bnb: Optional[Mode] = None,
    retriever_is_autoregressive: bool = False,
) -> None:
    # weight_decay, hub_model_id, hub_token, sanity_test are accepted and ignored, exactly like the reference (SURVEY §8a-6)
    args = dict(locals())

    def build() -> AutoModelForRagE2E:
        return AutoModelForRagE2E(retriever_name_or_path, generator_name_or_path, get_peft=use_peft, use_bnb=use_bnb,
                                  retriever_is_autoregressive=retriever_is_autoregressive)

    def tokenize(model: AutoModelForRagE2E, dataset):
        rtok, gtok = model.retriever_tokenizer, model.generator_tokenizer
        gtok.pad_token = gtok.eos_token                       # reference :301
        gtok.add_eos_token = True                             # reference :304

        def build(ex):                                        # closes over the tokenizers only (never the CUDA model)
            return preprocess_dataset(ex, retriever_tokenizer=rtok, generator_tokenizer=gtok,
                                      query_column_name=query_column_name, passage_column_name=passage_column_name,
                                      answer_column_name=answer_column_name, query_max_len=query_max_len,
                                      passage_max_len=passage_max_len, generator_max_len=generator_max_len)

        # single process like the reference (num_proc=1 there); in-process so no CUDA context is forked
        return dataset.map(build, batched=True, remove_columns=dataset.column_names, desc="Running tokenizer on dataset")

    recipe = Recipe(
        title="Running E2E training", tracker_project="peft_rag_e2e_learning", build_model=build, tokenize=tokenize,
        step=lambda m, b, s, gs: fused_rag_step(m, b, s, backward=True, grad_scale=gs), step_fn=fused_rag_step,
        banks=lambda m: m.trainable_banks(), repack=lambda m: m.repack(), save_final=_save_final(None))
    run_training(recipe, dataset_or_path=dataset_or_path, per_device_train_batch_size=per_device_train_batch_size,
                 learning_rate=learning_rate, logit_scale=logit_scale, num_train_epochs=num_train_epochs,
                 max_train_steps=max_train_steps, gradient_accumulation_steps=gradient_accumulation_steps,
                 lr_scheduler_type=lr_scheduler_type, num_warmup_steps=num_warmup_steps, output_dir=output_dir, seed=seed,
                 checkpointing_steps=checkpointing_steps, resume_from_checkpoint=resume_from_checkpoint,
                 with_tracking=with_tracking, report_to=report_to, config_for_tracker=args)


def main() -> None:
    a = vars(parse_args())
    a["dataset_or_path"] = a.pop("dataset_path")
    train_e2e(**a)


if __name__ == "__main__":
    main()
