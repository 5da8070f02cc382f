"""`train_retriever` — drop-in for the reference's dalm/training/retriever_only/train_retriever_only.py (signature
:175-203, script flags :54-172, loop :357-406): contrastive (in-batch negatives) LoRA training of the encoder."""
from __future__ import annotations

from argparse import Namespace
from typing import Any, Optional, Union

from transformers import SchedulerType

from ...models.retriever_only_base_model import AutoModelForSentenceEmbedding
from ..utils.loop import Recipe, build_parser, run_training
from ..utils.retriever_only_dataloader_utils import preprocess_dataset
from ..utils.train_utils import fused_retriever_step, save_adapter_dir

_FLAGS = [
    ("dataset_path", dict(type=str, default=None)),
    ("query_column_name", dict(type=str, default="Question")),
    ("passage_column_name", dict(type=str, default="Abstract")),
    ("query_max_len", dict(type=int, default=50)),
    ("passage_max_len", dict(type=int, default=160)),
    ("model_name_or_path", dict(type=str, required=True)),
    ("per_device_train_batch_size", dict(type=int, default=8)),      # script default 8; function / CLI default 32
    ("learning_rate", dict(type=float, default=1e-4)),
    ("logit_scale", dict(type=int, default=100)),
    ("weight_decay", dict(type=float, default=0.0)),
    ("num_train_epochs", dict(type=int, default=3)),
    ("max_train_steps", dict(type=int, default=None)),
    ("gradient_accumulation_steps", dict(type=int, default=1)),
    ("lr_scheduler_type", dict(type=SchedulerType, default=SchedulerType.LINEAR, choices=[s for s in SchedulerType])),
    ("num_warmup_steps", dict(type=int, default=0)),
    ("output_dir", dict(type=str, default=None)),
    ("seed", dict(type=int, default=None)),
    ("hub_model_id", dict(type=str, default=None)),
    ("hub_token", dict(type=str, default=None)),
    ("checkpointing_steps", dict(type=str, default=None)),
    ("resume_from_checkpoint", dict(type=str, default=None)),
    ("with_tracking", dict(action="store_true")),
    ("report_to", dict(type=str, default="all")),
    ("sanity_test", dict(action="store_true")),
    ("use_peft", dict(action="store_true")),
    ("use_bnb", dict(action="store_true")),
    ("is_autoregressive", dict(action="store_true")),
]


def parse_args() -> Namespace:
    return build_parser("contrastive retriever training (H100-native)", _FLAGS).parse_args()


def train_retriever(
    retriever_name_or_path: str,
    dataset_or_path: Any,
    passage_column_name: str = "Abstract",
    query_column_name: str = "Question",
    query_max_len: int = 50,
    passage_max_len: int = 128,
    per_device_train_batch_size: int = 32,
    learning_rate: float = 1e-4,
    logit_scale: int = 100,
    weight_decay: float = 0.0,
    num_train_epochs: int = 1,
    max_train_steps: Optional[int] = None,
    gradient_accumulation_steps: int = 1,
    lr_scheduler_type: SchedulerType = SchedulerType.LINEAR,
    num_warmup_steps: int = 0,
    output_dir: Optional[str] = None,
    seed: int = 42,
    hub_model_id: Optional[str] = None,
    hub_token: Optional[str] = None,
    checkpointing_steps: Optional[Union[int, str]] = None,
    resume_from_checkpoint: Optional[str] = None,
    with_tracking: bool = True,
    report_to: str = "all",
    sanity_test: bool = True,
    use_peft: bool = True,
    use_bnb: bool = True,
    is_autoregressive: bool = False,
) -> None:
    args = dict(locals())

    def build() -> AutoModelForSentenceEmbedding:
        m = AutoModelForSentenceEmbedding(retriever_name_or_path, use_bnb=use_bnb, get_peft=use_peft,
                                          is_autoregressive=is_autoregressive)
        if use_peft:
            m.print_trainable_parameters()                   # reference :259-260
        return m

    def tokenize(model: AutoModelForSentenceEmbedding, dataset):
        tok = model.tokenizer

        def build(ex):                                        # closes over the tokenizer only (never the CUDA model)
            return preprocess_dataset(ex, tok, query_column_name=query_column_name, passage_column_name=passage_column_name,
                                      query_max_len=query_max_len, passage_max_len=passage_max_len)

        return dataset.map(build, batched=True, remove_columns=dataset.column_names, desc="Running tokenizer on dataset")

    def save_final(model: AutoModelForSentenceEmbedding, output_dir: str) -> None:
        import os
        d = os.path.join(output_dir, "retriever")
        save_adapter_dir(model.model, d, "FEATURE_EXTRACTION")
        if model.tokenizer is not None:
            model.tokenizer.save_pretrained(d)

    recipe = Recipe(
        title="Running training", tracker_project="peft_contrastive_learning", build_model=build, tokenize=tokenize,
        step=lambda m, b, s, gs: fused_retriever_step(m, b, s, backward=True, grad_scale=gs), step_fn=fused_retriever_step,
        banks=lambda m: m.model.banks(), repack=lambda m: m.model.repack_lora(),
        save_final=save_final)
    run_training(recipe, dataset_or_path=dataset_or_path, per_device_train_batch_size=per_device_train_batch_size,
                 learning_rate=learning_rate, logit_scale=logit_scale, num_train_epochs=num_train_epochs,
                 max_train_steps=max_train_steps, gradient_accumulation_steps=gradient_accumulation_steps,
                 lr_scheduler_type=lr_scheduler_type, num_warmup_steps=num_warmup_steps, output_dir=output_dir, seed=seed,
                 checkpointing_steps=checkpointing_steps, resume_from_checkpoint=resume_from_checkpoint,
                 with_tracking=with_tracking, report_to=report_to, config_for_tracker=args)


def main() -> None:
    a = vars(parse_args())
    a["retriever_name_or_path"] = a.pop("model_name_or_path")
    a["dataset_or_path"] = a.pop("dataset_path")
    train_retriever(**a)


if __name__ == "__main__":
    main()
