"""`dalm` command line — the hot-path commands of the reference's typer app (dalm/cli.py:17,35-38,41-167,170-277):
`version`, `train-rag-e2e`, `train-retriever-only`, `eval-retriever`, `eval-rag` (:313-412), same argument order / option
names / defaults. `qa-gen` belongs to a subsystem outside this build's scope and says so."""
from __future__ import annotations

from enum import Enum
from typing import Optional

import typer
from typing_extensions import Annotated

from . import __version__

cli = typer.Typer(add_completion=False, help="H100-native DALM training step")


class DALMSchedulerType(str, Enum):
    LINEAR = "linear"
    COSINE = "cosine"
    COSINE_WITH_RESTARTS = "cosine_with_restarts"
    POLYNOMIAL = "polynomial"
    CONSTANT = "constant"
    CONSTANT_WITH_WARMUP = "constant_with_warmup"


class PeftMode(str, Enum):
    generator = "generator"
    retriever = "retriever"
    both = "both"


Arg, Opt = typer.Argument, typer.Option


@cli.command()
def version() -> None:
    """Print the current version of DALM"""
    print(f"🐾You are running DALM version: {__version__}")


@cli.command()
def train_rag_e2e(
    dataset_path: Annotated[str, Arg(help="hf dataset dir or csv file", show_default=False)],
    retriever_name_or_path: Annotated[str, Arg(help="retriever model directory / id", show_default=False)],
    generator_name_or_path: Annotated[str, Arg(help="(causal) generator model directory / id", show_default=False)],
    passage_column_name: Annotated[str, Opt(help="column holding the passage")] = "Abstract",
    query_column_name: Annotated[str, Opt(help="column holding the query")] = "Question",
    answer_column_name: Annotated[str, Opt(help="column holding the answer")] = "Answer",
    query_max_len: Annotated[int, Opt(help="max query tokens (truncation)")] = 50,
    passage_max_len: Annotated[int, Opt(help="max passage tokens (truncation)")] = 128,
    generator_max_len: Annotated[int, Opt(help="max generator-input tokens (truncation)")] = 256,
    per_device_train_batch_size: Annotated[int, Opt(help="batch size per GPU")] = 32,
    learning_rate: Annotated[float, Opt(help="initial learning rate after warmup")] = 1e-4,
    logit_scale: Annotated[int, Opt(help="similarity logit scale")] = 100,
    weight_decay: Annotated[float, Opt(help="accepted for compatibility (unused by the reference too)")] = 0.0,
    num_train_epochs: Annotated[int, Opt(help="epochs")] = 1,
    max_train_steps: Annotated[Optional[int], Opt(help="overrides num_train_epochs")] = None,
    gradient_accumulation_steps: Annotated[int, Opt(help="micro-steps per optimizer step")] = 1,
    lr_scheduler_type: Annotated[DALMSchedulerType, Opt(help="scheduler")] = DALMSchedulerType.LINEAR,
    num_warmup_steps: Annotated[int, Opt(help="warmup steps")] = 100,
    output_dir: Annotated[Optional[str], Opt(help="where to store the final adapters")] = None,
    seed: Annotated[int, Opt(help="seed")] = 42,
    hub_model_id: Annotated[Optional[str], Opt(help="accepted, unused")] = None,
    hub_token: Annotated[Optional[str], Opt(help="accepted, unused")] = None,
    checkpointing_steps: Annotated[Optional[str], Opt(help="save state every N steps or 'epoch'")] = None,
    resume_from_checkpoint: Annotated[Optional[str], Opt(help="checkpoint folder to resume from")] = None,
    with_tracking: Annotated[bool, Opt(help="enable experiment tracking")] = True,
    report_to: Annotated[str, Opt(help="tracker selection")] = "all",
    sanity_test: Annotated[bool, Opt(help="accepted, unused")] = True,
    use_peft: Annotated[Optional[PeftMode], Opt(help="which sub-models get LoRA adapters")] = None,
    use_bnb: Annotated[Optional[PeftMode], Opt(help="NF4 values for the named sub-models' Linear weights (bitsandbytes nf4 round trip at load; needs the same sub-model in --use-peft)")] = None,
    retriever_is_autoregressive: Annotated[bool, Opt(help="the retriever is a causal LM (Llama family): last hidden state, eos pooling, q_proj/v_proj adapters")] = False,
) -> None:
    """End-to-end train an in-domain model, including the retriever and generator"""
    from transformers import SchedulerType

    from .models.rag_e2e_base_model import Mode
    from .training.rag_e2e.train_rage2e import train_e2e

    kw = dict(locals())
    for k in ("SchedulerType", "Mode", "train_e2e"):
        kw.pop(k, None)
    kw["dataset_or_path"] = kw.pop("dataset_path")
    kw["lr_scheduler_type"] = SchedulerType(lr_scheduler_type.value)
    kw["use_peft"] = Mode(use_peft.value) if use_peft is not None else None
    kw["use_bnb"] = Mode(use_bnb.value) if use_bnb is not None else None
    train_e2e(**kw)


@cli.command()
def train_retriever_only(
    retriever_name_or_path: Annotated[str, Arg(help="retriever model directory / id", show_default=False)],
    dataset_path: Annotated[str, Arg(help="hf dataset dir or csv file", show_default=False)],
    passage_column_name: Annotated[str, Opt(help="column holding the passage")] = "Abstract",
    query_column_name: Annotated[str, Opt(help="column holding the query")] = "Question",
    query_max_len: Annotated[int, Opt(help="max query tokens (truncation)")] = 50,
    passage_max_len: Annotated[int, Opt(help="max passage tokens (truncation)")] = 128,
    per_device_train_batch_size: Annotated[int, Opt(help="batch size per GPU")] = 32,
    learning_rate: Annotated[float, Opt(help="initial learning rate after warmup")] = 1e-4,
    logit_scale: Annotated[int, Opt(help="similarity logit scale")] = 100,
    weight_decay: Annotated[float, Opt(help="accepted, unused")] = 0.0,
    num_train_epochs: Annotated[int, Opt(help="epochs")] = 3,
    max_train_steps: Annotated[Optional[int], Opt(help="overrides num_train_epochs")] = None,
    gradient_accumulation_steps: Annotated[int, Opt(help="micro-steps per optimizer step")] = 1,
    lr_scheduler_type: Annotated[DALMSchedulerType, Opt(help="scheduler")] = DALMSchedulerType.LINEAR,
    num_warmup_steps: Annotated[int, Opt(help="warmup steps")] = 0,
    output_dir: Annotated[Optional[str], Opt(help="where to store the final adapter")] = None,
    seed: Annotated[int, Opt(help="seed")] = 42,
    hub_model_id: Annotated[Optional[str], Opt(help="accepted, unused")] = None,
    hub_token: Annotated[Optional[str], Opt(help="accepted, unused")] = None,
    checkpointing_steps: Annotated[Optional[str], Opt(help="save state every N steps or 'epoch'")] = None,
    resume_from_checkpoint: Annotated[Optional[str], Opt(help="checkpoint folder to resume from")] = None,
    with_tracking: Annotated[bool, Opt(help="enable experiment tracking")] = True,
    report_to: Annotated[str, Opt(help="tracker selection")] = "all",
    sanity_test: Annotated[bool, Opt(help="accepted, unused")] = True,
    use_peft: Annotated[bool, Opt(help="train LoRA adapters")] = True,
    use_bnb: Annotated[bool, Opt(help="NF4 values for the Linear weights (bitsandbytes nf4 round trip at load, bf16 storage; applies with --use-peft)")] = True,
    is_autoregressive: Annotated[bool, Opt(help="the retriever is a causal LM (Llama family): last hidden state, eos pooling")] = False,
) -> None:
    """Train only the retriever using contrastive training"""
    from transformers import SchedulerType

    from .training.retriever_only.train_retriever_only import train_retriever

    kw = dict(locals())
    for k in ("SchedulerType", "train_retriever"):
        kw.pop(k, None)
    kw["dataset_or_path"] = kw.pop("dataset_path")
    kw["lr_scheduler_type"] = SchedulerType(lr_scheduler_type.value)
    train_retriever(**kw)


def _out_of_scope(name: str) -> None:
    print(f"`dalm {name}` belongs to a reference subsystem outside dalm_b200's scope (training / evaluation hot path only); "
          "see DESIGN.md.")
    raise typer.Exit(code=2)


class TorchDtype(str, Enum):                 # reference cli.py:24-27
    float16 = "float16"
    bfloat16 = "bfloat16"


@cli.command()
def eval_retriever(
    dataset_path: Annotated[str, typer.Argument(help="Path to the dataset to eval with. Can be an hf dataset dir, csv file, "
                                                     "or path to hub file.", show_default=False)],
    retriever_name_or_path: Annotated[str, typer.Option(help="Path to pretrained retriever or identifier from huggingface.co/models.")],
    retriever_peft_model_path: Annotated[Optional[str], typer.Option(help="Path to the fine-tuned retriever peft layers")] = None,
    passage_column_name: Annotated[str, typer.Option(help="Name of the column containing the passage")] = "Abstract",
    query_column_name: Annotated[str, typer.Option(help="Name of the column containing the query")] = "Question",
    embed_dim: Annotated[int, typer.Option(help="Dimension of the model embedding")] = 1024,
    max_length: Annotated[int, typer.Option(help="The max passage sequence length during tokenization. Longer sequences are truncated")] = 128,
    test_batch_size: Annotated[int, typer.Option(help="Batch size (per device) for the test dataloader.")] = 8,
    device: Annotated[str, typer.Option(help="Device. cpu or cuda.")] = "cuda",
    torch_dtype: Annotated[TorchDtype, typer.Option(help="torch.dtype to use for tensors. float16 or bfloat16.")] = TorchDtype.float16,
    top_k: Annotated[int, typer.Option(help="Top K retrieval")] = 10,
    is_autoregressive: Annotated[bool, typer.Option(help="Whether the model is autoregressive.")] = False,
) -> None:
    """Evaluate your retriever only"""
    from .eval.eval_retriever_only import evaluate_retriever

    evaluate_retriever(dataset_or_path=dataset_path, retriever_name_or_path=retriever_name_or_path,
                       retriever_peft_model_path=retriever_peft_model_path, passage_column_name=passage_column_name,
                       query_column_name=query_column_name, embed_dim=embed_dim, max_length=max_length,
                       test_batch_size=test_batch_size, device=device, torch_dtype=torch_dtype.value, top_k=top_k,
                       is_autoregressive=is_autoregressive)


@cli.command()
def eval_rag(
    dataset_path: Annotated[str, typer.Argument(help="Path to the dataset to eval with. Can be an hf dataset dir, csv file, "
                                                     "or path to hub file.", show_default=False)],
    retriever_name_or_path: Annotated[str, typer.Option(help="Path to pretrained retriever or identifier from huggingface.co/models.")],
    generator_name_or_path: Annotated[str, typer.Option(help="Path to pretrained (causal) generator or identifier from huggingface.co/models.")],
    retriever_peft_model_path: Annotated[Optional[str], typer.Option(help="Path to the fine-tuned retriever peft layers")] = None,
    generator_peft_model_path: Annotated[Optional[str], typer.Option(help="Path to the fine-tuned generator peft layers")] = None,
    passage_column_name: Annotated[str, typer.Option(help="Name of the column containing the passage")] = "Abstract",
    query_column_name: Annotated[str, typer.Option(help="Name of the column containing the query")] = "Question",
    answer_column_name: Annotated[str, typer.Option(help="Name of the column containing the Answer")] = "Answer",
    embed_dim: Annotated[int, typer.Option(help="Dimension of the model embedding")] = 1024,
    max_length: Annotated[int, typer.Option(help="The max passage sequence length during tokenization. Longer sequences are truncated")] = 128,
    test_batch_size: Annotated[int, typer.Option(help="Batch size (per device) for the test dataloader.")] = 8,
    query_batch_size: Annotated[int, typer.Option(help="Batch size (per device) for generator input")] = 16,
    device: Annotated[str, typer.Option(help="Device. cpu or cuda.")] = "cuda",
    torch_dtype: Annotated[TorchDtype, typer.Option(help="torch.dtype to use for tensors. float16 or bfloat16.")] = TorchDtype.float16,
    top_k: Annotated[int, typer.Option(help="Top K retrieval")] = 10,
    evaluate_generator: Annotated[bool, typer.Option(help="Enable generator evaluation. If false, equivalent to eval-retriever")] = True,
    retriever_is_autoregressive: Annotated[bool, typer.Option(help="Whether the retriever is autoregressive.")] = False,
) -> None:
    """Evaluate your end-to-end rag generator and retriever"""
    from .eval.eval_rag import evaluate_rag

    evaluate_rag(dataset_or_path=dataset_path, retriever_name_or_path=retriever_name_or_path,
                 generator_name_or_path=generator_name_or_path, retriever_peft_model_path=retriever_peft_model_path,
                 generator_peft_model_path=generator_peft_model_path, passage_column_name=passage_column_name,
                 query_column_name=query_column_name, answer_column_name=answer_column_name, embed_dim=embed_dim,
                 max_length=max_length, test_batch_size=test_batch_size, query_batch_size=query_batch_size, device=device,
                 torch_dtype=torch_dtype.value, top_k=top_k, evaluate_generator=evaluate_generator,
                 retriever_is_autoregressive=retriever_is_autoregressive)


@cli.command()
def qa_gen(                                   # reference cli.py:280-309: same arguments, so an existing command line parses
    dataset_path: Annotated[str, typer.Argument(help="Path to the input dataset.", show_default=False)],
    output_dir: Annotated[str, typer.Option(help="Output directory to store the resulting files")] = ".",
    passage_column_name: Annotated[str, typer.Option(help="Column name for the passage/text")] = "Abstract",
    title_column_name: Annotated[str, typer.Option(help="Column name for the title of the full document")] = "Title",
    batch_size: Annotated[int, typer.Option(help="Batch size (per device) for generating question answer pairs.")] = 100,
    sample_size: Annotated[int, typer.Option(help="Number of examples to process.")] = 1000,
    as_csv: Annotated[bool, typer.Option(help="Save the files as CSV.")] = True,
) -> None:
    """(reference command — QA-pair data generation — not part of the H100 hot-path build; exits with status 2)"""
    _out_of_scope("qa-gen")


if __name__ == "__main__":
    cli()
