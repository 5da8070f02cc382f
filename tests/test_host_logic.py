"""CPU: host-side logic of the drop-in surface — CLI, argparse defaults, resume parsing, loader sharding, scheduler."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cli_version_string():
    """reference tests/test_cli.py:6-8"""
    import dalm_b200
    out = subprocess.run([sys.executable, "-m", "dalm_b200.cli", "version"], capture_output=True, text=True, cwd=ROOT,
                         env=dict(os.environ, PYTHONIOENCODING="utf-8")).stdout.strip()
    assert out == f"🐾You are running DALM version: {dalm_b200.__version__}"


def test_cli_surface():
    import typer
    from typer.testing import CliRunner
    from dalm_b200.cli import cli
    group = typer.main.get_command(cli)
    e2e = group.commands["train-rag-e2e"]
    opts = {o for p in e2e.params for o in p.opts}
    for opt in ("--passage-column-name", "--query-max-len", "--generator-max-len", "--per-device-train-batch-size",
                "--logit-scale", "--lr-scheduler-type", "--num-warmup-steps", "--checkpointing-steps", "--use-peft",
                "--retriever-is-autoregressive", "--with-tracking", "--use-bnb", "--resume-from-checkpoint"):
        assert opt in opts, opt
    # positional order differs between the two commands (reference cli.py:41-60 vs :170-185)
    assert [p.name for p in e2e.params[:3]] == ["dataset_path", "retriever_name_or_path", "generator_name_or_path"]
    ro = group.commands["train-retriever-only"]
    assert [p.name for p in ro.params[:2]] == ["retriever_name_or_path", "dataset_path"]
    d = {p.name: p.default for p in ro.params}
    assert d["num_train_epochs"] == 3 and d["num_warmup_steps"] == 0 and d["use_peft"] is True and d["passage_max_len"] == 128
    d = {p.name: p.default for p in e2e.params}
    assert d["num_warmup_steps"] == 100 and d["per_device_train_batch_size"] == 32 and d["seed"] == 42
    assert CliRunner().invoke(cli, ["eval-rag"]).exit_code == 2


def test_dalm_alias_package():
    import dalm
    from dalm.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm.training.utils.train_utils import get_cosine_sim, compute_marginalized_loss_from_logits  # noqa: F401
    from dalm.training.rag_e2e.train_rage2e import train_e2e  # noqa: F401
    import dalm_b200.models.rag_e2e_base_model as real
    assert AutoModelForRagE2E is real.AutoModelForRagE2E and Mode.BOTH.value == "both"
    assert dalm.__version__ == "0.0.5"


def test_script_defaults_differ_like_reference(monkeypatch):
    """SURVEY §5: argparse defaults != function defaults (passage_max_len 160 vs 128, retriever bs 8 vs 32, ...)"""
    import inspect
    from dalm_b200.training.rag_e2e import train_rage2e as e2e
    from dalm_b200.training.retriever_only import train_retriever_only as ro
    monkeypatch.setattr(sys, "argv", ["x", "--retriever_name_or_path", "r", "--generator_name_or_path", "g"])
    a = e2e.parse_args()
    assert a.passage_max_len == 160 and a.seed is None and a.with_tracking is False and a.num_warmup_steps == 100
    sig = inspect.signature(e2e.train_e2e).parameters
    assert sig["passage_max_len"].default == 128 and sig["seed"].default == 42 and sig["with_tracking"].default is True
    assert sig["per_device_train_batch_size"].default == 32 and sig["use_peft"].default is None
    monkeypatch.setattr(sys, "argv", ["x", "--model_name_or_path", "r"])
    b = ro.parse_args()
    assert b.per_device_train_batch_size == 8 and b.num_train_epochs == 3 and b.use_peft is False
    sig = inspect.signature(ro.train_retriever).parameters
    assert sig["per_device_train_batch_size"].default == 32 and sig["num_train_epochs"].default == 1
    assert sig["use_peft"].default is True and list(sig)[:2] == ["retriever_name_or_path", "dataset_or_path"]


def test_resume_parsing():
    from dalm_b200.training.utils.loop import parse_resume
    assert parse_resume("/x/out/epoch_2", steps_per_epoch=50, loader_len=100, gas=2) == (3, None, 150)
    # step_30 with gas=2 -> 60 loader steps in; loader_len 25 -> epoch 2, 10 steps into it, 5 optimizer steps
    assert parse_resume("out/step_30/", steps_per_epoch=13, loader_len=25, gas=2) == (2, 10, 5)


class _CountingSet(torch.utils.data.Dataset):
    """dataset of the integers 0..n-1 that records which items were actually fetched"""

    def __init__(self, n):
        self.n, self.fetched = n, []

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        self.fetched.append(i)
        return i


def test_epoch_count_does_not_depend_on_world_size():
    """ADVICE r1 (medium): with max_train_steps=None, num_train_epochs=E must mean E passes on any number of ranks"""
    from dalm_b200.training.utils.loop import plan_schedule
    assert plan_schedule(100, 1, 1, None) == (100, 1)                  # 8 ranks shard this to 13 steps/epoch: still 1 epoch
    assert plan_schedule(100, 2, 3, None) == (150, 3)
    assert plan_schedule(100, 1, 1, 250) == (250, 3)                   # an explicit step budget decides the epoch count
    src = open(os.path.join(ROOT, "dalm_b200", "training", "utils", "loop.py")).read()
    assert src.index("plan_schedule(len(loader)") < src.index("accelerator.prepare(model")   # derived before sharding


def test_sharded_loader_matches_accelerate_semantics():
    from dalm_b200.accel import ShardedLoader
    mk = lambda: torch.utils.data.DataLoader(_CountingSet(10), batch_size=1, collate_fn=lambda f: f[0])
    seen = [list(ShardedLoader(mk(), r, 4)) for r in range(4)]
    assert seen[0] == [0, 4, 8] and seen[1] == [1, 5, 9] and seen[2] == [2, 6, 0] and seen[3] == [3, 7, 1]
    assert all(len(ShardedLoader(mk(), r, 4)) == 3 for r in range(4))
    assert list(ShardedLoader(mk(), 0, 1, skip=7)) == [7, 8, 9]
    sl = ShardedLoader(mk(), 1, 2)
    out = []
    for b in sl:
        out.append((b, sl.end_of_dataloader))
    assert out[-1] == (9, True) and not out[0][1]


def test_sharded_loader_fetches_only_its_own_batches():
    """ADVICE r1: a rank must not materialise (fetch + collate) the other ranks' batches; all ranks still walk the SAME
    shuffled permutation (shared seed), so their batches are disjoint and cover the epoch"""
    from dalm_b200.accel import ShardedLoader
    got = []
    for r in range(4):
        ds = _CountingSet(64)
        g = torch.Generator(); g.manual_seed(7)
        dl = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=True, generator=g, collate_fn=lambda f: list(f))
        batches = list(ShardedLoader(dl, r, 4))
        assert len(batches) == 4 and len(ds.fetched) == 16             # 64 / 4 per batch / 4 ranks: own samples only
        got.append([i for b in batches for i in b])
    flat = sorted(i for g_ in got for i in g_)
    assert flat == list(range(64))                                     # disjoint cover of one shared permutation


def test_dalm_alias_is_the_same_module_object():
    """ADVICE r1 (high): `import dalm.X` must BE dalm_b200.X, not a second execution of it"""
    import importlib
    import dalm  # noqa: F401
    import dalm_b200.models.rag_e2e_base_model as real
    from dalm.models.rag_e2e_base_model import AutoModelForRagE2E as A1
    from dalm.models.rag_e2e_base_model import AutoModelForRagE2E as A2
    import dalm.models.rag_e2e_base_model as alias
    assert alias is real and A1 is A2 and A1 is real.AutoModelForRagE2E
    assert sys.modules["dalm_b200.models.rag_e2e_base_model"] is real and real.__spec__.name == real.__name__
    for sub in ("training.utils.train_utils", "training.rag_e2e.train_rage2e", "training.retriever_only.train_retriever_only",
                "eval.utils", "cli", "utils", "models.retriever_only_base_model"):
        assert importlib.import_module("dalm." + sub) is importlib.import_module("dalm_b200." + sub)
    import dalm.training.utils.train_utils as tu
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    import dalm.models.retriever_only_base_model as ro
    assert ro.AutoModelForSentenceEmbedding is AutoModelForSentenceEmbedding     # isinstance checks in save_model_hook hold
    assert tu.save_model_hook.__module__ == "dalm_b200.training.utils.train_utils"


def test_scheduler_wrapper_and_accumulate():
    from dalm_b200.accel import Accelerator
    acc = Accelerator(gradient_accumulation_steps=2, cpu=True)
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0 / (1 + s))
    opt2, sched2 = acc.prepare(opt, sched)
    steps = []
    for i in range(4):
        with acc.accumulate(None):
            steps.append(acc.sync_gradients)
            sched2.step()
    assert steps == [False, True, False, True]
    assert sched.last_epoch == 2               # stepped only on sync steps (x num_processes == 1)
    assert acc.reduce(torch.tensor(3.0)).item() == 3.0


def test_collate_and_lora_bank_layout():
    from dalm_b200.training.utils.loop import collate
    b = collate([{"a": [1, 2], "n": 3}, {"a": [4, 5], "n": 6}])
    assert b["a"].dtype == torch.int64 and b["a"].tolist() == [[1, 2], [4, 5]] and b["n"].tolist() == [3, 6]
    from dalm_b200.engine.lora import LoraBank
    bank = LoraBank([("m.q", 16, 24), ("m.v", 16, 8)], device="cpu")
    assert bank.numel() == 8 * 16 + 24 * 8 + 8 * 16 + 8 * 8
    assert bank.A["m.q"].shape == (8, 16) and bank.B["m.q"].shape == (24, 8)
    assert bank.B["m.q"].abs().max() == 0 and bank.A["m.q"].abs().max() <= 0.25 + 1e-6      # U(-1/sqrt(in), 1/sqrt(in))
    bank.gA["m.v"].fill_(1.0)
    assert bank.grad.sum().item() == 8 * 16                  # views alias the flat gradient buffer
    sd = bank.peft_state_dict()
    assert "base_model.model.m.q.lora_A.weight" in sd
    bank2 = LoraBank([("m.q", 16, 24), ("m.v", 16, 8)], device="cpu", seed=5)
    bank2.load_peft_state_dict(sd)
    assert torch.equal(bank2.flat, bank.flat)


def test_head_chunk_rows_plans_whole_tiles_within_budget():
    """row-chunk planner of the chunked lm_head + CE head (dalm_b200/ops.py): 128-row aligned, scratch within the budget,
    fewest wasted tile waves among the next few chunk counts"""
    from dalm_b200 import ops
    # cfg-3: 4608 rows x 32000 logits, 80 MB budget, 148 SMs -> 4 chunks of 9 m-tiles (1 152 rows, 74 MB): 32 waves vs 36 for 6 x 6
    assert ops.head_chunk_rows(4608, 32000, 80 << 20, sms=148) == 1152
    # cfg-5: 36 864 rows x 65 024 logits: L2-sized chunks for a frozen head, 512 MB chunks for a trainable one
    r_l2, r_full = ops.head_chunk_rows(36864, 65024, 80 << 20, sms=132), ops.head_chunk_rows(36864, 65024, 512 << 20, sms=132)
    assert r_l2 % 128 == 0 and r_l2 * 65024 * 2 <= 80 << 20 and r_full % 128 == 0 and r_full * 65024 * 2 <= 512 << 20 and r_full > r_l2
    # tiny problems: one 128-row tile per chunk at least, never zero
    assert ops.head_chunk_rows(5, 504, 1, sms=132) == 128 and ops.head_chunk_rows(300, 1000, 128 * 1000 * 2, sms=132) == 128
    for M, Vp, budget in ((4608, 32000, 80 << 20), (200, 504, 128 * 504 * 2), (36864, 65024, 512 << 20), (1000, 30528, 64 << 20)):
        rows = ops.head_chunk_rows(M, Vp, budget, sms=132)
        assert rows >= 128 and rows % 128 == 0
        assert sum(min(rows, M - r0) for r0 in range(0, M, rows)) == M          # the chunks tile the rows exactly


def test_cross_rank_negatives_switch_is_off_by_default(monkeypatch):
    from dalm_b200.training.utils import negatives
    monkeypatch.delenv("DALM_B200_CROSS_RANK_NEGATIVES", raising=False)
    assert not negatives.enabled() and not negatives.active()           # the reference's rank-local negatives are the default
    monkeypatch.setenv("DALM_B200_CROSS_RANK_NEGATIVES", "1")
    assert negatives.enabled() and not negatives.active()               # a single-process run has nobody to gather from


def test_nf4_storage_switch(monkeypatch):
    from dalm_b200.engine import nf4store
    from dalm_b200.models import rag_e2e_base_model as m
    monkeypatch.delenv("DALM_B200_NF4_STORAGE", raising=False)
    assert not nf4store.storage_enabled() and not m._nf4_storage(True, False, "bert")
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    assert m._nf4_storage(True, False, "llama") and not m._nf4_storage(False, False, "llama")
    import pytest
    with pytest.raises(NotImplementedError):
        m._nf4_storage(True, False, "falcon")                            # built for BERT encoders and Llama decoders
    with pytest.raises(NotImplementedError):
        m._nf4_storage(True, True, "llama")                              # 4-bit base weights cannot be fully fine-tuned


def test_packed_dataset_yields_the_same_batches_as_the_reference_pipeline(tmp_path):
    """DALM_B200_PACKED_LOADER: the memory-mapped int32 matrix + one gather per batch gives exactly the tensors that DataLoader +
    collate give on the tokenised rows - same shuffle, same rank shards (world 2), short last batch included; the on-disk cache
    is re-used and rejected when the layout changes"""
    import numpy as np
    import torch
    from torch.utils.data import DataLoader
    from dalm_b200.accel import ShardedLoader
    from dalm_b200.training.utils.loop import collate
    from dalm_b200.training.utils.packed_dataset import PackedDataset
    rng = np.random.default_rng(0)
    rows = [{"retriever_query_input_ids": rng.integers(0, 30000, 5).tolist(), "retriever_query_attention_mask": rng.integers(0, 2, 5).tolist(),
             "generator_input_input_ids": rng.integers(0, 32000, 9).tolist(), "query_passage_input_len": int(rng.integers(1, 300))}
            for _ in range(23)]
    path = str(tmp_path / "cache" / "packed_x")
    packed = PackedDataset.from_rows(rows, path)
    assert packed.matrix.shape == (23, 5 + 5 + 9 + 1) and packed.matrix.dtype == np.int32 and len(packed) == 23
    assert [c[0] for c in packed.columns] == list(rows[0]) and packed.columns[-1][2] == 0       # the scalar feature
    again = PackedDataset.from_rows(rows, path)                                                    # served from <path>.npy (mmap)
    assert isinstance(again.matrix, np.memmap) and np.array_equal(again.matrix, packed.matrix)
    wider = [dict(r, extra=1) for r in rows]
    assert PackedDataset.from_rows(wider, path).matrix.shape[1] == 21                              # other layout: rebuilt, not re-used

    def loaders():
        out = []
        for ds, cf in ((rows, collate), (packed, packed.collate)):
            g = torch.Generator(); g.manual_seed(42)
            out.append(DataLoader(ds, shuffle=True, collate_fn=cf, batch_size=4, generator=g))
        return out
    ref, got = loaders()
    n = 0
    for a, b in zip(ref, got):
        assert list(a) == list(b)
        for k in a:
            assert a[k].dtype == b[k].dtype == torch.int64 and a[k].shape == b[k].shape and torch.equal(a[k], b[k])
        n += 1
    assert n == 6                                                                                   # 5 full batches + one of 3
    for rank in (0, 1):                                                                             # index-level rank shards
        ref, got = loaders()
        for a, b in zip(ShardedLoader(ref, rank, 2), ShardedLoader(got, rank, 2)):
            assert all(torch.equal(a[k], b[k]) for k in a)
    import pytest
    with pytest.raises(ValueError):
        PackedDataset.from_rows([rows[0], dict(rows[1], generator_input_input_ids=[1, 2])])       # ragged feature: refused
    # an HF `datasets.Dataset` (what `dataset.map(preprocess)` returns) goes column by column and gets a fingerprint-keyed cache name
    import datasets
    hf = datasets.Dataset.from_dict({k: [r[k] for r in rows] for k in rows[0]})
    cp = PackedDataset.cache_path(hf, str(tmp_path / "cache"))
    assert cp is not None and os.path.basename(cp).startswith("packed_")
    from_hf = PackedDataset.from_rows(hf, cp)
    assert np.array_equal(from_hf.matrix, packed.matrix) and from_hf.columns == packed.columns
    assert PackedDataset.cache_path(rows, str(tmp_path)) is None                                   # plain lists: no fingerprint, in memory
