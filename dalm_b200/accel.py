"""Minimal stand-in for the part of HF `accelerate` the two reference trainers use (reference
dalm/training/rag_e2e/train_rage2e.py:28-30,276-295,366-374,392,416-430,469-490,503-527 and the same spots of
train_retriever_only.py). `accelerate` is a third-party package that is not installed offline and is unpinned in the
reference; the behaviours mirrored here are its documented ones — data-parallel sharding with one process per GPU,
gradient averaging, grad-accumulation gating, scheduler stepping, state save/load hooks. "parity unpinned" (DESIGN.md).

Collectives go through torch.distributed: NCCL over NVLink on GPUs, gloo in the CPU tests.
"""
from __future__ import annotations

import contextlib
import json
import logging
import os
import random
import time
from typing import Any, Callable, Dict, Iterable, List, Optional

import numpy as np
import torch
import torch.distributed as dist


def set_seed(seed: int) -> None:
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def nccl_env_defaults() -> None:
    """Must run before the NCCL communicator is created. Caps the CTAs (= SMs) NCCL's kernels may occupy: collectives that
    overlap the backward share the GPU with persistent one-CTA-per-SM GEMMs, which are launched on the remaining SMs
    (GradientSync / ops.GEMM_MAX_CTAS). DALM_B200_NCCL_CTAS overrides (0 = leave NCCL's default)."""
    n = os.environ.get("DALM_B200_NCCL_CTAS", "16")
    if n != "0":
        os.environ.setdefault("NCCL_MAX_CTAS", n)


class _RankLogger(logging.LoggerAdapter):
    """accelerate.logging.get_logger: `main_process_only` kwarg (default True)"""

    def log(self, level, msg, *args, **kwargs):
        main_only = kwargs.pop("main_process_only", True)
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else int(os.environ.get("RANK", 0))
        if not main_only or rank == 0:
            if self.isEnabledFor(level):
                self.logger.log(level, msg, *args, **kwargs)


def get_logger(name: str) -> _RankLogger:
    return _RankLogger(logging.getLogger(name), {})


class _BatchSamplerShard:
    """Rank r's share of a batch sampler, batch-strided like accelerate's BatchSamplerShard(split_batches=False,
    even_batches=True): global batches r, r+W, r+2W, ...; a short final round is completed by wrapping around to the first
    batches so every rank runs the same number of steps. Only INDEX lists are walked for the other ranks' batches - no
    sample of theirs is fetched or collated (every rank draws the same permutation from the shared, equally-seeded generator)."""

    def __init__(self, batch_sampler, rank: int, world: int, skip: int = 0):
        self.batch_sampler, self.rank, self.world, self.skip = batch_sampler, rank, world, skip

    def __len__(self) -> int:
        return max((len(self.batch_sampler) + self.world - 1) // self.world - self.skip, 0)

    def __iter__(self):
        first: List[Any] = []
        group: List[Any] = []
        emitted = 0
        for idx in self.batch_sampler:
            if len(first) < self.world:
                first.append(idx)
            group.append(idx)
            if len(group) == self.world:
                if emitted >= self.skip:
                    yield group[self.rank]
                emitted += 1
                group = []
        if group:
            pad = 0
            while len(group) < self.world:
                group.append(first[pad % len(first)])
                pad += 1
            if emitted >= self.skip:
                yield group[self.rank]


class ShardedLoader:
    """Per-rank view of a DataLoader (accelerate's `prepare(dataloader)`): the same dataset / collate_fn / pinning behind a
    `_BatchSamplerShard`, so a rank only materialises its own batches. `end_of_dataloader` is True while the last batch of
    an epoch is being consumed (what `Accelerator.accumulate` needs to force a gradient sync there)."""

    def __init__(self, loader, rank: int, world: int, skip: int = 0):
        self.loader, self.rank, self.world, self.skip = loader, rank, world, skip
        self.end_of_dataloader = False
        self.shard = _BatchSamplerShard(loader.batch_sampler, rank, world, skip)
        self._inner = torch.utils.data.DataLoader(loader.dataset, batch_sampler=self.shard, collate_fn=loader.collate_fn,
                                                  num_workers=loader.num_workers, pin_memory=loader.pin_memory)

    def __len__(self) -> int:
        return len(self.shard)

    def __iter__(self):
        self.end_of_dataloader = False
        total = len(self)
        for i, b in enumerate(self._inner):
            self.end_of_dataloader = i == total - 1
            yield b


class GradientSync:
    """The data-parallel exchange of one optimizer step as ONE collective (SURVEY C1/C2). The reference gets it implicitly:
    DDP averages the gradients (train_rage2e.py:416-418,471) and `accelerator.reduce(loss, "sum")` sums the scalar loss
    (:469) - two or more NCCL calls per step. Here every small trainable bank (the LoRA banks: 1.18 M + 4.19 M floats at
    cfg-3) has its flat gradient buffer RE-HOMED into one fp32 arena

        arena = [ bank_0.grad | bank_1.grad | ... | loss slot ]

    and `reduce(loss)` issues a single all-reduce(AVG) over it; the loss slot is pre-multiplied by the world size so that
    its average IS the rank sum the reference logs. Banks too large to copy around (a fully fine-tuned model's fp32 gradient
    bank: 27 GB at 7 B) stay where they are and are averaged in place, in buckets (see `reduce_large`).
    Build it BEFORE a step is captured into a CUDA graph: re-homing changes the kernels' output pointers."""

    ARENA_LIMIT = 64 << 20        # floats per bank (256 MB): anything larger is a dense bank and is reduced in place

    def __init__(self, banks, world: int, device, nccl: bool):
        self.world, self.nccl, self.grad_scale = world, nccl, 1.0
        self.small = [b for b in banks if hasattr(b, "rebind_grad") and b.grad.numel() <= self.ARENA_LIMIT]
        self.large = [b for b in banks if b not in self.small]
        pad = lambda n: (n + 63) // 64 * 64
        total = sum(pad(b.grad.numel()) for b in self.small) + 64
        self.arena = torch.zeros(total, dtype=torch.float32, device=device)
        off = 0
        if world > 1:                                          # single-process runs keep their buffers: nothing to exchange
            for b in self.small:
                n = b.grad.numel()
                b.rebind_grad(self.arena[off:off + n])
                off += pad(n)
        self.loss_slot = self.arena[total - 64:total - 63]
        self.collectives = 0                                   # issued so far (bench / tests read it)
        # full fine-tuning: per-layer buckets are averaged on a side stream WHILE the backward of the layers below runs
        # (what DDP's bucketed hooks give the reference, train_rage2e.py:416-418,471). `armed` is switched off on
        # gradient-accumulation micro-steps. Collectives issued from hooks cannot sit inside a captured CUDA graph: such
        # runs launch eagerly (a 230 ms step hides the launch cost).
        self.armed = True
        self.side = None
        self.gemm_cap = 0
        if world > 1 and self.large and nccl:
            reserve = int(os.environ.get("NCCL_MAX_CTAS", "0") or 0)
            if reserve > 0:                                    # leave NCCL's CTAs their SMs (see ops.GEMM_MAX_CTAS): applied from the
                sms = torch.cuda.get_device_properties(device).multi_processor_count
                self.gemm_cap = max(sms - reserve, 64)         # first bucket of a backward until the step's last collective is queued
        if world > 1 and self.large:
            if torch.cuda.is_available() and torch.device(device).type == "cuda":
                self.side = torch.cuda.Stream(device=device)
            for b in self.large:
                if hasattr(b, "bucket_hook"):
                    b.bucket_hook = self._on_bucket

    @property
    def overlaps_backward(self) -> bool:
        """True when collectives are issued during the backward (the step must not be a single captured CUDA graph)"""
        return self.world > 1 and any(getattr(b, "bucket_hook", None) is not None for b in self.large)

    def _on_bucket(self, bank, lo: int, hi: int) -> None:
        if not self.armed or self.world == 1:
            return
        if self.gemm_cap:
            from . import ops
            ops.GEMM_MAX_CTAS = self.gemm_cap                   # collectives are in flight from here on: the forward ran at full width
        if self.side is not None:
            self.side.wait_stream(torch.cuda.current_stream())     # the wgrads that produced [lo, hi) are ordered before it
            with torch.cuda.stream(self.side):
                self._avg(bank.grad[lo:hi])
        else:
            self._avg(bank.grad[lo:hi])
        bank.reduced.append((lo, hi))

    def _avg(self, t: torch.Tensor) -> None:
        if self.nccl:
            dist.all_reduce(t, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
            t.div_(self.world)
        self.collectives += 1

    def reduce_large(self) -> None:
        """whatever the backward did not announce (embedding / norm / bias gradients, or everything when no hook fired)"""
        for b in self.large:
            rest = b.unreduced_ranges() if hasattr(b, "unreduced_ranges") else [(0, b.grad.numel())]
            for lo, hi in rest:
                self._avg(b.grad[lo:hi])
            if hasattr(b, "reduced"):
                b.reduced = []
        if self.gemm_cap:
            from . import ops
            ops.GEMM_MAX_CTAS = 0
        if self.side is not None:
            torch.cuda.current_stream().wait_stream(self.side)      # bucket all-reduces must land before the optimizer

    def reduce(self, loss: torch.Tensor) -> torch.Tensor:
        """average every bank's gradients over the ranks and return the rank-SUMMED loss (0-d fp32 view into the arena,
        stream-ordered like any other tensor)"""
        if self.world == 1:
            return loss
        torch.mul(loss.detach().reshape(1).float(), float(self.world), out=self.loss_slot)
        self._avg(self.arena)
        self.reduce_large()
        return self.loss_slot[0]


class _SchedulerWrapper:
    """accelerate's AcceleratedScheduler: only steps when the optimizer really stepped, and num_processes times per
    step (split_batches=False) so that a schedule written for single-process step counts keeps its shape."""

    def __init__(self, sched, acc: "Accelerator"):
        self.sched, self.acc = sched, acc

    def step(self, *a, **k):
        if not self.acc.sync_gradients:
            return
        for _ in range(self.acc.num_processes):
            self.sched.step(*a, **k)

    def __getattr__(self, name):
        return getattr(self.sched, name)


class JsonlTracker:
    """stand-in for accelerate's trackers ("all" => tensorboard/wandb/...): metrics appended to <project_dir>/metrics.jsonl"""

    def __init__(self, project_dir: Optional[str]):
        self.path = os.path.join(project_dir, "metrics.jsonl") if project_dir else None
        self.project = None

    def start(self, project: str, config: Optional[Dict]) -> None:
        self.project = project
        if self.path:
            os.makedirs(os.path.dirname(self.path), exist_ok=True)
            with open(self.path, "a") as f:
                f.write(json.dumps({"project": project, "config": {k: str(v) for k, v in (config or {}).items()}}) + "\n")

    def log(self, values: Dict, step: Optional[int]) -> None:
        if self.path:
            with open(self.path, "a") as f:
                f.write(json.dumps({"step": step, "time": time.time(),
                                    **{k: float(v) for k, v in values.items()}}) + "\n")


class Accelerator:
    def __init__(self, log_with: Optional[str] = None, project_dir: Optional[str] = None,
                 gradient_accumulation_steps: int = 1, cpu: bool = False):
        world = int(os.environ.get("WORLD_SIZE", "1"))
        self.use_cuda = torch.cuda.is_available() and not cpu
        nccl_env_defaults()
        if world > 1 and not (dist.is_available() and dist.is_initialized()):
            if self.use_cuda:
                torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
            dist.init_process_group(backend="nccl" if self.use_cuda else "gloo")
        self.num_processes = dist.get_world_size() if dist.is_initialized() else 1
        self.process_index = dist.get_rank() if dist.is_initialized() else 0
        self.local_process_index = int(os.environ.get("LOCAL_RANK", self.process_index))
        self.device = torch.device("cuda", self.local_process_index) if self.use_cuda else torch.device("cpu")
        self.is_main_process = self.process_index == 0
        self.is_local_main_process = self.local_process_index == 0
        self.gradient_accumulation_steps = gradient_accumulation_steps
        self.sync_gradients = True
        self._accum_step = 0
        self._loader: Optional[ShardedLoader] = None
        self._save_hooks: List[Callable] = []
        self._load_hooks: List[Callable] = []
        self._models: List[torch.nn.Module] = []
        self._optimizers: List[Any] = []
        self._schedulers: List[Any] = []
        self.tracker = JsonlTracker(project_dir) if log_with else None
        self.project_dir = project_dir

    @property
    def state(self) -> str:
        return (f"Distributed environment: {'MULTI_GPU' if self.num_processes > 1 else 'NO'}\n"
                f"Num processes: {self.num_processes}\nProcess index: {self.process_index}\nDevice: {self.device}\n")

    # ---- object preparation ------------------------------------------------------------------------------------
    def prepare(self, *objs):
        out = []
        for o in objs:
            if isinstance(o, torch.utils.data.DataLoader):
                self._loader = ShardedLoader(o, self.process_index, self.num_processes)
                out.append(self._loader)
            elif isinstance(o, torch.nn.Module):
                self._models.append(o)
                out.append(o)
            elif isinstance(o, torch.optim.Optimizer):
                self._optimizers.append(o)
                out.append(o)
            elif hasattr(o, "step") and hasattr(o, "get_last_lr"):
                w = _SchedulerWrapper(o, self)
                self._schedulers.append(w)
                out.append(w)
            else:
                out.append(o)
        return tuple(out) if len(out) > 1 else out[0]

    def skip_first_batches(self, loader: ShardedLoader, num_batches: int) -> ShardedLoader:
        return ShardedLoader(loader.loader, loader.rank, loader.world, skip=num_batches)

    def unwrap_model(self, model):
        return model

    def get_state_dict(self, model):
        return model.state_dict()

    # ---- step control ------------------------------------------------------------------------------------------
    @contextlib.contextmanager
    def accumulate(self, model=None):
        self._accum_step += 1
        end = self._loader.end_of_dataloader if self._loader is not None else False
        self.sync_gradients = (self._accum_step % self.gradient_accumulation_steps == 0) or end
        yield

    def backward(self, loss: torch.Tensor) -> None:
        (loss / self.gradient_accumulation_steps).backward()

    def average_gradients(self, flat_grads: Iterable[torch.Tensor]) -> None:
        """DDP's gradient mean over ranks (reference: implicit in accelerator.prepare/backward), one all-reduce per
        flat LoRA gradient buffer, issued only on steps where the optimizer will step."""
        if self.num_processes == 1 or not self.sync_gradients:
            return
        nccl = dist.get_backend() == "nccl"
        for g in flat_grads:
            if nccl:
                dist.all_reduce(g, op=dist.ReduceOp.AVG)         # one pass: no separate divide over a 27 GB full-FT buffer
            else:
                dist.all_reduce(g, op=dist.ReduceOp.SUM)
                g.div_(self.num_processes)

    def gradient_sync(self, banks) -> GradientSync:
        """the step's single-collective reducer over the given trainable banks (see GradientSync)"""
        nccl = self.num_processes > 1 and dist.get_backend() == "nccl"
        return GradientSync(list(banks), self.num_processes, self.device, nccl)

    def reduce(self, tensor: torch.Tensor, reduction: str = "sum") -> torch.Tensor:
        if self.num_processes == 1:
            return tensor
        t = tensor.clone()
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        if reduction == "mean":
            t /= self.num_processes
        return t

    def wait_for_everyone(self) -> None:
        if self.num_processes > 1:
            dist.barrier()

    def print(self, *a, **k) -> None:
        if self.is_local_main_process:
            print(*a, **k)

    # ---- tracking ----------------------------------------------------------------------------------------------
    def init_trackers(self, project_name: str, config: Optional[Dict] = None) -> None:
        if self.tracker and self.is_main_process:
            self.tracker.start(project_name, config)

    def log(self, values: Dict, step: Optional[int] = None) -> None:
        if self.tracker and self.is_main_process:
            self.tracker.log(values, step)

    def end_training(self) -> None:
        pass

    # ---- checkpoints -------------------------------------------------------------------------------------------
    def register_save_state_pre_hook(self, hook: Callable) -> None:
        self._save_hooks.append(hook)

    def register_load_state_pre_hook(self, hook: Callable) -> None:
        self._load_hooks.append(hook)

    def save_state(self, output_dir: str) -> str:
        if self.is_main_process:
            os.makedirs(output_dir, exist_ok=True)
            weights = [dict() for _ in self._models]
            for h in self._save_hooks:
                h(list(self._models), weights, output_dir)
            for i, o in enumerate(self._optimizers):
                torch.save(o.state_dict(), os.path.join(output_dir, f"optimizer{'' if i == 0 else '_' + str(i)}.bin"))
            for i, s in enumerate(self._schedulers):
                torch.save(s.sched.state_dict(), os.path.join(output_dir, f"scheduler{'' if i == 0 else '_' + str(i)}.bin"))
            torch.save({"python": random.getstate(), "numpy": np.random.get_state(), "torch": torch.get_rng_state()},
                       os.path.join(output_dir, "random_states_0.pkl"))
        self.wait_for_everyone()
        return output_dir

    def load_state(self, input_dir: str) -> None:
        for h in self._load_hooks:
            h(list(self._models), input_dir)
        for i, o in enumerate(self._optimizers):
            p = os.path.join(input_dir, f"optimizer{'' if i == 0 else '_' + str(i)}.bin")
            if os.path.exists(p):
                o.load_state_dict(torch.load(p, map_location="cpu", weights_only=False))
        for i, s in enumerate(self._schedulers):
            p = os.path.join(input_dir, f"scheduler{'' if i == 0 else '_' + str(i)}.bin")
            if os.path.exists(p):
                s.sched.load_state_dict(torch.load(p, map_location="cpu", weights_only=False))
