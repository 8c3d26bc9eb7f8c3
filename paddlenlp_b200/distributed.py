"""Data-parallel plumbing: one process per GPU, torch.distributed (NCCL over NVLink 5 / NVSwitch) as the carrier.

Replaces the reference's `paddle.distributed.init_parallel_env()` (trainer/training_args.py:1617-1625) and
`paddle.DataParallel` bucketed reducer / `fused_allreduce_gradients` (trainer.py:1934-1954, 1079-1110) with an
all-reduce(SUM) of the flat bf16 gradient buffer per optimizer step — issued range by range (one decoder layer at a time)
on a side stream as the last micro-batch's backward finalises them, or as ONE call when overlap is off; the 1/world_size
mean is folded into the optimizer kernel's grad_scale.  Pure replication: no parameter or optimizer-state sharding.
"""
from __future__ import annotations

import contextlib
import os
from typing import Optional

import torch
import torch.distributed as dist


def get_world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def get_rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def init_parallel_env(backend: Optional[str] = None):
    """Initialise from torchrun-style env (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 or (dist.is_available() and dist.is_initialized()):
        return
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    if backend == "nccl":
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group(backend="nccl", device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
    else:
        dist.init_process_group(backend=backend)


def allreduce_flat_(flat: torch.Tensor, group=None) -> torch.Tensor:
    """In-place SUM all-reduce of one contiguous buffer (the whole model's gradients)."""
    if get_world_size() > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    return flat


def broadcast_flat_(flat: torch.Tensor, src: int = 0, group=None) -> torch.Tensor:
    """Rank-0 parameter broadcast at wrap time (what paddle.DataParallel does in its constructor)."""
    if get_world_size() > 1:
        dist.broadcast(flat, src=src, group=group)
    return flat


def shard_rows(global_batch: int, rank: Optional[int] = None, world: Optional[int] = None):
    """Rows of a global batch owned by `rank`: contiguous blocks, rank r takes rows r*B : (r+1)*B (SURVEY.md §8d)."""
    rank = get_rank() if rank is None else rank
    world = get_world_size() if world is None else world
    if global_batch % world:
        raise ValueError(f"global batch {global_batch} is not divisible by world size {world}")
    per = global_batch // world
    return rank * per, (rank + 1) * per


class DataParallel(torch.nn.Module):
    """paddle.DataParallel stand-in: forwards to the wrapped model, owns the gradient exchange.

    The reference's reducer all-reduces 25 MB buckets while backward is still running (SURVEY.md §8a a12).  Here the
    gradients live in one flat buffer that is final piecewise — lm_head first (untied models only), then decoder layer
    L-1 ... 0, then the embedding and the norm/bias vectors — during the backward of the LAST micro-batch of an optimizer step.
    With tied embeddings there is no head range: the head's term goes into the embedding gradient at the start of backward,
    and that range is reported once, after the lookup's scatter has added to it.  The engine
    reports each finished range (`grad_ready_hook`); the range is all-reduced on a side stream while the remaining layers
    are still being differentiated, and `sync_gradients()` reduces whatever is left and joins.  Micro-batches run under
    `no_sync()` accumulate locally, exactly like the reference (trainer.py:1049-1075)."""

    def __init__(self, layers, find_unused_parameters: bool = False, group=None, overlap: bool = True):
        super().__init__()
        self._layers = layers
        self.group = group
        self._sync = True
        self.overlap = overlap
        self._pending = []          # (lo, hi, work) of ranges already handed to the collective
        self._comm_stream = None
        engine = getattr(layers, "engine", None)
        if engine is not None:
            broadcast_flat_(engine.flat_params, 0, group)

    def forward(self, *a, **kw):
        self.prepare_backward()
        return self._layers(*a, **kw)

    def prepare_backward(self):
        """Arm (or disarm, under no_sync) the overlap hook for the next engine.backward()."""
        eng = self._layers.engine
        eng.grad_ready_hook = self._on_ready if (self._sync and self.overlap and get_world_size() > 1) else None

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient accumulation micro-steps skip the exchange (trainer.py:1049-1075)."""
        old, self._sync = self._sync, False
        try:
            yield
        finally:
            self._sync = old

    def _on_ready(self, lo: int, hi: int):
        flat = self._layers.engine.flat_grads
        if hi <= lo:
            return
        if flat.is_cuda:
            if self._comm_stream is None:
                self._comm_stream = torch.cuda.Stream(device=flat.device)
            ev = torch.cuda.Event()
            ev.record()                                   # the range is final at this point of the compute stream
            with torch.cuda.stream(self._comm_stream):
                self._comm_stream.wait_event(ev)
                work = dist.all_reduce(flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        else:
            work = dist.all_reduce(flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        self._pending.append((lo, hi, work))

    def sync_gradients(self):
        """All-reduce every range of the flat gradient buffer that was not already reduced during backward, then make the
        current stream wait for all of them."""
        eng = self._layers.engine
        eng.grad_ready_hook = None
        flat = eng.flat_grads
        if get_world_size() > 1:
            done = sorted((lo, hi) for lo, hi, _ in self._pending)
            pos = 0
            for lo, hi in done + [(flat.numel(), flat.numel())]:
                if lo > pos:
                    dist.all_reduce(flat[pos:lo], op=dist.ReduceOp.SUM, group=self.group)
                pos = max(pos, hi)
            for _, _, work in self._pending:
                work.wait()
        self._pending = []

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self._layers, name)
