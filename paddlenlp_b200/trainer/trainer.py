"""Trainer — the pure data-parallel subset of paddlenlp/trainer/trainer.py on the native engine.

Call pattern reproduced (SURVEY.md §3.1):
    Trainer(model, criterion, args, data_collator, train_dataset, ..., optimizers=(None, lr_scheduler))   :273-286
    .train()                        :687   -> _inner_training_loop :855
       training_step                :2211  (H2D of the batch, bf16 O2 forward, loss / grad_accum, loss.backward())
       gradient exchange            :1934-1954 / :1079-1110  -> ONE all-reduce of the flat gradient buffer
       optimizer.step / lr_scheduler.step / optimizer.clear_grad     :1171-1185
       _maybe_log_save_evaluate     :1388-1455 (all-gathered mean loss, speed_metrics keys of trainer_utils.py:351-380;
                                    evaluate() every eval_steps or at epoch end, then the checkpoint keeps the best metric)
    .evaluate() / .predict()        :2846-3286 (evaluation_loop, prediction_step)
Differences by design: the whole model's gradients live in one buffer, so there are no reducer buckets; gradient
averaging (1/world) is folded into the optimizer kernel; the step is host-sync free except at logging steps.
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
import random
import re
import shutil
import time
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional

import numpy as np
import torch

from .. import distributed as dist_env
from .. import ops
from ..optimizer import AdamW, ClipGradByGlobalNorm, get_scheduler
from ..utils.batch_sampler import DistributedBatchSampler
from .trainer_utils import EvalLoopOutput, EvalPrediction, IntervalStrategy, PredictionOutput
from .training_args import TrainingArguments


@dataclass
class TrainOutput:
    global_step: int
    training_loss: float
    metrics: Dict[str, float]


class TrainerCallback:
    def on_train_begin(self, args, state, control, **kw): ...
    def on_step_begin(self, args, state, control, **kw): ...
    def on_step_end(self, args, state, control, **kw): ...
    def on_log(self, args, state, control, logs=None, **kw): ...
    def on_evaluate(self, args, state, control, metrics=None, **kw): ...
    def on_train_end(self, args, state, control, **kw): ...


class PrinterCallback(TrainerCallback):
    def on_log(self, args, state, control, logs=None, **kw):
        if args.should_log and logs is not None:
            print(", ".join(f"{k}: {v}" for k, v in logs.items()), flush=True)


PREFIX_CHECKPOINT_DIR = "checkpoint"              # trainer_utils.py
TRAINER_STATE_NAME = "trainer_state.json"         # trainer.py:168
SCHEDULER_NAME = "scheduler.pdparams"             # trainer.py:171
TRAINING_ARGS_NAME = "training_args.json"


@dataclass
class TrainerState:
    """trainer_callback.py:47-118 (the fields the data-parallel loop maintains) with the same JSON round trip."""
    epoch: Optional[float] = 0.0
    global_step: int = 0
    max_steps: int = 0
    num_train_epochs: int = 0
    total_flos: float = 0
    log_history: Optional[List[Dict[str, float]]] = None
    best_metric: Optional[float] = None
    best_model_checkpoint: Optional[str] = None
    is_local_process_zero: bool = True
    is_world_process_zero: bool = True
    trial_name: Optional[str] = None
    trial_params: Optional[Dict[str, Any]] = None

    def __post_init__(self):
        if self.log_history is None:
            self.log_history = []

    def save_to_json(self, json_path: str):
        with open(json_path, "w", encoding="utf-8") as f:
            f.write(json.dumps(dataclasses.asdict(self), indent=2, sort_keys=True) + "\n")

    @classmethod
    def load_from_json(cls, json_path: str):
        with open(json_path, encoding="utf-8") as f:
            return cls(**json.load(f))


def get_last_checkpoint(folder: str) -> Optional[str]:
    """trainer_utils.py get_last_checkpoint: the `checkpoint-N` sub-directory with the largest N, or None."""
    if not os.path.isdir(folder):
        return None
    best = None
    for name in os.listdir(folder):
        m = re.fullmatch(PREFIX_CHECKPOINT_DIR + r"-(\d+)", name)
        if m and os.path.isdir(os.path.join(folder, name)) and (best is None or int(m.group(1)) > best[0]):
            best = (int(m.group(1)), name)
    return os.path.join(folder, best[1]) if best else None


class _PhaseTimers:
    """CUDA-event phase timers with the reference's four phase names (plugins/timer.py: read-data,
    forward-backward, all-reduce, optimizer-step); resolved lazily so they never block the stream."""

    NAMES = ("read-data", "forward-backward", "all-reduce", "optimizer-step")

    def __init__(self, enabled: bool):
        self.enabled = enabled
        self.pending: List = []
        self.totals = {n: 0.0 for n in self.NAMES}

    def start(self, name):
        if not self.enabled:
            return None
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
        return (name, e0)

    def stop(self, tok):
        if tok is None:
            return
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.pending.append((tok[0], tok[1], e1))

    def collect(self) -> Dict[str, float]:
        for name, e0, e1 in self.pending:
            e1.synchronize()
            self.totals[name] += e0.elapsed_time(e1)
        self.pending.clear()
        out, self.totals = self.totals, {n: 0.0 for n in self.NAMES}
        return out


class IterableDatasetShard(torch.utils.data.IterableDataset):
    """trainer_utils.py IterableDatasetShard: every process iterates the whole stream; of each group of
    `batch_size * num_processes` samples, process i keeps samples [i * batch_size, (i + 1) * batch_size).  A trailing partial
    group is dropped (drop_last) or completed by wrapping around to the first samples."""

    def __init__(self, dataset, batch_size: int = 1, drop_last: bool = False, num_processes: int = 1, process_index: int = 0):
        self.dataset, self.batch_size, self.drop_last = dataset, batch_size, drop_last
        self.num_processes, self.process_index = num_processes, process_index

    def __iter__(self):
        real = self.batch_size * self.num_processes
        lo, hi = self.process_index * self.batch_size, (self.process_index + 1) * self.batch_size
        first, cur = None, []
        for el in self.dataset:
            cur.append(el)
            if len(cur) == real:
                yield from cur[lo:hi]
                if first is None:
                    first = list(cur)
                cur = []
        if cur and not self.drop_last:
            if first is None:
                first = list(cur)
            while len(cur) < real:
                cur += first
            yield from cur[lo:hi]


def set_seed(seed: int = 1234, topo=None):
    """trainer_utils.py set_seed (pure data parallel: the same seed on every rank; data order is de-correlated by the sampler)."""
    import numpy as np

    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def speed_metrics(split, start_time, num_samples=None, num_steps=None, seq_length=None, model_flops=None):
    """trainer_utils.py:351-380 — the runtime / samples-per-second / tokens-per-second-per-device / hardware-TFLOPS keys."""
    runtime = time.time() - start_time
    result = {f"{split}_runtime": round(runtime, 4)}
    if num_samples is not None:
        sps = num_samples / runtime
        result[f"{split}_samples_per_second"] = round(sps, 4)
        if seq_length is not None:
            tps = sps * seq_length / dist_env.get_world_size()
            result[f"{split}_tokens_per_second_per_device"] = round(tps, 4)
            if model_flops is not None:
                result[f"{split}_hardware_tflops_per_device"] = round(tps * model_flops / seq_length / 2 ** 40, 2)
    if num_steps is not None:
        result[f"{split}_steps_per_second"] = round(num_steps / runtime, 4)
    return result


def _pad_concat(a: Optional[np.ndarray], b: np.ndarray, padding_index: int = -100) -> np.ndarray:
    """trainer_utils nested_concat: concatenate along the batch axis, right-padding axis 1 with padding_index when the
    sequence lengths differ."""
    if a is None:
        return b
    if a.ndim == 1 or a.shape[1] == b.shape[1]:
        return np.concatenate((a, b), axis=0)
    shape = (a.shape[0] + b.shape[0], max(a.shape[1], b.shape[1])) + a.shape[2:]
    out = np.full(shape, padding_index, dtype=a.dtype)
    out[:a.shape[0], :a.shape[1]] = a
    out[a.shape[0]:, :b.shape[1]] = b
    return out


def _batch_size(inputs) -> Optional[int]:
    """trainer_utils find_batch_size: leading dimension of the first tensor of a batch."""
    for v in (inputs.values() if isinstance(inputs, dict) else inputs):
        if isinstance(v, torch.Tensor) and v.dim() > 0:
            return v.shape[0]
    return None


def default_data_collator(features: List[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
    out = {}
    for k in features[0]:
        out[k] = torch.stack([torch.as_tensor(f[k]) for f in features])
    return out


class Trainer:
    def __init__(self, model=None, criterion=None, args: Optional[TrainingArguments] = None, data_collator=None,
                 train_dataset=None, eval_dataset=None, tokenizer=None, compute_metrics=None,
                 callbacks: Optional[List[TrainerCallback]] = None, optimizers=(None, None)):
        if args is None:
            args = TrainingArguments()
        self.args = args
        self.model = model
        self.criterion = criterion
        self.data_collator = data_collator or default_data_collator
        self.train_dataset = train_dataset
        self.eval_dataset = eval_dataset
        self.tokenizer = tokenizer
        self.compute_metrics = compute_metrics
        self.optimizer, self.lr_scheduler = optimizers
        self.callbacks = list(callbacks or []) + [PrinterCallback()]
        self.state = TrainerState(log_history=[])
        self.control = None
        self.model_wrapped = model
        self.timers = _PhaseTimers(not args.skip_profile_timer)
        torch.manual_seed(args.seed)

    # ------------------------------------------------------------------------------------------------
    def get_train_dataloader(self):
        """trainer.py:1457-1530 (_get_train_sampler / get_train_dataloader): a SHUFFLING batch sampler — `BatchSampler(shuffle=True)`
        for one process, `DistributedBatchSampler(shuffle=True)` across ranks — re-seeded per epoch (`set_epoch`) so that resume
        can skip the consumed batches deterministically; an IterableDataset is sharded by rank (`IterableDatasetShard`)."""
        a = self.args
        ds = self.train_dataset
        if ds is None:
            raise ValueError("Trainer: training requires a train_dataset.")
        world, rank = a.dataset_world_size, a.dataset_rank
        if isinstance(ds, torch.utils.data.IterableDataset):
            if world > 1:
                ds = IterableDatasetShard(ds, batch_size=a.per_device_train_batch_size, drop_last=a.dataloader_drop_last,
                                          num_processes=world, process_index=rank)
            return torch.utils.data.DataLoader(ds, batch_size=a.per_device_train_batch_size, collate_fn=self.data_collator,
                                               num_workers=a.dataloader_num_workers, pin_memory=True)
        sampler = self._get_train_sampler()
        if hasattr(sampler, "batch_size") and not isinstance(sampler, torch.utils.data.Sampler):
            # a BATCH sampler (paddlenlp.utils.batch_sampler.DistributedBatchSampler — what run_pretrain.py:341-349 returns)
            return torch.utils.data.DataLoader(ds, batch_sampler=sampler, collate_fn=self.data_collator,
                                               num_workers=a.dataloader_num_workers, pin_memory=True)
        return torch.utils.data.DataLoader(ds, batch_size=a.per_device_train_batch_size, sampler=sampler, shuffle=False,
                                           collate_fn=self.data_collator, drop_last=a.dataloader_drop_last,
                                           num_workers=a.dataloader_num_workers, pin_memory=True)

    def _get_train_sampler(self, shuffle: bool = True):
        """trainer.py:1328-1347.  Subclasses override it the way llm/run_pretrain.py:341-349 does (PretrainingTrainer keeps the
        file order: shuffle=False).  DistributedSampler with one replica is a seeded shuffling sampler with set_epoch(): the same
        class serves the single-process and the data-parallel case."""
        a = self.args
        world, rank = a.dataset_world_size, a.dataset_rank
        return torch.utils.data.distributed.DistributedSampler(self.train_dataset, num_replicas=max(1, world),
                                                               rank=rank if world > 1 else 0, shuffle=shuffle, seed=int(a.seed),
                                                               drop_last=a.dataloader_drop_last)

    def create_optimizer_and_scheduler(self, num_training_steps: int):
        self.create_scheduler(num_training_steps)
        self.create_optimizer(self.lr_scheduler)

    def create_scheduler(self, num_training_steps: int):
        a = self.args
        if self.lr_scheduler is None:
            warmup = a.warmup_steps if a.warmup_steps > 0 else int(a.warmup_ratio * num_training_steps)
            decay = a.decay_steps if a.decay_steps > 0 else num_training_steps
            self.lr_scheduler = get_scheduler(a.lr_scheduler_type, learning_rate=a.learning_rate, num_warmup_steps=warmup,
                                              num_training_steps=decay, num_cycles=a.num_cycles)
        return self.lr_scheduler

    def create_optimizer(self, lr_scheduler=None):
        a = self.args
        if self.optimizer is None:
            # trainer.py:1730-1748: decay only parameters without "bias"/"norm" in the name == the matrices, which the
            # engine lays out first in the flat buffer (decay_end).
            self.optimizer = AdamW(learning_rate=(lr_scheduler.get_lr if lr_scheduler is not None else a.learning_rate),
                                   beta1=a.adam_beta1, beta2=a.adam_beta2, epsilon=a.adam_epsilon,
                                   weight_decay=a.weight_decay,
                                   grad_clip=ClipGradByGlobalNorm(a.max_grad_norm) if a.max_grad_norm > 0 else None,
                                   multi_precision=True, engine=self._engine())
        return self.optimizer

    def _engine(self):
        m = self.model
        return getattr(m, "engine", None) or getattr(getattr(m, "_layers", None), "engine", None)

    def _wrap_model(self, model):
        # trainer.py:1934-1954: world_size > 1 and not hybrid -> paddle.DataParallel(model)
        if self.args.world_size > 1 and not isinstance(model, dist_env.DataParallel):
            model = dist_env.DataParallel(model, find_unused_parameters=bool(self.args.ddp_find_unused_parameters))
        return model

    # ------------------------------------------------------------------------------------------------
    def _prepare_inputs(self, inputs: Dict[str, Any]) -> Dict[str, Any]:
        """Pinned host -> device (trainer.py:2099-2114)."""
        dev = self._engine().device
        ms = inputs.get("attn_mask_startend_row_indices")
        if isinstance(ms, torch.Tensor) and not ms.is_cuda:
            ops.check_mask_form(ms)             # every batch, before the copy: a host check adds no device sync to the step
        out = {}
        for k, v in inputs.items():
            if isinstance(v, torch.Tensor):
                if not v.is_cuda and not v.is_pinned():
                    v = v.pin_memory()
                out[k] = v.to(dev, non_blocking=True)
            else:
                out[k] = v
        return out

    def compute_loss(self, model, inputs, return_outputs=False):
        """trainer.py:2157-2197: criterion(outputs, labels) when a criterion is given, else the model's own loss.

        With the built-in pre-training criterion (LlamaPretrainingCriterion / Qwen2PretrainingCriterion: masked-mean fp32 CE)
        the labels are handed to the model so that the fused head + criterion path runs (same value, no second logits
        buffer) with the criterion's ignore_index.  Any other callable receives differentiable logits: the model keeps its
        activations and `loss.backward()` feeds d(logits) into the engine's explicit backward."""
        if self.criterion is not None:
            from ..transformers.llama.modeling import LlamaPretrainingCriterion

            inputs = dict(inputs)
            labels = inputs.pop("labels")
            inner = getattr(model, "_layers", model)
            if isinstance(self.criterion, LlamaPretrainingCriterion) and hasattr(inner, "criterion"):
                old = inner.criterion.ignore_index
                inner.criterion.ignore_index = self.criterion.ignore_index
                try:
                    outputs = model(**inputs, labels=labels)
                finally:
                    inner.criterion.ignore_index = old
                loss = outputs[0] if isinstance(outputs, (tuple, list)) else outputs.loss
            else:
                outputs = model(**inputs)
                logits = outputs[0] if isinstance(outputs, (tuple, list)) else outputs.logits
                loss = self.criterion(logits, labels)
        else:
            outputs = model(**inputs)
            loss = outputs[0] if isinstance(outputs, (tuple, list)) else outputs.loss
        return (loss, outputs) if return_outputs else loss

    def training_step(self, model, inputs) -> torch.Tensor:
        """trainer.py:2211-2244."""
        inputs = self._prepare_inputs(inputs)
        loss = self.compute_loss(model, inputs)
        if self.args.gradient_accumulation_steps > 1:
            loss = loss / self.args.gradient_accumulation_steps
        loss.backward()
        return loss.detach()

    # ------------------------------------------------------------------------------------------------
    def train(self, resume_from_checkpoint=None) -> TrainOutput:
        a = self.args
        if resume_from_checkpoint is None:
            resume_from_checkpoint = a.resume_from_checkpoint
        if resume_from_checkpoint is True:                       # trainer.py:569-580: newest checkpoint-N in output_dir
            resume_from_checkpoint = get_last_checkpoint(a.output_dir)
            if resume_from_checkpoint is None:
                raise ValueError(f"No valid checkpoint found in output directory ({a.output_dir})")
        if resume_from_checkpoint:
            self._load_from_checkpoint(resume_from_checkpoint)
        dl = self.get_train_dataloader()
        if a.evaluation_strategy != IntervalStrategy.NO and self.eval_dataset is None:
            raise ValueError(f"evaluation_strategy={a.evaluation_strategy}: training with evaluation requires an eval_dataset")
        accum = max(1, a.gradient_accumulation_steps)
        try:
            steps_per_epoch = max(len(dl) // accum, 1)
        except TypeError:
            steps_per_epoch = None
        if a.max_steps > 0:
            max_steps = a.max_steps
            epochs = math.ceil(max_steps / steps_per_epoch) if steps_per_epoch else 10 ** 9
        else:
            if steps_per_epoch is None:
                raise ValueError("max_steps must be set for iterable datasets")
            max_steps = math.ceil(a.num_train_epochs * steps_per_epoch)
            epochs = math.ceil(a.num_train_epochs)
        self.state.max_steps = max_steps
        if a.amp_master_grad:
            # trainer.py:1921-1960: fp32 main_grad for every parameter, before the optimizer and the data-parallel wrapper
            getattr(self.model, "_layers", self.model).set_master_grad(True)
        # wrap first: the wrapper broadcasts rank 0's parameters, and AdamW copies its fp32 master weights from the
        # parameters it finds, so every rank starts from rank 0's weights even when the ranks initialised differently
        model = self._wrap_model(self.model)
        self.model_wrapped = model
        self.create_optimizer_and_scheduler(max_steps)
        engine = self._engine()
        world = a.world_size
        self.optimizer.grad_scale = 1.0 / world
        self.optimizer.clear_grad()
        # trainer.py:872-905: restore state, then skip the epochs / batches already consumed
        epochs_trained, skip_batches = 0, 0
        if resume_from_checkpoint:
            self._load_optimizer_and_scheduler(resume_from_checkpoint)
            self.state = TrainerState.load_from_json(os.path.join(resume_from_checkpoint, TRAINER_STATE_NAME))
            self.state.max_steps = max_steps
            self._load_rng_state(resume_from_checkpoint)
            if not a.ignore_data_skip and steps_per_epoch:
                epochs_trained = self.state.global_step // steps_per_epoch
                skip_batches = (self.state.global_step % steps_per_epoch) * accum
        self.state.num_train_epochs = epochs
        self.state.is_world_process_zero = a.process_index == 0
        for cb in self.callbacks:
            cb.on_train_begin(a, self.state, self.control)

        dev = engine.device
        tr_loss = torch.zeros((), dtype=torch.float32, device=dev)
        logged_loss_total = 0.0
        logged_step = 0
        t_log = time.time()
        t_start = t_log
        seq_len = a.max_seq_length or getattr(self.model.config, "seq_length", None)
        done = False
        logged_step = self.state.global_step
        for epoch in range(epochs_trained, epochs):
            for sampler in (getattr(dl, "batch_sampler", None), getattr(dl, "sampler", None)):
                if hasattr(sampler, "set_epoch"):
                    sampler.set_epoch(epoch)
                    break
            it = iter(dl)
            step = -1
            if epoch == epochs_trained and skip_batches:
                for _ in range(skip_batches):                    # trainer.py:1005-1020 (skip_first_batches)
                    next(it)
                step = skip_batches - 1
            while True:
                tok = self.timers.start("read-data")
                try:
                    inputs = next(it)
                except StopIteration:
                    break
                self.timers.stop(tok)
                step += 1
                if step % accum == 0:
                    for cb in self.callbacks:
                        cb.on_step_begin(a, self.state, self.control)
                last_micro = (step + 1) % accum == 0
                tok = self.timers.start("forward-backward")
                if world > 1 and not last_micro:
                    with model.no_sync():            # trainer.py:1049-1075: accumulation micro-steps skip the exchange
                        tr_loss += self.training_step(model, inputs)
                else:
                    tr_loss += self.training_step(model, inputs)
                self.timers.stop(tok)
                if not last_micro:
                    continue
                tok = self.timers.start("all-reduce")
                if world > 1:
                    model.sync_gradients()
                self.timers.stop(tok)
                tok = self.timers.start("optimizer-step")
                self.optimizer.step()
                self.lr_scheduler.step()
                self.optimizer.clear_grad()
                self.timers.stop(tok)
                self.state.global_step += 1
                self.state.epoch = epoch + (step + 1) / max(1, (steps_per_epoch or 1) * accum)
                for cb in self.callbacks:
                    cb.on_step_end(a, self.state, self.control)
                gs = self.state.global_step
                if (a.logging_steps > 0 and gs % a.logging_steps == 0) or (a.logging_first_step and gs == 1):
                    # trainer.py:1388-1455: mean of the all-gathered loss over the interval
                    loss_t = tr_loss.clone()
                    if world > 1:
                        torch.distributed.all_reduce(loss_t)
                        loss_t /= world
                    loss_val = loss_t.item()
                    tr_loss.zero_()
                    nsteps = gs - logged_step
                    dt = time.time() - t_log
                    samples = nsteps * a.per_device_train_batch_size * accum * world
                    logs = {"loss": round(loss_val / nsteps, 8), "learning_rate": float(f"{self.optimizer.get_lr():.3e}"),
                            "global_step": gs, "interval_runtime": round(dt, 4),
                            "interval_samples_per_second": round(samples / dt, 4),
                            "interval_steps_per_second": round(nsteps / dt, 4)}
                    if seq_len:
                        tps = samples / dt * seq_len / world
                        logs["interval_tokens_per_second_per_device"] = round(tps, 4)
                        if hasattr(self.model, "get_model_flops"):
                            logs["interval_hardware_tflops_per_device"] = round(
                                tps * self.model.get_model_flops(seq_length=seq_len) / seq_len / 2 ** 40, 2)
                            logs["interval_algorithmic_tflops_per_device"] = round(
                                tps * self.model.get_algorithmic_flops_per_token(seq_len) / 1e12, 2)
                    if not a.skip_profile_timer:
                        logs.update({f"timer_{k}_ms": round(v, 2) for k, v in self.timers.collect().items()})
                    if math.isnan(loss_val) or math.isinf(loss_val):
                        raise ValueError(f"PaddleRecall error(102): Loss contains inf or nan values, its value is {loss_val}")
                    logged_loss_total += loss_val
                    logged_step = gs
                    t_log = time.time()
                    self.log(logs)
                metrics = None
                if a.evaluation_strategy == IntervalStrategy.STEPS and gs % a.eval_steps == 0:
                    metrics = self.evaluate()
                if a.save_strategy == IntervalStrategy.STEPS and a.save_steps > 0 and gs % a.save_steps == 0:
                    self._save_checkpoint(model, metrics=metrics)
                if gs >= max_steps:
                    done = True
                    break
            metrics = None                                       # trainer_callback.py:463-474: epoch-end events
            if a.evaluation_strategy == IntervalStrategy.EPOCH:
                metrics = self.evaluate()
            if a.save_strategy == IntervalStrategy.EPOCH:
                self._save_checkpoint(model, metrics=metrics)
            if done:
                break
        torch.cuda.synchronize(dev)
        if a.load_best_model_at_end and self.state.best_model_checkpoint is not None:    # trainer.py:1231-1260
            self._load_from_checkpoint(self.state.best_model_checkpoint)
        if self.state.global_step > logged_step:
            loss_t = tr_loss.clone()
            if world > 1:
                torch.distributed.all_reduce(loss_t)
                loss_t /= world
            logged_loss_total += loss_t.item()
        runtime = time.time() - t_start
        gs = max(1, self.state.global_step)
        metrics = {"train_runtime": round(runtime, 4),
                   "train_samples_per_second": round(gs * a.per_device_train_batch_size * accum * world / runtime, 4),
                   "train_steps_per_second": round(gs / runtime, 4), "train_loss": logged_loss_total / gs}
        for cb in self.callbacks:
            cb.on_train_end(a, self.state, self.control)
        return TrainOutput(self.state.global_step, logged_loss_total / gs, metrics)

    # ------------------------------------------------------------------------------------------------
    # evaluation  (trainer.py:1555-1660 eval / test dataloaders, :2846-3286 evaluate, predict, evaluation_loop,
    # prediction_step)
    # ------------------------------------------------------------------------------------------------
    def _get_eval_sampler(self, eval_dataset):
        """Every sample once, in order: sequential batches for one process; across ranks, DistributedBatchSampler without
        shuffling, whose last global batch wraps around to the first samples (evaluation_loop truncates them away)."""
        a = self.args
        if a.dataset_world_size <= 1:
            return torch.utils.data.BatchSampler(torch.utils.data.SequentialSampler(eval_dataset),
                                                 batch_size=a.per_device_eval_batch_size, drop_last=False)
        return DistributedBatchSampler(eval_dataset, batch_size=a.per_device_eval_batch_size, num_replicas=a.dataset_world_size,
                                       rank=a.dataset_rank, shuffle=False, drop_last=False)

    def _eval_dataloader(self, ds):
        a = self.args
        if isinstance(ds, torch.utils.data.IterableDataset):
            if a.dataset_world_size > 1:
                ds = IterableDatasetShard(ds, batch_size=a.per_device_eval_batch_size, drop_last=a.dataloader_drop_last,
                                          num_processes=a.dataset_world_size, process_index=a.dataset_rank)
            return torch.utils.data.DataLoader(ds, batch_size=a.per_device_eval_batch_size, collate_fn=self.data_collator)
        return torch.utils.data.DataLoader(ds, batch_sampler=self._get_eval_sampler(ds), collate_fn=self.data_collator,
                                           num_workers=a.dataloader_num_workers)

    def get_eval_dataloader(self, eval_dataset=None):
        if eval_dataset is None and self.eval_dataset is None:
            raise ValueError("Trainer: evaluation requires an eval_dataset.")
        return self._eval_dataloader(eval_dataset if eval_dataset is not None else self.eval_dataset)

    def get_test_dataloader(self, test_dataset):
        if test_dataset is None:
            raise ValueError("Trainer: prediction requires a test_dataset.")
        return self._eval_dataloader(test_dataset)

    def evaluate(self, eval_dataset=None, ignore_keys: Optional[List[str]] = None, metric_key_prefix: str = "eval"):
        """Loss (and `compute_metrics` of the predictions, when given) over the evaluation set; logged and returned."""
        dl = self.get_eval_dataloader(eval_dataset)
        start = time.time()
        output = self.evaluation_loop(dl, description="Evaluation",
                                      prediction_loss_only=True if self.compute_metrics is None else None,
                                      ignore_keys=ignore_keys, metric_key_prefix=metric_key_prefix,
                                      max_eval_iters=self.args.max_evaluate_steps)
        total_batch = self.args.eval_batch_size * self.args.dataset_world_size
        output.metrics.update(speed_metrics(metric_key_prefix, start, num_samples=output.num_samples,
                                            num_steps=math.ceil(output.num_samples / total_batch)))
        self.log(output.metrics)
        self.state.log_history[-1].setdefault("global_step", self.state.global_step)
        for cb in self.callbacks:
            cb.on_evaluate(self.args, self.state, self.control, metrics=output.metrics)
        return output.metrics

    def predict(self, test_dataset, ignore_keys: Optional[List[str]] = None, metric_key_prefix: str = "test"):
        dl = self.get_test_dataloader(test_dataset)
        start = time.time()
        output = self.evaluation_loop(dl, description="Prediction", ignore_keys=ignore_keys,
                                      prediction_loss_only=True if self.compute_metrics is None else None,
                                      metric_key_prefix=metric_key_prefix, max_eval_iters=self.args.max_evaluate_steps)
        total_batch = self.args.per_device_eval_batch_size * self.args.dataset_world_size
        output.metrics.update(speed_metrics(metric_key_prefix, start, num_samples=output.num_samples,
                                            num_steps=math.ceil(output.num_samples / total_batch)))
        return PredictionOutput(predictions=output.predictions, label_ids=output.label_ids, metrics=output.metrics)

    def _nested_gather(self, t: torch.Tensor) -> torch.Tensor:
        """Concatenation over ranks (rank order) along axis 0; every rank passes the same shape."""
        world = self.args.world_size
        if world <= 1:
            return t
        parts = [torch.empty_like(t) for _ in range(world)]
        torch.distributed.all_gather(parts, t.contiguous())
        return torch.cat(parts, dim=0)

    def _pad_across_processes(self, t: torch.Tensor, padding_index: int = -100) -> torch.Tensor:
        """Right-pad axis 1 to the longest sequence of any rank, so that _nested_gather can stack the batches."""
        if self.args.world_size <= 1 or t.dim() < 2:
            return t
        n = torch.tensor([t.shape[1]], device=t.device)
        torch.distributed.all_reduce(n, op=torch.distributed.ReduceOp.MAX)
        n = int(n.item())
        if n == t.shape[1]:
            return t
        out = t.new_full((t.shape[0], n) + tuple(t.shape[2:]), padding_index)
        out[:, :t.shape[1]] = t
        return out

    def evaluation_loop(self, dataloader, description: str, prediction_loss_only: Optional[bool] = None,
                        ignore_keys: Optional[List[str]] = None, metric_key_prefix: str = "eval",
                        max_eval_iters: Optional[int] = -1) -> EvalLoopOutput:
        """trainer.py:3016-3104.  Each batch's loss, repeated batch-size times, is gathered over the ranks; predictions and
        labels are gathered, padded with -100 and concatenated in sample order.  All three are truncated to num_samples
        (len(dataset), or batch * world * max_eval_iters when the iterations are capped), so the samples the sampler
        repeats to even out the ranks are dropped, and eval_loss is the mean of what remains.  The losses stay on the
        device until that mean: a loss-only evaluation synchronises once."""
        a = self.args
        prediction_loss_only = prediction_loss_only if prediction_loss_only is not None else a.prediction_loss_only
        max_eval_iters = max_eval_iters if max_eval_iters is not None else -1
        model = self.model
        batch_size = getattr(dataloader.batch_sampler, "batch_size", None) or dataloader.batch_size
        world = a.dataset_world_size
        num_samples = batch_size * world * max_eval_iters if max_eval_iters > 0 else None
        losses: List[torch.Tensor] = []
        all_preds = all_labels = None
        observed = 0
        model.eval()
        # evaluation draws nothing from the host RNG that training may use (the DataLoader seeds itself from it)
        with torch.random.fork_rng(devices=[]):
            for step, inputs in enumerate(dataloader):
                bs = _batch_size(inputs)
                if bs is not None:
                    observed += bs
                    batch_size = bs
                loss, logits, labels = self.prediction_step(model, inputs, prediction_loss_only, ignore_keys=ignore_keys)
                if loss is not None:
                    losses.append(self._nested_gather(loss.detach().float().reshape(1).repeat(batch_size)))
                if labels is not None:
                    labels = self._nested_gather(self._pad_across_processes(labels.detach()))
                    all_labels = _pad_concat(all_labels, labels.cpu().numpy())
                if logits is not None:
                    logits = self._nested_gather(self._pad_across_processes(logits.detach()))
                    all_preds = _pad_concat(all_preds, logits.float().cpu().numpy() if logits.is_floating_point()
                                            else logits.cpu().numpy())
                if max_eval_iters > 0 and step >= max_eval_iters - 1:
                    break
        model.train()
        if num_samples is None:
            try:
                num_samples = len(dataloader.dataset)
            except TypeError:                                    # an iterable dataset: what the ranks saw
                num_samples = observed * world
        if all_preds is not None:
            all_preds = all_preds[:num_samples]
        if all_labels is not None:
            all_labels = all_labels[:num_samples]
        metrics = {}
        if self.compute_metrics is not None and all_preds is not None and all_labels is not None:
            metrics = dict(self.compute_metrics(EvalPrediction(predictions=all_preds, label_ids=all_labels)))
        if losses:
            metrics[f"{metric_key_prefix}_loss"] = torch.cat(losses)[:num_samples].double().mean().item()
        for key in list(metrics):
            if not key.startswith(f"{metric_key_prefix}_"):
                metrics[f"{metric_key_prefix}_{key}"] = metrics.pop(key)
        return EvalLoopOutput(predictions=all_preds, label_ids=all_labels, metrics=metrics, num_samples=num_samples)

    def _fused_eval_ignore_index(self) -> Optional[int]:
        """ignore_index of the built-in pre-training criterion when it computes the loss (no criterion, or a
        LlamaPretrainingCriterion / Qwen2PretrainingCriterion), else None: a custom criterion needs the logits."""
        from ..transformers.llama.modeling import LlamaPretrainingCriterion

        inner = getattr(self.model, "_layers", self.model)
        if self._engine() is None or not isinstance(getattr(inner, "criterion", None), LlamaPretrainingCriterion):
            return None
        if self.criterion is None:
            return inner.criterion.ignore_index
        return self.criterion.ignore_index if isinstance(self.criterion, LlamaPretrainingCriterion) else None

    def _forward_eval(self, inputs, ignore_index: int, predictions: bool):
        """engine.forward_eval on a prepared batch: (loss_out [2], preds [B, S] or None), on the device."""
        from ..transformers.llama.modeling import _resolve_mask

        ms = _resolve_mask(inputs.get("attention_mask"), inputs.get("attn_mask_startend_row_indices"))
        return self._engine().forward_eval(inputs["input_ids"], inputs["labels"], inputs.get("position_ids"), ignore_index,
                                           attn_mask_startend_row_indices=ms, predictions=predictions)

    def prediction_step(self, model, inputs, prediction_loss_only: bool, ignore_keys: Optional[List[str]] = None):
        """(loss, logits, labels) of one batch, each optional.  With the built-in criterion a loss-only step runs the
        engine's chunked evaluation forward (no [T, V] logits); otherwise the model forward (or compute_loss with a
        custom criterion) under no_grad."""
        has_labels = inputs.get("labels") is not None
        inputs = self._prepare_inputs(inputs)
        labels = inputs["labels"] if has_labels else None
        ignore_keys = list(ignore_keys or [])
        with torch.no_grad():
            if has_labels and prediction_loss_only:
                ign = self._fused_eval_ignore_index()
                if ign is not None:
                    loss_out, _ = self._forward_eval(inputs, ign, predictions=False)
                    return loss_out[0], None, None
            if has_labels:
                loss, outputs = self.compute_loss(model, inputs, return_outputs=True)
                loss = loss.mean().detach()
                if isinstance(outputs, dict):
                    logits = tuple(v for k, v in outputs.items() if k not in ignore_keys + ["loss"] and v is not None)
                else:
                    logits = tuple(outputs[1:])
            else:
                loss = None
                outputs = model(**inputs)
                if isinstance(outputs, dict):
                    logits = tuple(v for k, v in outputs.items() if k not in ignore_keys and v is not None)
                else:
                    logits = tuple(outputs) if isinstance(outputs, (tuple, list)) else (outputs,)
        if prediction_loss_only:
            return loss, None, None
        logits = logits[0] if len(logits) == 1 else logits
        return loss, logits, labels

    def log_metrics(self, split: str, metrics: Dict[str, float]):
        """trainer_utils.py log_metrics: formatted dump of a metrics dict (rank 0)."""
        if self.args.process_index != 0:
            return
        print(f"***** {split} metrics *****", flush=True)
        width = max((len(str(k)) for k in metrics), default=0)
        for k in sorted(metrics):
            print(f"  {str(k):<{width}} = {metrics[k]}", flush=True)

    def save_metrics(self, split: str, metrics: Dict[str, float], combined: bool = True):
        if self.args.process_index != 0:
            return
        os.makedirs(self.args.output_dir, exist_ok=True)
        with open(os.path.join(self.args.output_dir, f"{split}_results.json"), "w") as f:
            json.dump(metrics, f, indent=4, sort_keys=True)

    def save_state(self):
        if self.args.process_index == 0:
            os.makedirs(self.args.output_dir, exist_ok=True)
            self.state.save_to_json(os.path.join(self.args.output_dir, TRAINER_STATE_NAME))

    def log(self, logs: Dict[str, float]):
        self.state.log_history.append(dict(logs))
        for cb in self.callbacks:
            cb.on_log(self.args, self.state, self.control, logs=logs)

    def save_model(self, output_dir: Optional[str] = None):
        """trainer.py:2294-2330: rank 0 writes config + safetensors shards + training args."""
        output_dir = output_dir or self.args.output_dir
        if self.args.process_index == 0:
            m = getattr(self.model, "_layers", self.model)
            m.save_pretrained(output_dir)
            with open(os.path.join(output_dir, TRAINING_ARGS_NAME), "w", encoding="utf-8") as f:
                f.write(self.args.to_json_string() + "\n")

    # ------------------------------------------------------------------------------------------------
    # checkpoint save / resume  (trainer.py:2363-2525 _save_checkpoint, :569-640 _load_from_checkpoint,
    # :2595-2680 _load_optimizer_and_scheduler, :1752-1814 _load_rng_state; unified_checkpoint.py:301-540)
    # ------------------------------------------------------------------------------------------------
    def _rng_states(self):
        dev = self._engine().device
        return {"python": random.getstate(), "numpy": __import__("numpy").random.get_state(),
                "cpu": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state(dev) if dev.type == "cuda" else None}

    def _save_checkpoint(self, model=None, metrics=None):
        from ..transformers import conversion_utils as cu

        a = self.args
        out = os.path.join(a.output_dir, f"{PREFIX_CHECKPOINT_DIR}-{self.state.global_step}")
        world = a.world_size
        if metrics is not None and a.metric_for_best_model is not None:          # trainer.py:2463-2477
            key = a.metric_for_best_model if a.metric_for_best_model.startswith("eval_") else f"eval_{a.metric_for_best_model}"
            value = metrics[key]
            better = np.greater if a.greater_is_better else np.less
            if self.state.best_metric is None or self.state.best_model_checkpoint is None or better(value, self.state.best_metric):
                self.state.best_metric = value
                self.state.best_model_checkpoint = out
        rng = self._rng_states()
        if world > 1:                                            # trainer.py:2495-2500: one list entry per rank
            rng_list = [None] * world
            torch.distributed.all_gather_object(rng_list, rng)
        if a.process_index == 0:
            tmp = out + ".tmp"
            shutil.rmtree(tmp, ignore_errors=True)
            os.makedirs(tmp)
            if self._engine().device.type == "cuda":
                torch.cuda.synchronize(self._engine().device)
            m = getattr(self.model, "_layers", self.model)
            m.save_pretrained(tmp, unified_checkpoint=True)
            if not a.save_only_model:
                cu.save_sharded(self.optimizer.named_optimizer_state(), tmp, cu.SAFE_OPTIMIZER_NAME,
                                cu.SAFE_OPTIMIZER_INDEX_NAME, always_index=True)
                cu.save_sharded(self.optimizer.named_master_weights(), tmp, cu.SAFE_MASTER_WEIGHTS_NAME,
                                cu.SAFE_MASTER_WEIGHTS_INDEX_NAME, always_index=True)
                torch.save(self.lr_scheduler.state_dict(), os.path.join(tmp, SCHEDULER_NAME))
            self.state.save_to_json(os.path.join(tmp, TRAINER_STATE_NAME))
            with open(os.path.join(tmp, TRAINING_ARGS_NAME), "w", encoding="utf-8") as f:
                f.write(a.to_json_string() + "\n")
            if world > 1:
                torch.save(rng_list, os.path.join(tmp, f"rng_state_{world}.pth"))
            else:
                torch.save(rng, os.path.join(tmp, "rng_state.pth"))
            shutil.rmtree(out, ignore_errors=True)
            os.replace(tmp, out)                                 # a crash mid-save never leaves a half checkpoint-N
            self._rotate_checkpoints()
        if world > 1:
            torch.distributed.barrier()
        return out

    def _rotate_checkpoints(self):
        """trainer.py:2549-2585: keep the newest `save_total_limit` checkpoint-N directories, and never the best one: it
        is moved to second-newest, and with a limit of 1 the newest is kept too (so that training can resume)."""
        limit = self.args.save_total_limit
        if not limit or limit <= 0:
            return
        found = []
        for name in os.listdir(self.args.output_dir):
            m = re.fullmatch(PREFIX_CHECKPOINT_DIR + r"-(\d+)", name)
            if m:
                found.append((int(m.group(1)), os.path.join(self.args.output_dir, name)))
        paths = [p for _, p in sorted(found)]
        best = self.state.best_model_checkpoint
        if best is not None and best in paths:
            i = paths.index(best)
            paths.insert(max(i, len(paths) - 2), paths.pop(i))
            if limit == 1 and paths[-1] != best:
                limit = 2
        for path in paths[:max(0, len(paths) - limit)]:
            shutil.rmtree(path, ignore_errors=True)

    def _load_from_checkpoint(self, checkpoint: str):
        from ..transformers import conversion_utils as cu

        if not os.path.isdir(checkpoint) or not cu.has_safetensors(checkpoint):
            raise ValueError(f"Can't find a valid checkpoint at {checkpoint}")
        m = getattr(self.model, "_layers", self.model)
        m._load_streaming(cu.iter_sharded(checkpoint), convert_from_hf=False)

    def _load_optimizer_and_scheduler(self, checkpoint: str):
        from ..transformers import conversion_utils as cu

        if not cu.has_safetensors(checkpoint, cu.SAFE_OPTIMIZER_NAME, cu.SAFE_OPTIMIZER_INDEX_NAME):
            # save_only_model checkpoints: fresh moments, master weights re-derived from the bf16 parameters
            self.optimizer.sync_master_from_params()
            return
        state = TrainerState.load_from_json(os.path.join(checkpoint, TRAINER_STATE_NAME))
        self.optimizer.load_named_state(
            cu.iter_sharded(checkpoint, cu.SAFE_OPTIMIZER_NAME, cu.SAFE_OPTIMIZER_INDEX_NAME),
            cu.iter_sharded(checkpoint, cu.SAFE_MASTER_WEIGHTS_NAME, cu.SAFE_MASTER_WEIGHTS_INDEX_NAME),
            step=state.global_step)
        sched = os.path.join(checkpoint, SCHEDULER_NAME)
        if os.path.isfile(sched):
            self.lr_scheduler.set_state_dict(torch.load(sched))

    def _load_rng_state(self, checkpoint: str):
        a = self.args
        world = a.world_size
        path = os.path.join(checkpoint, f"rng_state_{world}.pth" if world > 1 else "rng_state.pth")
        if not os.path.isfile(path):
            return                                               # trainer.py:1777-1783: warn-and-continue
        st = torch.load(path, weights_only=False)
        if world > 1:
            st = st[a.process_index]
        random.setstate(st["python"])
        __import__("numpy").random.set_state(st["numpy"])
        torch.set_rng_state(st["cpu"])
        dev = self._engine().device
        if st.get("cuda") is not None and dev.type == "cuda":
            torch.cuda.set_rng_state(st["cuda"], dev)
