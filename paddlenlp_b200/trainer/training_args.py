"""TrainingArguments — the data-parallel subset of paddlenlp/trainer/training_args.py (fields of SURVEY.md Appendix C).

Derived fields follow :982-1064 (world_size -> data_parallel_degree, use_hybrid_parallel False for pure DP) and
:1765-1775 (train_batch_size).  Anything requesting sharding / tensor / pipeline parallelism raises: this build
covers pure data-parallel replication only.
"""
from __future__ import annotations

import json
import os
from dataclasses import asdict, dataclass, field
from typing import Optional

from .. import distributed as dist_env
from .trainer_utils import IntervalStrategy


class _SchedulerName(str):
    """A plain string that also answers `.value` (the reference's SchedulerType enum member: run_pretrain.py:518 reads
    `training_args.lr_scheduler_type.value`)."""

    @property
    def value(self):
        return str(self)


@dataclass
class TrainingArguments:
    output_dir: str = "./output"
    do_train: bool = True
    per_device_train_batch_size: int = 8
    gradient_accumulation_steps: int = 1
    max_steps: int = -1
    num_train_epochs: float = 1.0
    learning_rate: float = 5e-5
    min_learning_rate: Optional[float] = None
    weight_decay: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_epsilon: float = 1e-8
    max_grad_norm: float = 1.0
    warmup_steps: int = 0
    warmup_ratio: float = 0.0
    decay_steps: int = 0
    lr_scheduler_type: str = "linear"
    num_cycles: float = 0.5
    logging_steps: int = 500
    logging_first_step: bool = False
    save_steps: int = 0
    save_strategy: str = "steps"                  # "no" / "steps" (every save_steps) / "epoch"
    # evaluation (training_args.py:396-420, 739-779): defaults and __post_init__ rules of the reference
    evaluation_strategy: str = "no"               # "no" / "steps" (every eval_steps) / "epoch"
    eval_steps: Optional[int] = None              # falls back to logging_steps
    per_device_eval_batch_size: int = 8
    eval_accumulation_steps: Optional[int] = None  # accepted; predictions are moved to the host after every batch
    prediction_loss_only: bool = False
    max_evaluate_steps: int = -1                  # > 0: evaluate on that many batches per process only
    load_best_model_at_end: bool = False
    metric_for_best_model: Optional[str] = None
    greater_is_better: Optional[bool] = None
    save_total_limit: Optional[int] = None
    resume_from_checkpoint: Optional[str] = None
    save_only_model: bool = False
    seed: int = 42
    bf16: bool = True
    fp16: bool = False
    fp16_opt_level: str = "O2"
    amp_master_grad: bool = False                 # fp32 gradients: accumulation, DP exchange, clipping and AdamW in fp32
    recompute: bool = False
    dataloader_num_workers: int = 0
    dataloader_drop_last: bool = True
    disable_tqdm: bool = True
    skip_profile_timer: bool = True
    skip_memory_metrics: bool = True
    ddp_find_unused_parameters: Optional[bool] = None
    ignore_data_skip: bool = False
    device: str = "gpu"
    max_seq_length: Optional[int] = None
    # fields the reference's training scripts read (llm/run_pretrain.py:358-575); inert on the pure data-parallel path
    overwrite_output_dir: bool = False
    do_eval: bool = False                         # True with evaluation_strategy "no" means "steps"
    do_predict: bool = False
    autotuner_benchmark: bool = False
    sequence_parallel: bool = False
    fuse_sequence_parallel_allreduce: bool = False
    enable_linear_fused_grad_add: bool = False
    no_recompute_layers: Optional[list] = None
    sharding_parallel_config: Optional[str] = None
    should_load_dataset: bool = True
    unified_checkpoint: bool = True
    # parallelism knobs accepted for compatibility; only the pure-DP values are implemented
    tensor_parallel_degree: int = 1
    pipeline_parallel_degree: int = 1
    sharding: str = ""
    sharding_parallel_degree: int = -1
    sep_parallel_degree: int = 1
    context_parallel_degree: int = 1
    # LlmMetaConfig switches (configuration_utils.py:230-314); all map to the single native path
    use_flash_attention: bool = True
    use_fused_rms_norm: bool = True
    use_fused_rope: bool = True

    def __post_init__(self):
        if self.fp16:
            raise NotImplementedError("fp16 + GradScaler: the hot path is bf16 (no loss scaling, trainer.py:451)")
        if self.fp16_opt_level != "O2":
            raise NotImplementedError("only AMP level O2 (bf16 parameters + fp32 master weights) is implemented")
        for name in ("tensor_parallel_degree", "pipeline_parallel_degree", "sep_parallel_degree", "context_parallel_degree"):
            if getattr(self, name) not in (1, -1):
                raise NotImplementedError(f"{name}={getattr(self, name)}: pure data parallelism only")
        if self.sharding:
            raise NotImplementedError("sharding (ZeRO) stages: pure data-parallel replication only")
        if self.device not in ("gpu", "cuda"):
            raise NotImplementedError("device must be 'gpu': there is no CPU / XPU / NPU path")
        if self.sequence_parallel or self.enable_linear_fused_grad_add:
            raise NotImplementedError("sequence_parallel / enable_linear_fused_grad_add belong to the tensor-parallel path")
        self.lr_scheduler_type = _SchedulerName(getattr(self.lr_scheduler_type, "value", self.lr_scheduler_type))
        # training_args.py:926-970
        self.evaluation_strategy = IntervalStrategy(self.evaluation_strategy)
        self.save_strategy = IntervalStrategy(self.save_strategy)
        if self.do_eval is False and self.evaluation_strategy != IntervalStrategy.NO:
            self.do_eval = True
        if self.do_eval and self.evaluation_strategy == IntervalStrategy.NO:
            self.evaluation_strategy = IntervalStrategy.STEPS
        if self.evaluation_strategy == IntervalStrategy.STEPS and not self.eval_steps:
            if self.logging_steps > 0:
                self.eval_steps = self.logging_steps
            else:
                raise ValueError(f"evaluation strategy {self.evaluation_strategy} requires either non-zero --eval_steps or "
                                 "--logging_steps")
        if self.load_best_model_at_end:
            if self.evaluation_strategy != self.save_strategy:
                raise ValueError("--load_best_model_at_end requires the save and eval strategy to match, but found\n- "
                                 f"Evaluation strategy: {self.evaluation_strategy}\n- Save strategy: {self.save_strategy}")
            if self.evaluation_strategy == IntervalStrategy.STEPS and self.save_steps % self.eval_steps != 0:
                raise ValueError("--load_best_model_at_end requires the saving steps to be a round multiple of the evaluation "
                                 f"steps, but found {self.save_steps}, which is not a round multiple of {self.eval_steps}.")
        if self.load_best_model_at_end and self.metric_for_best_model is None:
            self.metric_for_best_model = "loss"
        if self.greater_is_better is None and self.metric_for_best_model is not None:
            self.greater_is_better = self.metric_for_best_model not in ["loss", "eval_loss"]
        dist_env.init_parallel_env()

    def print_config(self, args=None, key=""):
        """training_args.py print_config: dump an arguments object (rank 0)."""
        if self.process_index != 0:
            return
        obj = self if args is None else args
        print("=" * 60 + f"\n{key or type(obj).__name__} Configuration Arguments".center(60))
        for k, v in sorted(vars(obj).items()):
            print(f"{k:30}: {v}")

    # -- derived (training_args.py:1006-1064) --
    @property
    def world_size(self) -> int:
        return dist_env.get_world_size()

    @property
    def process_index(self) -> int:
        return dist_env.get_rank()

    @property
    def local_rank(self) -> int:
        return int(os.environ.get("LOCAL_RANK", "0")) if self.world_size > 1 else -1

    @property
    def data_parallel_degree(self) -> int:
        return self.world_size

    @property
    def dataset_world_size(self) -> int:
        return self.world_size

    @property
    def dataset_rank(self) -> int:
        return self.process_index

    @property
    def use_hybrid_parallel(self) -> bool:
        return False

    @property
    def train_batch_size(self) -> int:
        return self.per_device_train_batch_size

    @property
    def eval_batch_size(self) -> int:
        return self.per_device_eval_batch_size

    @property
    def should_log(self) -> bool:
        return self.process_index == 0

    def to_dict(self):
        d = asdict(self)
        for k in ("lr_scheduler_type", "evaluation_strategy", "save_strategy"):
            d[k] = str(d[k])
        return d

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2)
