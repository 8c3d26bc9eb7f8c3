"""paddlenlp.trainer surface kept by this build: Trainer, TrainingArguments, PdArgumentParser, TrainOutput, get_last_checkpoint,
set_seed, speed_metrics, and the evaluation types EvalPrediction / IntervalStrategy (the names llm/run_pretrain.py:28-35 and
llm/run_finetune.py import)."""
from .argparser import PdArgumentParser
from .trainer import (IterableDatasetShard, PrinterCallback, TrainOutput, Trainer, TrainerCallback, TrainerState, get_last_checkpoint,
                      set_seed, speed_metrics)
from .trainer_utils import EvalLoopOutput, EvalPrediction, IntervalStrategy, PredictionOutput
from .training_args import TrainingArguments
