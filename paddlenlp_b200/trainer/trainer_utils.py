"""Evaluation types of paddlenlp/trainer/trainer_utils.py: IntervalStrategy, EvalPrediction, EvalLoopOutput, PredictionOutput."""
from __future__ import annotations

from enum import Enum
from typing import Dict, NamedTuple, Optional, Tuple, Union

import numpy as np


class IntervalStrategy(str, Enum):
    """When the Trainer evaluates or saves: never, every `eval_steps` / `save_steps` optimizer steps, or at each epoch end.
    A member compares equal to its string value."""

    NO = "no"
    STEPS = "steps"
    EPOCH = "epoch"

    def __str__(self):
        return self.value


class EvalPrediction(NamedTuple):
    """What `compute_metrics` receives: the gathered predictions and labels of the whole evaluation set."""

    predictions: Union[np.ndarray, Tuple[np.ndarray]]
    label_ids: Union[np.ndarray, Tuple[np.ndarray]]


class EvalLoopOutput(NamedTuple):
    predictions: Union[np.ndarray, Tuple[np.ndarray]]
    label_ids: Optional[Union[np.ndarray, Tuple[np.ndarray]]]
    metrics: Optional[Dict[str, float]]
    num_samples: Optional[int]


class PredictionOutput(NamedTuple):
    predictions: Union[np.ndarray, Tuple[np.ndarray]]
    label_ids: Optional[Union[np.ndarray, Tuple[np.ndarray]]]
    metrics: Optional[Dict[str, float]]
