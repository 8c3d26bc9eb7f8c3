"""paddlenlp/utils/llm_utils.py: the token-accuracy `compute_metrics` and `CausalLMTrainer` that llm/run_finetune.py imports."""
from __future__ import annotations

from typing import Dict

import numpy as np

from ..trainer import Trainer


def compute_metrics(eval_preds) -> Dict[str, float]:
    """Token accuracy over the positions whose label is not -100 (llm_utils.py:46-54)."""
    preds = np.asarray(eval_preds.predictions).reshape(-1)
    labels = np.asarray(eval_preds.label_ids).reshape(-1)
    keep = labels != -100
    return {"accuracy": float(np.mean(preds[keep] == labels[keep])) if keep.any() else 0.0}


class CausalLMTrainer(Trainer):
    """Trainer whose predictions are the arg-max token of each position ([B, S, 1]) rather than the [B, S, V] logits
    (llm_utils.py:262-292: "argmax here to avoid gather all logits").  With the built-in criterion the loss and the
    arg-max come from the engine's chunked evaluation forward, so the logits never exist in full."""

    def __init__(self, do_generation: bool, gen_args, data_args, **kwargs):
        super().__init__(**kwargs)
        if do_generation:
            raise NotImplementedError("CausalLMTrainer(do_generation=True): evaluation by generation is not implemented")
        self.do_generation = do_generation
        self.gen_args = gen_args
        self.data_args = data_args

    def prediction_step(self, model, inputs, prediction_loss_only: bool, ignore_keys=None):
        if prediction_loss_only or inputs.get("labels") is None:
            return super().prediction_step(model, inputs, prediction_loss_only, ignore_keys)
        ign = self._fused_eval_ignore_index()
        if ign is None:                                          # a custom criterion: arg-max of its logits
            from .. import ops

            loss, logits, labels = super().prediction_step(model, inputs, prediction_loss_only, ignore_keys)
            if isinstance(logits, (list, tuple)):
                logits = logits[0]
            preds = ops.argmax(logits.reshape(-1, logits.shape[-1]).contiguous()).view(*logits.shape[:-1], 1)
            return loss, preds, labels
        inputs = self._prepare_inputs(inputs)
        loss_out, preds = self._forward_eval(inputs, ign, predictions=True)
        return loss_out[0], preds[..., None], inputs["labels"]

    def log(self, logs: Dict[str, float], **kwargs) -> None:
        if "loss" in logs:
            logs["ppl"] = np.exp(logs["loss"])
        if "eval_loss" in logs:
            logs["eval_ppl"] = np.exp(logs["eval_loss"])
        super().log(logs, **kwargs)
