"""Trainer evaluation without a GPU: the evaluation arguments and their reference rules, the eval sampler, and the
evaluation_loop aggregation (stubbed prediction_step) on one process and on two gloo processes, against the reference
formula computed by hand: each batch's loss counts once per sample, the samples the sampler repeats to even out the ranks
are truncated away, and eval_loss is the mean."""
import os
import socket

import numpy as np
import pytest
import torch

from paddlenlp_b200.trainer import EvalPrediction, IntervalStrategy, PdArgumentParser, Trainer, TrainingArguments
from paddlenlp_b200.utils.llm_utils import compute_metrics


# ---- TrainingArguments (reference training_args.py:926-970) ----
def test_do_eval_and_evaluation_strategy_imply_each_other():
    a = TrainingArguments(do_eval=True, logging_steps=7)
    assert a.evaluation_strategy == IntervalStrategy.STEPS == "steps" and a.eval_steps == 7
    b = TrainingArguments(evaluation_strategy="epoch")
    assert b.do_eval and b.evaluation_strategy == "epoch" and b.eval_steps is None
    c = TrainingArguments()
    assert not c.do_eval and c.evaluation_strategy == "no"
    assert TrainingArguments(evaluation_strategy="steps", eval_steps=3, logging_steps=7).eval_steps == 3
    with pytest.raises(ValueError, match="eval_steps"):
        TrainingArguments(evaluation_strategy="steps", logging_steps=0)
    with pytest.raises(ValueError):
        TrainingArguments(evaluation_strategy="sometimes")


def test_eval_defaults_and_batch_size():
    a = TrainingArguments()
    assert (a.per_device_eval_batch_size, a.eval_batch_size, a.max_evaluate_steps) == (8, 8, -1)
    assert a.eval_accumulation_steps is None and a.prediction_loss_only is False
    assert a.load_best_model_at_end is False and a.metric_for_best_model is None and a.greater_is_better is None
    assert TrainingArguments(per_device_eval_batch_size=3).eval_batch_size == 3
    assert TrainingArguments(save_strategy="no").save_strategy == IntervalStrategy.NO


def test_load_best_model_at_end_rules():
    with pytest.raises(ValueError, match="save and eval strategy to match"):
        TrainingArguments(load_best_model_at_end=True, evaluation_strategy="epoch", save_strategy="steps")
    with pytest.raises(ValueError, match="round multiple"):
        TrainingArguments(load_best_model_at_end=True, evaluation_strategy="steps", eval_steps=4, save_steps=6)
    a = TrainingArguments(load_best_model_at_end=True, evaluation_strategy="steps", eval_steps=3, save_steps=6)
    assert a.metric_for_best_model == "loss" and a.greater_is_better is False
    assert TrainingArguments(metric_for_best_model="accuracy").greater_is_better is True
    assert TrainingArguments(metric_for_best_model="eval_loss").greater_is_better is False
    assert TrainingArguments(metric_for_best_model="accuracy", greater_is_better=False).greater_is_better is False


def test_sft_config_eval_and_save_keys_survive_parse_dict():
    """The evaluation and save keys of the reference's llm/config/llama/sft_argument.json."""
    cfg = {"output_dir": "./checkpoints/llama_sft_ckpts", "per_device_train_batch_size": 1, "gradient_accumulation_steps": 2,
           "per_device_eval_batch_size": 8, "eval_accumulation_steps": 16, "num_train_epochs": 1, "learning_rate": 3e-05,
           "warmup_steps": 30, "logging_steps": 1, "evaluation_strategy": "epoch", "save_strategy": "epoch", "bf16": True,
           "do_train": True, "do_eval": True, "load_best_model_at_end": True, "metric_for_best_model": "accuracy",
           "save_total_limit": 1}
    (a,) = PdArgumentParser(TrainingArguments).parse_dict(cfg)
    assert a.evaluation_strategy == "epoch" and a.save_strategy == "epoch" and a.do_eval
    assert (a.per_device_eval_batch_size, a.eval_accumulation_steps, a.save_total_limit) == (8, 16, 1)
    assert a.load_best_model_at_end and a.metric_for_best_model == "accuracy" and a.greater_is_better is True
    d = a.to_dict()
    assert d["evaluation_strategy"] == "epoch" and type(d["evaluation_strategy"]) is str


# ---- evaluation_loop with a stubbed prediction_step ----
class _Stub(torch.nn.Module):
    pass


class _Samples(torch.utils.data.Dataset):
    """Sample i: input_ids = [i] * (2 + i % 3) padded to 4 with -100 labels beyond; labels = i on the real positions."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        ln = 2 + i % 3
        lab = torch.full((4,), -100, dtype=torch.int64)
        lab[:ln] = i
        return {"input_ids": torch.full((4,), i, dtype=torch.int64), "labels": lab}


def _loss_of(idx):
    return 0.25 * float(sum(idx)) + 1.0


class _StubTrainer(Trainer):
    """prediction_step without a model: the batch loss is a function of the sample indices, the predictions are the
    sample index at every position."""

    def prediction_step(self, model, inputs, prediction_loss_only, ignore_keys=None):
        assert not model.training
        idx = inputs["input_ids"][:, 0].tolist()
        loss = torch.tensor(_loss_of(idx))
        if prediction_loss_only:
            return loss, None, None
        return loss, inputs["input_ids"][:, :, None], inputs["labels"]


def _expected(n, bs, world, iters=-1):
    """The reference formula by hand: global batch g holds rank r's slice [r*bs, (r+1)*bs) of the padded index list."""
    order = list(range(n))
    per = -(-n // world)
    order += order[:per * world - n]
    glob = bs * world
    losses, preds = [], []
    steps = -(-len(order) // glob) if iters <= 0 else iters
    for g in range(steps):
        chunk = order[g * glob:(g + 1) * glob]
        k = len(chunk) // world if len(chunk) < glob else bs
        for r in range(world):
            b = chunk[r * k:(r + 1) * k]
            losses += [_loss_of(b)] * len(b)
            preds += b
    num = n if iters <= 0 else bs * world * iters
    return float(np.mean(losses[:num])), preds[:num], num


def _trainer(tmp, n, bs, **kw):
    args = TrainingArguments(output_dir=str(tmp), per_device_eval_batch_size=bs, **kw)
    return _StubTrainer(model=_Stub(), args=args, eval_dataset=_Samples(n), compute_metrics=compute_metrics)


def test_eval_sampler_is_sequential_and_keeps_the_last_batch(tmp_path):
    t = _trainer(tmp_path, 7, 2)
    assert [b["input_ids"][:, 0].tolist() for b in t.get_eval_dataloader()] == [[0, 1], [2, 3], [4, 5], [6]]


def test_evaluation_loop_uneven_last_batch(tmp_path):
    t = _trainer(tmp_path, 7, 2)
    out = t.evaluation_loop(t.get_eval_dataloader(), "Evaluation", metric_key_prefix="eval")
    want, preds, num = _expected(7, 2, 1)
    assert out.num_samples == num == 7
    assert out.metrics["eval_loss"] == pytest.approx(want, rel=1e-12)
    assert out.predictions[:, 0, 0].tolist() == preds
    assert out.metrics["eval_accuracy"] == 1.0 and t.model.training
    m = t.evaluate()
    assert m["eval_loss"] == pytest.approx(want, rel=1e-12) and "eval_runtime" in m and "eval_samples_per_second" in m
    assert t.state.log_history[-1]["eval_loss"] == m["eval_loss"]
    p = t.predict(_Samples(5))
    assert p.metrics["test_loss"] == pytest.approx(_expected(5, 2, 1)[0], rel=1e-12) and p.predictions.shape == (5, 4, 1)


def test_evaluation_loop_max_eval_iters(tmp_path):
    t = _trainer(tmp_path, 7, 2, max_evaluate_steps=2)
    m = t.evaluate()
    want, _, num = _expected(7, 2, 1, iters=2)
    assert num == 4 and m["eval_loss"] == pytest.approx(want, rel=1e-12)


def test_loss_only_evaluation_without_compute_metrics(tmp_path):
    args = TrainingArguments(output_dir=str(tmp_path), per_device_eval_batch_size=3)
    t = _StubTrainer(model=_Stub(), args=args, eval_dataset=_Samples(7))
    m = t.evaluate()
    assert m["eval_loss"] == pytest.approx(_expected(7, 3, 1)[0], rel=1e-12) and "eval_accuracy" not in m


def test_compute_metrics_token_accuracy():
    preds = np.array([[[3], [5], [7], [1]], [[2], [2], [9], [0]]])
    labels = np.array([[3, 4, 7, -100], [-100, 2, 8, 0]])
    # kept positions: (3,3) (5,4) (7,7) | (2,2) (9,8) (0,0): 4 of 6 equal
    assert compute_metrics(EvalPrediction(predictions=preds, label_ids=labels))["accuracy"] == pytest.approx(4 / 6)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, tmp, n, bs, iters, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank))
    torch.distributed.init_process_group("gloo", rank=rank, world_size=world)
    try:
        t = _trainer(tmp, n, bs, max_evaluate_steps=iters)
        batches = [b["input_ids"][:, 0].tolist() for b in t.get_eval_dataloader()]
        m = t.evaluate()
        out = t.evaluation_loop(t.get_eval_dataloader(), "Evaluation", max_eval_iters=iters)
        q.put((rank, batches, m["eval_loss"], out.predictions[:, 0, 0].tolist(), out.label_ids.shape, out.num_samples))
    finally:
        torch.distributed.destroy_process_group()


@pytest.mark.parametrize("n,bs,iters", [(7, 2, -1), (9, 2, -1), (7, 2, 1)])
def test_evaluation_loop_two_ranks_over_gloo(tmp_path, n, bs, iters):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path), n, bs, iters, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want, preds, num = _expected(n, bs, 2, iters)
    order = list(range(n)) + list(range(n))[: -(-n // 2) * 2 - n]
    for rank, batches, loss, got_preds, label_shape, got_num in res:
        assert batches[0] == order[rank * bs:(rank + 1) * bs]               # rank r takes slice r of each global batch
        assert sum(len(b) for b in batches) == -(-n // 2)
        assert loss == pytest.approx(want, rel=1e-12)                       # the same eval_loss on both ranks
        assert got_preds == preds and got_num == num and label_shape[0] == num
