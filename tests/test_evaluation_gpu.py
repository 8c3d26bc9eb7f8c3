"""Evaluation on the GPU: the fused cross-entropy + arg-max row pass against ce_fwd and argmax bit for bit, the engine's
chunked forward_eval against forward_loss + argmax bit for bit and in peak memory, and Trainer.evaluate / predict /
evaluation during training / load_best_model_at_end / CausalLMTrainer on tiny models."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import llama_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


# ---- row pass ----
@pytest.mark.parametrize("V", [512, 32001, 128256, 151936])
def test_row_pass_matches_ce_fwd_and_argmax_bit_for_bit(V):
    from paddlenlp_b200 import ops

    T = 512 if V < 100000 else 192
    ld = (V + 7) // 8 * 8
    g = torch.Generator(device=DEV).manual_seed(V)
    full = (torch.randn(T, ld, generator=g, device=DEV) * 4).to(torch.bfloat16)
    logits = full[:, :V]
    # planted ties: the row maximum at two or more columns (the lower index must win), a constant row, an all -inf row
    # and a row with a NaN; bf16 rows of 128 k values also tie by themselves
    for r in range(0, 32, 4):
        a, b = sorted(torch.randint(0, V, (2,), generator=g, device=DEV).tolist())
        logits[r, a] = logits[r, b] = 60.0
        logits[r + 1, V - 1] = logits[r + 1, V // 2] = logits[r + 1, 3] = 60.0
    logits[33] = 1.5
    logits[34] = -float("inf")
    logits[35, V // 3] = float("nan")
    labels = torch.randint(0, V, (T,), generator=g, device=DEV)
    labels[::7] = -100
    labels[5::11] = V + 3                                        # out of range: loss 0, like ignore_index
    labels[6::13] = -5
    loss_out, loss_tok, _ = ops.ce_fwd(logits, labels)
    want_pred = ops.argmax(logits)
    row0 = logits[0].float()
    assert int(want_pred[0]) == int((row0 == row0.max()).nonzero()[0, 0])      # the lower index of the planted tie

    lt = torch.full((T,), 7.0, device=DEV)
    pred = torch.full((T,), -1, dtype=torch.int64, device=DEV)
    for lo, hi in ((0, 128), (128, T - 37), (T - 37, T)):       # the row range of each call is a chunk of the matrix
        ops.ce_rows_fwd(logits[lo:hi], labels, lt, pred, lo)
    assert torch.equal(_bits(lt), _bits(loss_tok))
    assert torch.equal(pred, want_pred)
    assert torch.equal(_bits(ops.ce_reduce(lt)), _bits(loss_out))

    lt2 = torch.full((T,), 7.0, device=DEV)
    ops.ce_rows_fwd(logits, labels, lt2, None, 0)               # loss only
    assert torch.equal(_bits(lt2), _bits(loss_tok))


# ---- engine ----
def _cfg_model(kind, V=1000):
    import paddlenlp_b200.transformers as T

    kw = dict(vocab_size=V, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
              num_key_value_heads=1, max_position_embeddings=512, seq_length=256, rope_theta=500000.0, rms_norm_eps=1e-5)
    if kind == "qwen2":
        m = T.Qwen2ForCausalLM(T.Qwen2Config(**kw))
    else:
        m = T.LlamaForCausalLM(T.LlamaConfig(tie_word_embeddings=(kind == "tied"), **kw))
    with torch.no_grad():                                        # larger than the 0.02 init, so that logits are not flat
        m.engine.flat_params.mul_(4)
        if m.engine.qkv_bias:
            for i in range(m.engine.L):
                m.engine.p[f"l{i}.qkv_b"].normal_(0, 0.5)
        m.engine.params_changed()
    return m


def _packed_rows(B, S, cuts):
    """FlashMask start rows of packed documents ending at `cuts` (and S): every column -> end of its document."""
    ms = torch.empty(B, S, dtype=torch.int32)
    lo = 0
    for hi in list(cuts) + [S]:
        ms[:, lo:hi] = hi
        lo = hi
    return ms


@pytest.mark.parametrize("kind,S,flashmask,positions", [
    ("llama", 200, False, False),        # T = 400: three 128-row chunks, a 16-row tail folded into the third
    ("qwen2", 225, False, True),         # T = 450: a 66-row tail stays a chunk of its own
    ("tied", 200, False, False),
    ("llama", 225, True, False),
])
def test_forward_eval_is_forward_loss_and_argmax(kind, S, flashmask, positions, monkeypatch):
    from paddlenlp_b200 import ops
    from paddlenlp_b200.transformers import decoder_engine

    m = _cfg_model(kind)
    eng = m.engine
    B, V = 2, eng.V
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(0, V, (B, S), generator=g)
    labels = torch.randint(0, V, (B, S), generator=g)
    labels[:, :30] = -100
    pos = torch.arange(S).repeat(B, 1) + 7 if positions else None
    ms = _packed_rows(B, S, (60, 130)) if flashmask else None
    want_out, logits = eng.forward_loss(ids, labels, pos, keep_for_backward=False, attn_mask_startend_row_indices=ms)
    want_pred = ops.argmax(logits.view(-1, V)).view(B, S)
    monkeypatch.setattr(decoder_engine, "EVAL_LOGITS_CHUNK_BYTES", 128 * V * 2)
    chunks = eng._eval_chunks(B * S)
    assert len(chunks) == 3 + (S == 225) and all((hi - lo) > 64 for lo, hi in chunks)
    for pred in (True, False):
        out, preds = eng.forward_eval(ids, labels, pos, attn_mask_startend_row_indices=ms, predictions=pred)
        assert torch.equal(_bits(out), _bits(want_out)), (out.tolist(), want_out.tolist())
        if pred:
            assert preds.shape == (B, S) and torch.equal(preds, want_pred)
        else:
            assert preds is None


def test_forward_eval_peak_memory_saves_the_logits():
    """V = 128 256, T = 8192: forward_loss holds the whole [T, V] bf16 logits, forward_eval one chunk of rows."""
    from paddlenlp_b200.transformers import decoder_engine

    m = _cfg_model("llama", V=128256)
    eng = m.engine
    B, S, V = 2, 4096, eng.V
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, V, (B, S), generator=g).to(DEV)
    labels = torch.randint(0, V, (B, S), generator=g).to(DEV)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del out
        return p

    p_loss = peak(lambda: eng.forward_loss(ids, labels, keep_for_backward=False))
    p_eval = peak(lambda: eng.forward_eval(ids, labels))
    T = B * S
    rows = max(hi - lo for lo, hi in eng._eval_chunks(T))
    saving = (T - rows) * V * 2
    assert rows < T and rows * V * 2 <= decoder_engine.EVAL_LOGITS_CHUNK_BYTES
    print(f"peak forward_loss {p_loss / 2**30:.3f} GiB, forward_eval {p_eval / 2**30:.3f} GiB, "
          f"expected saving {saving / 2**30:.3f} GiB")
    assert p_loss - p_eval >= saving - (32 << 20)


# ---- Trainer ----
class _Data(torch.utils.data.Dataset):
    def __init__(self, n, S, V, sft=False, seed=1234):
        g = torch.Generator().manual_seed(seed)
        self.tok = torch.randint(1, V, (n, S + 1), generator=g)
        self.sft = sft

    def __len__(self):
        return self.tok.shape[0]

    def __getitem__(self, i):
        ids, labels = self.tok[i, :-1].clone(), self.tok[i, 1:].clone()
        if self.sft:                                  # prompt tokens carry label -100
            labels[: 40 + 5 * i] = -100
        return {"input_ids": ids, "labels": labels}


def _tiny(kind="llama"):
    import paddlenlp_b200.transformers as T

    kw = dict(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
              num_key_value_heads=1, max_position_embeddings=256, seq_length=128, rope_theta=500000.0, rms_norm_eps=1e-5)
    return T.Qwen2ForCausalLM(T.Qwen2Config(**kw)) if kind == "qwen2" else T.LlamaForCausalLM(T.LlamaConfig(**kw))


def _by_formula(batch_losses, batch_sizes, n):
    per_sample = np.concatenate([np.full(b, float(l), dtype=np.float64) for l, b in zip(batch_losses, batch_sizes)])
    return float(per_sample[:n].mean())


@pytest.mark.parametrize("kind,sft", [("llama", False), ("qwen2", True)])
def test_evaluate_matches_forward_loss_by_the_reference_formula(kind, sft, tmp_path):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    m = _tiny(kind)
    ds = _Data(7, 128, 512, sft)
    args = TrainingArguments(output_dir=str(tmp_path), per_device_eval_batch_size=2)
    t = Trainer(model=m, args=args, eval_dataset=ds)
    metrics = t.evaluate()
    losses, sizes = [], []
    for lo in range(0, 7, 2):
        b = [ds[i] for i in range(lo, min(7, lo + 2))]
        ids = torch.stack([x["input_ids"] for x in b])
        lab = torch.stack([x["labels"] for x in b])
        losses.append(m.engine.forward_loss(ids, lab, keep_for_backward=False)[0][0].item())
        sizes.append(len(b))
    assert metrics["eval_loss"] == pytest.approx(_by_formula(losses, sizes, 7), rel=1e-12)
    assert t.state.log_history[-1]["eval_loss"] == metrics["eval_loss"] and m.training

    p = t.predict(ds)
    assert p.metrics["test_loss"] == pytest.approx(metrics["eval_loss"], rel=1e-12) and p.predictions is None


def _train(tmp, evaluate, callback=None):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    m = _tiny()
    extra = dict(evaluation_strategy="steps", eval_steps=2) if evaluate else {}
    args = TrainingArguments(output_dir=str(tmp), per_device_train_batch_size=2, per_device_eval_batch_size=2, max_steps=8,
                             learning_rate=2e-3, warmup_steps=1, logging_steps=1, max_seq_length=128, **extra)
    t = Trainer(model=m, args=args, train_dataset=_Data(8, 128, 512), eval_dataset=_Data(5, 128, 512, seed=9))
    if callback is not None:
        t.callbacks.append(callback(t))
    t.train()
    return t


def test_evaluation_during_training_does_not_change_training(tmp_path):
    """Every evaluation leaves the training state (bf16 weights, fp32 master weights, both moments, optimizer step, host and
    device RNG) bit for bit as it found it.  Two training runs agree bit for bit only up to their first backward (the
    attention backward's fp32 reduce-adds have no fixed order), so the loss histories are compared to the accumulation noise
    the checkpoint-resume test allows."""
    from paddlenlp_b200.trainer import TrainerCallback

    changed = []

    def check(t):
        def state():
            o = t.optimizer
            return [t.model.engine.flat_params.clone(), o.master.clone(), o.exp_avg.clone(), o.exp_avg_sq.clone(),
                    torch.tensor(o.step_count), torch.get_rng_state(), torch.cuda.get_rng_state()]

        class Check(TrainerCallback):
            def on_step_end(self, args, st, control, **kw):
                self.before = state()

            def on_evaluate(self, args, st, control, metrics=None, **kw):
                changed.append([i for i, (a, b) in enumerate(zip(self.before, state())) if not torch.equal(a, b)])

        return Check()

    t0 = _train(tmp_path / "a", False)
    t1 = _train(tmp_path / "b", True, check)
    assert changed == [[], [], [], []]
    l0 = [h["loss"] for h in t0.state.log_history if "loss" in h]
    l1 = [h["loss"] for h in t1.state.log_history if "loss" in h]
    assert len(l0) == len(l1) == 8 and l0[0] == l1[0]
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 2e-3
    ev = [h for h in t1.state.log_history if "eval_loss" in h]
    assert [h["global_step"] for h in ev] == [2, 4, 6, 8]
    assert t1.evaluate()["eval_loss"] == ev[-1]["eval_loss"]         # the last evaluation saw the final weights


def test_evaluation_strategy_without_eval_dataset_raises_before_training(tmp_path):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    m = _tiny()
    args = TrainingArguments(output_dir=str(tmp_path), per_device_train_batch_size=2, max_steps=2, do_eval=True, logging_steps=1)
    t = Trainer(model=m, args=args, train_dataset=_Data(8, 128, 512))
    with pytest.raises(ValueError, match="eval_dataset"):
        t.train()
    assert t.state.global_step == 0


def test_epoch_strategies(tmp_path):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    m = _tiny()
    args = TrainingArguments(output_dir=str(tmp_path), per_device_train_batch_size=2, per_device_eval_batch_size=2,
                             num_train_epochs=2, learning_rate=2e-3, logging_steps=1, evaluation_strategy="epoch",
                             save_strategy="epoch")
    t = Trainer(model=m, args=args, train_dataset=_Data(8, 128, 512), eval_dataset=_Data(3, 128, 512, seed=9))
    t.train()
    assert [h["global_step"] for h in t.state.log_history if "eval_loss" in h] == [4, 8]
    assert sorted(d for d in os.listdir(tmp_path) if d.startswith("checkpoint-")) == ["checkpoint-4", "checkpoint-8"]


def test_load_best_model_at_end_keeps_and_loads_the_best_checkpoint(tmp_path):
    from paddlenlp_b200.trainer import Trainer, TrainerCallback, TrainingArguments

    m = _tiny()
    at_step = {}

    class Snap(TrainerCallback):
        def on_step_end(self, args, state, control, **kw):
            at_step[state.global_step] = m.engine.flat_params.clone()

    holder = {}

    def planted(p):                                              # the planted best: the evaluation after step 4
        assert p.predictions.shape[:2] == p.label_ids.shape
        return {"planted": 1.0 if holder["t"].state.global_step == 4 else 0.0}

    args = TrainingArguments(output_dir=str(tmp_path), per_device_train_batch_size=2, per_device_eval_batch_size=2, max_steps=8,
                             learning_rate=2e-3, logging_steps=1, evaluation_strategy="steps", eval_steps=2, save_steps=2,
                             save_total_limit=1, load_best_model_at_end=True, metric_for_best_model="planted")
    t = Trainer(model=m, args=args, train_dataset=_Data(8, 128, 512), eval_dataset=_Data(3, 128, 512, seed=9),
                compute_metrics=planted, callbacks=[Snap()])
    holder["t"] = t
    t.train()
    assert t.state.best_model_checkpoint == os.path.join(str(tmp_path), "checkpoint-4") and t.state.best_metric == 1.0
    assert sorted(d for d in os.listdir(tmp_path) if d.startswith("checkpoint-")) == ["checkpoint-4", "checkpoint-8"]
    assert not torch.equal(at_step[8], at_step[4])
    assert torch.equal(m.engine.flat_params, at_step[4])


def test_causal_lm_trainer_reports_accuracy_and_ppl(tmp_path):
    from paddlenlp_b200 import ops
    from paddlenlp_b200.trainer import Trainer, TrainingArguments
    from paddlenlp_b200.utils.llm_utils import CausalLMTrainer, compute_metrics

    m = _tiny("qwen2")
    ds = _Data(5, 128, 512, sft=True)
    args = TrainingArguments(output_dir=str(tmp_path), per_device_eval_batch_size=2)
    t = CausalLMTrainer(do_generation=False, gen_args=None, data_args=None, model=m, args=args, eval_dataset=ds,
                        compute_metrics=compute_metrics)
    metrics = t.evaluate()
    hit = tot = 0
    for lo in range(0, 5, 2):
        b = [ds[i] for i in range(lo, min(5, lo + 2))]
        ids = torch.stack([x["input_ids"] for x in b])
        lab = torch.stack([x["labels"] for x in b]).view(-1)
        _, logits = m.engine.forward_loss(ids, lab, keep_for_backward=False)
        pred = ops.argmax(logits.view(-1, 512)).cpu()
        keep = lab != -100
        hit += int((pred[keep] == lab[keep]).sum())
        tot += int(keep.sum())
    assert metrics["eval_accuracy"] == pytest.approx(hit / tot, abs=1e-12)
    assert metrics["eval_ppl"] == pytest.approx(math.exp(metrics["eval_loss"]), rel=1e-9)
    base = Trainer(model=m, args=args, eval_dataset=ds).evaluate()
    assert metrics["eval_loss"] == pytest.approx(base["eval_loss"], rel=1e-12)
    with pytest.raises(NotImplementedError):
        CausalLMTrainer(do_generation=True, gen_args=None, data_args=None, model=m, args=args)


def test_eval_loss_against_the_oracle(tmp_path):
    """The tiny model's eval_loss against the oracle's bf16 forward + criterion, by the reference formula (1e-3 relative)."""
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    cfg = R.RefConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=1, max_position_embeddings=256, rope_theta=500000.0)
    w = R.init_weights(cfg, seed=21)
    w = {k: (v * 3).to(torch.bfloat16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    m = _tiny()
    m.set_state_dict(w)
    ds = _Data(7, 128, 512, sft=True)
    t = Trainer(model=m, args=TrainingArguments(output_dir=str(tmp_path), per_device_eval_batch_size=2), eval_dataset=ds)
    got = t.evaluate()["eval_loss"]
    losses, sizes = [], []
    for lo in range(0, 7, 2):
        b = [ds[i] for i in range(lo, min(7, lo + 2))]
        ids = torch.stack([x["input_ids"] for x in b])
        lab = torch.stack([x["labels"] for x in b])
        losses.append(float(R.criterion(R.model_forward(ids, w, cfg, "bf16"), lab)))
        sizes.append(len(b))
    want = _by_formula(losses, sizes, 7)
    print(f"eval_loss {got:.6f} oracle {want:.6f}")
    assert abs(got - want) <= 1e-3 * abs(want)
