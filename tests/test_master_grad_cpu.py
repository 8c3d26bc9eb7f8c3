"""amp_master_grad host logic without a device: the fp32-gradient entry points of the C-ABI, the Trainer reaching the engine's
switch before it builds the optimizer, and the switch itself (buffer, views, refusal while gradients are pending)."""
import math
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# new entry point -> the ctypes argument types it must have (its bf16 twin's, with the gradient as an fp32 pointer)
NEW_ENTRY_POINTS = {
    "b200_gemm_bf16_f32": "P P P I64 I64 I64 I64 I64 I64 I I I P",
    "b200_rmsnorm_bwd_f32": "P P P P P P P I P I64 I64 P",
    "b200_colsum_f32": "P P I P I64 I64 I64 P",
    "b200_embedding_bwd_f32": "P P P I64 I64 I64 P",
    "b200_grad_sqnorm_f32": "P P P I64 F P",
    "b200_adamw_step_f32": "P P P P P P I64 I64 F F F F F I64 F F P",
}


def test_fp32_gradient_entry_points_declared_and_bound():
    from paddlenlp_b200 import _lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200nlp.h")).read(), flags=re.S)
    names = {"P": _lib.P, "I64": _lib.I64, "I": _lib.I, "F": _lib.F}
    for name, sig in NEW_ENTRY_POINTS.items():
        decl = re.search(rf"\bint {name}\(([^;]*)\);", src)
        assert decl is not None, f"{name} not declared in include/b200nlp.h"
        assert "float*" in decl.group(1), name                     # the gradient operand is typed fp32 in the header
        assert _lib._SIGNATURES[name] == [names[t] for t in sig.split()], name
    assert "#define B200NLP_ABI_VERSION 2" in src


class _StubEngine:
    def __init__(self):
        self.calls = []
        self.grads = {"w": torch.zeros(4, dtype=torch.bfloat16)}

    def set_master_grad(self, enable=True):
        self.calls.append(enable)
        self.grads = {"w": torch.zeros(4, dtype=torch.float32 if enable else torch.bfloat16)}

    def named_views(self, grads=False, flat=None):
        return self.grads


class _Stop(Exception):
    pass


def _stub_trainer(tmp_path, amp_master_grad):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments
    from paddlenlp_b200.transformers.model_utils import PretrainedModel

    model = PretrainedModel(types.SimpleNamespace(seq_length=8))
    model.engine = _StubEngine()
    model._named = {"w": torch.nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))}
    model._named["w"].grad = model.engine.grads["w"]
    data = [{"input_ids": torch.zeros(8, dtype=torch.int64), "labels": torch.zeros(8, dtype=torch.int64)}] * 4
    args = TrainingArguments(output_dir=str(tmp_path), per_device_train_batch_size=1, gradient_accumulation_steps=4, max_steps=1,
                             amp_master_grad=amp_master_grad)
    trainer = Trainer(model=model, args=args, train_dataset=data)

    def stop(*_a, **_k):
        raise _Stop()                                        # the optimizer would be built here: the switch must precede it

    trainer.create_optimizer_and_scheduler = stop
    return trainer, model


@pytest.mark.parametrize("flag", [True, False])
def test_trainer_switches_engine_before_the_optimizer(tmp_path, flag):
    trainer, model = _stub_trainer(tmp_path, flag)
    with pytest.raises(_Stop):
        trainer.train()
    assert model.engine.calls == ([True] if flag else [])
    assert trainer.optimizer is None
    p = model._named["w"]
    if flag:                                                  # the reference's convention: fp32 main_grad, no .grad
        assert p.grad is None and p.main_grad.dtype == torch.float32
    else:
        assert p.grad is not None and p.grad.dtype == torch.bfloat16 and not hasattr(p, "main_grad")


def _bare_engine():
    """A DecoderEngine's gradient-buffer state without a device (the constructor needs CUDA)."""
    from paddlenlp_b200.transformers.decoder_engine import BF16, DecoderEngine

    eng = object.__new__(DecoderEngine)
    eng._offsets = {"a": (0, (2, 4)), "b": (8, (3,))}
    eng.numel = 16
    eng.device = torch.device("cpu")
    eng.flat_grads = torch.zeros(eng.numel, dtype=BF16)
    eng.g = {n: eng.flat_grads[o:o + math.prod(s)].view(s) for n, (o, s) in eng._offsets.items()}
    eng.grads_fresh = True
    eng._saved = None
    return eng


def test_switch_reallocates_the_gradient_buffer_and_refuses_pending_gradients():
    eng = _bare_engine()
    eng.grads_fresh = False                                   # a backward's gradients wait for an optimizer step
    with pytest.raises(RuntimeError, match="pending"):
        eng.set_master_grad(True)
    assert eng.flat_grads.dtype == torch.bfloat16 and not eng.master_grad
    eng.grads_fresh = True
    eng._saved = {}                                           # a forward waits for its backward
    with pytest.raises(RuntimeError, match="pending"):
        eng.set_master_grad(True)
    eng._saved = None
    eng.set_master_grad(True)
    assert eng.master_grad and eng.flat_grads.dtype == torch.float32 and eng.flat_grads.numel() == 16
    for name, (off, shape) in eng._offsets.items():             # views alias the new buffer at the same element offsets
        v = eng.g[name]
        assert v.dtype == torch.float32 and tuple(v.shape) == shape
        assert v.data_ptr() == eng.flat_grads.data_ptr() + 4 * off
    buf = eng.flat_grads
    eng.set_master_grad(True)                                 # already fp32: nothing to do, even with gradients pending
    assert eng.flat_grads is buf
    eng.set_master_grad(False)
    assert eng.flat_grads.dtype == torch.bfloat16 and eng.g["b"].dtype == torch.bfloat16
