"""amp_master_grad on the GPU: the fp32-output weight-gradient GEMM, the engine's fp32 gradients over one and four micro-batches,
clip + AdamW on fp32 gradients, and the Trainer with amp_master_grad=True (losses, main_grad, checkpoint resume).

The attention backward adds dQ / dK / dV with fp32 reduce-adds in no fixed order, so two backward passes agree bit for bit only
above the first attention they meet.  The engine tests therefore check each weight-gradient GEMM on the operands it was given
in that very backward, and compare whole-model gradients of separate passes with tolerances."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BF16 = torch.bfloat16
F32 = torch.float32


def _ops():
    from paddlenlp_b200 import ops

    return ops


def _rand(*shape, scale=0.5, seed=0, dtype=BF16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def _mat(rows, cols, seed):
    """bf16 [rows, cols] view with the leading dimension padded to a multiple of 8 elements."""
    return _rand(rows, -(-cols // 8) * 8, seed=seed)[:, :cols]


def _acc(a, b, trans_a, trans_b):
    """The GEMM kernel's own fp32 accumulators (split-K GEMM with one split into a zeroed buffer: exact)."""
    from paddlenlp_b200 import _lib

    K, M = a.shape if trans_a else a.shape[::-1]
    N = b.shape[0] if trans_b else b.shape[1]
    ws = torch.zeros(M, N, dtype=F32, device=DEV)
    _lib.call("b200_gemm_bf16_splitk", _lib.ptr(a), _lib.ptr(b), None, None, _lib.ptr(ws), M, N, K, a.stride(0), b.stride(0),
              N, 1 if trans_a else 0, 0 if trans_b else 1, 1, _lib.stream_ptr())
    return ws


# (M, N, K, trans_a, trans_b): trans_a + MN-major B is the dW form (X^T dY, also the tied head's dlogits^T hf)
GEMM_SHAPES = [
    (48, 200, 256, True, False),       # 64-row tiles, partial N tile
    (64, 256, 192, True, False),       # 64-row tiles, exact
    (520, 328, 384, True, False),      # 128-row tiles, partial M and N tiles
    (1040, 4104, 256, True, False),    # 9 x 17 = 153 tiles: more than one persistent wave
    (130, 264, 200, False, False),     # other operand majors
    (33, 72, 136, False, True),
    (200, 136, 128, True, True),
]


@pytest.mark.parametrize("M,N,K,trans_a,trans_b", GEMM_SHAPES)
def test_gemm_fp32_output(M, N, K, trans_a, trans_b):
    ops = _ops()
    a = _mat(*((K, M) if trans_a else (M, K)), seed=M + N)
    b = _mat(*((N, K) if trans_b else (K, N)), seed=K)
    acc = _acc(a, b, trans_a, trans_b)
    ldc = -(-(N + 9) // 4) * 4                                    # C is a strided view with sentinels on every side
    buf = torch.full((M + 3, ldc), 7.25, dtype=F32, device=DEV)
    c = buf[1:M + 1, 4:4 + N]
    sentinel = buf.clone()

    # (a) overwrite: the accumulators themselves; rounded, the bf16 GEMM's output; close to the fp64 product
    ops.gemm(a, b, out=c, trans_a=trans_a, trans_b=trans_b)
    torch.cuda.synchronize()
    assert torch.equal(c, acc)
    assert torch.equal(c.to(BF16), ops.gemm(a, b, trans_a=trans_a, trans_b=trans_b))
    A64 = (a.t() if trans_a else a).double()
    B64 = (b.t() if trans_b else b).double()
    bound = 2 * K * 2.0 ** -24 * (A64.abs() @ B64.abs())          # fp32 accumulation of K products
    assert bool(((c.double() - A64 @ B64).abs() <= bound).all())

    # (b) accumulate onto a random fp32 C0: C0 + C_fresh in fp32, one add per element (subnormal sums flush to zero)
    c0 = _rand(M, N, scale=3.0, seed=5, dtype=F32)
    c.copy_(c0)
    ops.gemm(a, b, out=c, trans_a=trans_a, trans_b=trans_b, accumulate=True)
    want = c0 + acc
    normal = want.abs() >= 2.0 ** -126
    assert torch.equal(c[normal], want[normal])
    assert bool((c[~normal] == 0).all())

    # (c) nothing outside the view was written
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[1:M + 1, 4:4 + N] = False
    assert torch.equal(buf[mask], sentinel[mask])


def test_gemm_fp32_output_argument_errors():
    from paddlenlp_b200 import _lib

    ops = _ops()
    M, N, K = 64, 72, 64
    a, b = _mat(K, M, 1), _mat(K, N, 2)
    buf = torch.full((M, N + 8), float("nan"), dtype=F32, device=DEV)
    for view in (buf.view(-1)[: M * (N + 2)].view(M, N + 2)[:, :N],   # ldc % 4 != 0
                 buf[:, 1:1 + N]):                                     # base 4 bytes off
        with pytest.raises(_lib.B200Error, match="gemm_f32"):
            ops.gemm(a, b, out=view, trans_a=True)
    with pytest.raises(_lib.B200Error, match="ldc"):
        _lib.call("b200_gemm_bf16_f32", _lib.ptr(a), _lib.ptr(b), _lib.ptr(buf), M, N, K, a.stride(0), b.stride(0), N - 4, 1, 1, 0,
                  _lib.stream_ptr())                                   # ldc < N
    torch.cuda.synchronize()
    assert bool(buf.isnan().all())
    with pytest.raises(ValueError):
        ops.gemm(a, b, out=buf[:, :N], trans_a=True, bias=torch.zeros(N, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------------------------------------------------------
def _engine(model_type, tied, head_dim, recompute):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.transformers.decoder_engine import DecoderEngine

    nh = 256 // head_dim
    kw = dict(vocab_size=512, hidden_size=256, intermediate_size=640, num_hidden_layers=2, num_attention_heads=nh,
              num_key_value_heads=max(1, nh // 2), max_position_embeddings=256, rope_theta=10000.0, rms_norm_eps=1e-5,
              tie_word_embeddings=tied, recompute=recompute)
    cfg = T.Qwen2Config(**kw) if model_type == "qwen2" else T.LlamaConfig(**kw)
    eng = DecoderEngine(cfg, device=DEV)
    eng.init_weights(7)
    if eng.qkv_bias:                                         # non-zero biases, so that the bias path matters
        eng.p[[n for n in eng.p if n.endswith("qkv_b")][0]].normal_(0, 0.02)
        eng.params_changed()
    return eng


def _batch(seed, B=2, S=128, V=512):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, S + 1), generator=g)
    return ids[:, :-1].to(DEV), ids[:, 1:].to(DEV)


class _GemmRecorder:
    """Wraps ops.gemm: every call with an fp32 output (the engine's weight gradients) is checked on the spot against the
    bf16 GEMM of the same operands (fresh) or against C_old + the fp32 GEMM of the same operands (accumulate)."""

    def __init__(self, ops):
        self.orig = ops.gemm
        self.checked = 0

    def __call__(self, a, b, out=None, **kw):
        if out is None or out.dtype != F32:
            return self.orig(a, b, out=out, **kw)
        old = out.clone() if kw.get("accumulate") else None
        self.orig(a, b, out=out, **kw)
        ta, tb = kw.get("trans_a", False), kw.get("trans_b", False)
        if old is None:
            assert torch.equal(out.to(BF16), self.orig(a, b, trans_a=ta, trans_b=tb)), "fp32 dW rounded != bf16 dW"
        else:
            fresh = self.orig(a, b, out=torch.empty_like(out), trans_a=ta, trans_b=tb)
            want = old + fresh
            normal = want.abs() >= 2.0 ** -126
            assert torch.equal(out[normal], want[normal]), "fp32 accumulation is not C_old + fresh"
        self.checked += 1
        return out


def _mat_names(eng):
    return [n for n, (o, _) in eng._offsets.items() if o < eng.decay_end]


def _relerr(x, ref):
    return float((x.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-30))


ENGINE_CONFIGS = [("llama", False, 128, False), ("llama", True, 64, True), ("qwen2", False, 64, False),
                  ("qwen2", True, 128, True), ("llama", False, 64, True), ("qwen2", False, 128, False)]


@pytest.mark.parametrize("model_type,tied,head_dim,recompute", ENGINE_CONFIGS)
def test_engine_one_micro_batch(model_type, tied, head_dim, recompute, monkeypatch):
    ops = _ops()
    eng = _engine(model_type, tied, head_dim, recompute)
    ids, lab = _batch(0)
    eng.forward_loss(ids, lab)
    eng.backward()
    g16 = {n: v.clone() for n, v in eng.g.items()}
    eng.clear_grad()
    eng.set_master_grad(True)
    assert eng.flat_grads.dtype == F32 and eng.flat_grads.numel() == eng.numel
    rec = _GemmRecorder(ops)
    monkeypatch.setattr(ops, "gemm", rec)
    eng.forward_loss(ids, lab)
    eng.backward()
    monkeypatch.undo()
    # the weight-gradient GEMMs: 4 per layer and the head's (untied) or the head's term of the embedding gradient (tied)
    assert rec.checked == 4 * eng.L + 1
    ulp = 2.0 ** -8
    for n in _mat_names(eng):
        # other passes' attention sums differ in the last bits: the matrices agree with the bf16 mode's to bf16 noise
        assert _relerr(eng.g[n], g16[n].float()) < (3 * ulp if n == "embed" else 1e-2), n
    for n, (o, _) in eng._offsets.items():
        if o >= eng.decay_end:                                  # norm weights, biases: one rounding apart
            assert _relerr(eng.g[n], g16[n].float()) <= ulp, n


@pytest.mark.parametrize("model_type,tied", [("llama", False), ("qwen2", True)])
def test_engine_four_micro_batches(model_type, tied, monkeypatch):
    ops = _ops()
    eng = _engine(model_type, tied, 128, False)
    batches = [_batch(10 + i) for i in range(4)]
    eng.set_master_grad(True)
    singles = []
    for ids, lab in batches:                                    # each micro-batch's fp32 gradient on its own
        eng.clear_grad()
        eng.forward_loss(ids, lab)
        eng.backward()
        singles.append(eng.flat_grads.clone())
    eng.clear_grad()
    rec = _GemmRecorder(ops)
    monkeypatch.setattr(ops, "gemm", rec)
    for ids, lab in batches:
        eng.forward_loss(ids, lab)
        eng.backward()
    monkeypatch.undo()
    assert rec.checked == 4 * (4 * eng.L + 1)                   # every dW GEMM: C_old + fresh, bit for bit
    acc32 = eng.flat_grads.clone()
    in_order = singles[0] + singles[1] + singles[2] + singles[3]
    exact64 = sum(s.double() for s in singles)
    eng.clear_grad()
    eng.set_master_grad(False)
    for ids, lab in batches:
        eng.forward_loss(ids, lab)
        eng.backward()
    acc16 = eng.flat_grads.float()
    v32 = eng.named_views(flat=acc32)
    vin = eng.named_views(flat=in_order)
    v64 = eng.named_views(flat=exact64)
    v16 = eng.named_views(flat=acc16)
    for k in v32:
        # separate passes: same up to the attention backward's unordered sums (bf16 noise in the activation gradients)
        assert _relerr(v32[k], vin[k]) < 1e-6, k
    for k in v32:
        print(f"{k}: relative L2 distance from the fp64 sum of the 4 micro-batches: fp32 gradients "
              f"{_relerr(v32[k], v64[k]):.2e}, bf16 gradients {_relerr(v16[k], v64[k]):.2e}")
    e32, e16 = _relerr(acc32, exact64), _relerr(acc16, exact64)
    print(f"whole buffer: fp32 gradients {e32:.2e}, bf16 gradients {e16:.2e}")
    assert e32 < e16 / 2


# ---------------------------------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------------------------------
def test_sqnorm_and_adamw_on_fp32_gradients():
    ops = _ops()
    n, decay_end = 1 << 20, 3 << 18
    g16 = _rand(n, scale=1e-2, seed=3)
    g32 = g16.float()
    assert torch.equal(ops.grad_sqnorm(g16, scale=0.5), ops.grad_sqnorm(g32, scale=0.5))
    p0 = _rand(n, scale=0.02, seed=4)
    state = []
    for g in (g16, g32):
        p = p0.clone()
        master, m, v = p.float(), torch.zeros(n, dtype=F32, device=DEV), torch.zeros(n, dtype=F32, device=DEV)
        for step in range(1, 4):
            sq = ops.grad_sqnorm(g, scale=0.5)
            ops.adamw_step(p, g, master, m, v, sq, decay_end=decay_end, lr=1e-3, beta1=0.9, beta2=0.95, eps=1e-8,
                           weight_decay=0.1, step=step, grad_scale=0.5, max_grad_norm=0.01)
        state.append((p, master, m, v))
    for x16, x32 in zip(*state):
        assert torch.equal(x16, x32)
    gen = _rand(n + 5, scale=1.0, seed=6, dtype=F32) * torch.logspace(-2, 2, n + 5, device=DEV)
    got = float(ops.grad_sqnorm(gen, scale=2.0))
    ref = float((gen.double() * 2.0).square().sum())
    assert abs(got - ref) <= 1e-6 * ref


# ---------------------------------------------------------------------------------------------------------------------------
# Trainer
# ---------------------------------------------------------------------------------------------------------------------------
class _Toy(torch.utils.data.Dataset):
    def __init__(self, n, S=128, V=512):
        self.tok = torch.randint(1, V, (n, S + 1), generator=torch.Generator().manual_seed(1234))

    def __len__(self):
        return self.tok.shape[0]

    def __getitem__(self, i):
        return {"input_ids": self.tok[i, :-1].clone(), "labels": self.tok[i, 1:].clone()}


def _trainer(out_dir, master, save_steps=0, max_steps=10):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    model = T.LlamaForCausalLM(T.LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                                             num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=256,
                                             seq_length=128, rope_theta=500000.0, rms_norm_eps=1e-5))
    args = TrainingArguments(output_dir=str(out_dir), per_device_train_batch_size=1, gradient_accumulation_steps=4,
                             max_steps=max_steps, learning_rate=1e-3, weight_decay=0.01, warmup_steps=2, logging_steps=1,
                             max_seq_length=128, lr_scheduler_type="cosine", save_steps=save_steps, amp_master_grad=master)
    return Trainer(model=model, args=args, train_dataset=_Toy(40))


def test_trainer_amp_master_grad(tmp_path):
    import shutil

    on = _trainer(tmp_path / "on", True, save_steps=5)
    on.train()
    off = _trainer(tmp_path / "off", False)
    off.train()
    eng = on.model.engine
    assert eng.flat_grads.dtype == F32
    base = eng.flat_grads.data_ptr()
    views = eng.named_views(grads=True)
    for name, p in on.model.named_parameters():
        assert p.grad is None and p.main_grad.dtype == F32, name
        assert p.main_grad.data_ptr() == views[name].data_ptr() and base <= p.main_grad.data_ptr() < base + 4 * eng.numel
    l_on = [h["loss"] for h in on.state.log_history]
    l_off = [h["loss"] for h in off.state.log_history]
    assert len(l_on) == len(l_off) == 10
    assert l_on[0] == l_off[0]                                # the first step's losses come before any update
    assert max(abs(x - y) for x, y in zip(l_on, l_off)) < 2e-2
    # resume from checkpoint-5 in fp32-gradient mode: step 6 as in the uninterrupted run
    shutil.copytree(tmp_path / "on" / "checkpoint-5", tmp_path / "res" / "checkpoint-5")
    res = _trainer(tmp_path / "res", True)
    res.train(resume_from_checkpoint=True)
    l_res = [h["loss"] for h in res.state.log_history]
    assert l_res[:6] == l_on[:6]
    assert max(abs(x - y) for x, y in zip(l_res[6:], l_on[6:])) < 2e-3
    assert math.isfinite(l_res[-1])
