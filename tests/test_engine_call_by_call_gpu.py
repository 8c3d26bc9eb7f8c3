"""DecoderEngine's training step checked call by call against fp64, at every preset's width, with bf16 and fp32 gradients.

The kernel tests check each kernel on random operands of the right shape; the whole-model tests judge a gradient by one
relative error per tensor, which accepts a wrong 128 x 256 tile of a weight gradient, a dropped accumulate on one matrix or
one wrong RMSNorm row.  Here every ops.* function the engine calls is wrapped.  Each call is checked on the spot against
fp64 of the operands it actually received (plus what an accumulated gradient view held before the call), with the per
element, per tile and per row checkers of the kernel tests.  Outputs the engine lets an op allocate are handed to the kernel
pre-filled with NaN, and the gradient buffer is NaN before the first micro-batch, so an element that is never written, or
a view that is accumulated into instead of written, fails as non-finite.

Numeric checks prove each kernel right on its inputs, not that the engine gave it the right inputs.  So the checker also
labels every tensor an op returns or writes (l{i}.n1, l{i}.qkv, l{i}.dgu, ...) and the parameter and gradient views
(p.<name>, g.<name>), by device address range, so that a column view such as q, k or v resolves to its packed buffer and its
column offset.  schedule() states, call by call, which labels and flags (accumulate, backward, ...) each op must receive in
_layer_fwd / _layer_bwd order; the checker matches every call against it, which also fixes the exact call count of every
op kind, recomputed forwards included.  With recompute=True every activation the backward recomputes must be bit-identical
to the one the forward produced.

Cases: two decoder layers, the real vocabulary, two micro-batches (fresh, then accumulated), backward(grad_scale=0.5).
The sabotage tests at the bottom put a plain-Python fault under the checker and show that it raises.
"""
import contextlib
import dataclasses
import io
import math
from collections import Counter

import pytest
import torch

from oracle import llama_ref as R
from test_attention_training_at_scale_gpu import FRONT, check_backward, check_forward, pipeline_mask, reference
from test_kernels_at_scale_gpu import (BF16_REL, GEMM_C, ROW_TOL, assert_gemm_close, assert_rows_close,  # noqa: F401
                                       assert_within_ulps, bf16_ulp, fp64_reference, sm_count)
from test_master_grad_at_scale_gpu import (ENGINE_GEMM_C32, assert_colsum_close, assert_gemm_f32_close, assert_scatter_close,
                                           check_bound)

DEV = "cuda:0"
BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
NAN = float("nan")
# Per-element allowance of the fp32 accumulation in the bf16-output GEMMs that read dlogits: dhf = dlogits @ head^T (or
# dlogits @ E, K = V) and the lm-head / tied-embedding weight gradient.  A row of dlogits holds one term (p - 1) grad_scale /
# count at its label among V softmax terms ~1e5 times smaller, and a vocabulary column one such term per token labelled with
# it: the accumulator carries the large term and every later k-step adds values below its last bits, so the error grows
# linearly in K (see ENGINE_GEMM_C32).  Measured on an H100 80GB HBM3 (700 W power limit) over every case below: c_need
# <= 3.2e-4 for dhf (K = V; Qwen2-7B, V 152 064) and <= 2.1e-5 for the bf16 head weight gradient, against <= 2.6e-6 for
# every other GEMM of the step (GEMM_C).  c is ~4x the worst.
ENGINE_GEMM_C = 1.3e-3
CE_ROWS = 1024                 # rows of the fp64 cross-entropy reference at a time


# ----------------------------------------------------------------------------------------------------------
# Labels: which op produced a tensor, by device address range
# ----------------------------------------------------------------------------------------------------------
def span(t):
    """[lo, hi) byte addresses covered by the elements of t (non-negative strides)."""
    lo = t.data_ptr()
    if t.numel() == 0:
        return lo, lo
    ext = sum((n - 1) * s for n, s in zip(t.shape, t.stride()))
    return lo, lo + (ext + 1) * t.element_size()


class Labels:
    """Names of tensors by address range.  The tensors are held, so no address is reused while its name is known.  A name
    given to exactly the range of an earlier one replaces it (an in-place op: logits -> dlogits)."""

    def __init__(self):
        self.entries = []                  # (lo, hi, name, tensor)

    def add(self, t, name):
        lo, hi = span(t)
        self.entries = [e for e in self.entries if (e[0], e[1]) != (lo, hi)]
        self.entries.append((lo, hi, name, t))

    def name(self, t):
        """The name of the smallest labelled range containing t: `name` for exactly that range, `name+off` (element offset
        of t's first element) for a view inside it, '?' when no labelled range contains t, None for None."""
        if t is None:
            return None
        lo, hi = span(t)
        best = None
        for e in self.entries:
            if e[0] <= lo and hi <= e[1] and (best is None or e[1] - e[0] < best[1] - best[0]):
                best = e
        if best is None:
            return "?"
        if (best[0], best[1]) == (lo, hi):
            return best[2]
        return f"{best[2]}+{(lo - best[0]) // t.element_size()}"


# ----------------------------------------------------------------------------------------------------------
# The schedule: every op call of one forward_loss + backward, in order, with the labels of its operands
# ----------------------------------------------------------------------------------------------------------
FIELDS = {                     # operand (label) and flag fields per op, with the value of an operand the engine omits
    "embedding_fwd": dict(table="?", out=None),
    "rmsnorm_fwd": dict(x="?", w="?", out=None, rstd=None),
    "gemm": dict(a="?", b="?", out=None, bias=None, residual=None, trans_a=False, trans_b=False, accumulate=False),
    "rope_inplace": dict(x="?", backward=False, position_ids=False),
    "flash_attn_fwd": dict(q="?", k="?", v="?", out=None, mask=False),
    "flash_attn_bwd": dict(q="?", k="?", v="?", o="?", dout="?", lse="?", dq="?", dk="?", dv="?", mask=False),
    "gemm_swiglu": dict(x="?", w="?", gate_up=None, out=None),
    "gemm_swiglu_bwd": dict(dy="?", w_down="?", gate_up="?", dgate_up=None),
    "swiglu_fwd": dict(gate_up="?", out=None),
    "swiglu_bwd": dict(gate_up="?", dout="?", dgate_up=None),
    "ce_fwd": dict(logits="?"),
    "ce_bwd_": dict(logits="?", loss_tok="?", lse="?", loss_out="?"),
    "rmsnorm_bwd": dict(dy="?", x="?", w="?", rstd="?", dw="?", dres=None, accumulate_dw=False, dx=None),
    "colsum": dict(a="?", out="?", accumulate=False),
    "embedding_bwd": dict(dout="?", dtable="?"),
}


@dataclasses.dataclass(frozen=True)
class Geometry:
    L: int
    nh: int
    kvh: int
    d: int
    tied: bool
    fused: bool                # SwiGLU in the GEMM epilogues (I % 64 == 0)
    bias: bool                 # Qwen2 q/k/v bias
    recompute: bool
    pos: bool = False          # position_ids given
    mask: bool = False         # FlashMask start rows given


@dataclasses.dataclass
class Call:
    op: str
    args: dict
    outs: tuple = ()
    key: str = None            # a layer-forward op: the same key marks the op in the recomputed forward
    recomputed: bool = False


def _call(op, outs=(), key=None, recomputed=False, **args):
    unknown = set(args) - set(FIELDS[op])
    assert not unknown, f"{op}: unknown fields {unknown}"
    return Call(op, {**FIELDS[op], **args}, tuple(outs), key, recomputed)


def _layer_fwd_calls(i, x, g, recomputed):
    n = lambda s: f"l{i}.{s}"           # noqa: E731
    p = lambda s: f"p.l{i}.{s}"         # noqa: E731
    qn, kn = g.nh * g.d, g.kvh * g.d
    C = []

    def call(op, outs=(), **args):
        C.append(_call(op, outs, key=f"l{i}.fwd{len(C)}", recomputed=recomputed, **args))

    call("rmsnorm_fwd", (n("n1"), n("rstd1")), x=x, w=p("ln1"))
    call("gemm", (n("qkv"),), a=n("n1"), b=p("qkv_w"), bias=p("qkv_b.f32") if g.bias else None)
    call("rope_inplace", (n("qkv"),), x=n("qkv"), backward=False, position_ids=g.pos)
    call("flash_attn_fwd", (n("attn"), n("lse")), q=n("qkv+0"), k=n(f"qkv+{qn}"), v=n(f"qkv+{qn + kn}"), mask=g.mask)
    call("gemm", (n("x1"),), a=n("attn"), b=p("o_w"), residual=x)
    call("rmsnorm_fwd", (n("n2"), n("rstd2")), x=n("x1"), w=p("ln2"))
    if g.fused:
        call("gemm_swiglu", (n("gu"), n("m")), x=n("n2"), w=p("gu_w"))
    else:
        call("gemm", (n("gu"),), a=n("n2"), b=p("gu_w"))
        call("swiglu_fwd", (n("m"),), gate_up=n("gu"))
    call("gemm", (n("x2"),), a=n("m"), b=p("down_w"), residual=n("x1"))
    return C


def schedule(g: Geometry, acc: bool):
    """Every op call of forward_loss + backward (decoder_engine.py: hidden_states, _layer_fwd, backward, _layer_bwd) with
    the labels its operands must carry and its flags; `acc`: the backward accumulates (a micro-batch after the first).
    Layer i's input is `emb` (i = 0) or l{i-1}.x2, its output gradient l{i}.dx2 and its input gradient l{i-1}.dx2 or
    `demb`."""
    E = []

    def call(op, outs=(), **args):
        E.append(_call(op, outs, **args))

    qn, kn = g.nh * g.d, g.kvh * g.d
    layer_in = lambda i: "emb" if i == 0 else f"l{i - 1}.x2"        # noqa: E731
    call("embedding_fwd", ("emb",), table="p.embed")
    for i in range(g.L):
        E += _layer_fwd_calls(i, layer_in(i), g, recomputed=False)
    last = f"l{g.L - 1}.x2"
    call("rmsnorm_fwd", ("hf", "rstd_f"), x=last, w="p.norm")
    if g.tied:
        call("gemm", ("logits",), a="hf", b="p.embed", trans_b=True)
    else:
        call("gemm", ("logits",), a="hf", b="p.head")
    call("ce_fwd", ("loss_out", "loss_tok", "ce_lse"), logits="logits")
    call("ce_bwd_", ("dlogits",), logits="logits", loss_tok="loss_tok", lse="ce_lse", loss_out="loss_out")
    if g.tied:
        call("gemm", ("dhf",), a="dlogits", b="p.embed")
        call("gemm", (), a="dlogits", b="hf", out="g.embed", trans_a=True, accumulate=acc)
    else:
        call("gemm", ("dhf",), a="dlogits", b="p.head", trans_b=True)
        call("gemm", (), a="hf", b="dlogits", out="g.head", trans_a=True, accumulate=acc)
    call("rmsnorm_bwd", (f"l{g.L - 1}.dx2",), dy="dhf", x=last, w="p.norm", rstd="rstd_f", dw="g.norm", accumulate_dw=acc)
    for i in reversed(range(g.L)):
        n = lambda s: f"l{i}.{s}"       # noqa: E731
        p = lambda s: f"p.l{i}.{s}"     # noqa: E731
        gr = lambda s: f"g.l{i}.{s}"    # noqa: E731
        if g.recompute:
            E += _layer_fwd_calls(i, layer_in(i), g, recomputed=True)
        if g.fused:
            call("gemm_swiglu_bwd", (n("dgu"),), dy=n("dx2"), w_down=p("down_w"), gate_up=n("gu"))
            call("gemm", (), a=n("m"), b=n("dx2"), out=gr("down_w"), trans_a=True, accumulate=acc)
        else:
            call("gemm", (n("dm"),), a=n("dx2"), b=p("down_w"), trans_b=True)
            call("gemm", (), a=n("m"), b=n("dx2"), out=gr("down_w"), trans_a=True, accumulate=acc)
            call("swiglu_bwd", (n("dgu"),), gate_up=n("gu"), dout=n("dm"))
        call("gemm", (n("dn2"),), a=n("dgu"), b=p("gu_w"), trans_b=True)
        call("gemm", (), a=n("n2"), b=n("dgu"), out=gr("gu_w"), trans_a=True, accumulate=acc)
        call("rmsnorm_bwd", (n("dx1"),), dy=n("dn2"), x=n("x1"), w=p("ln2"), rstd=n("rstd2"), dw=gr("ln2"), dres=n("dx2"),
             accumulate_dw=acc)
        call("gemm", (n("dattn"),), a=n("dx1"), b=p("o_w"), trans_b=True)
        call("gemm", (), a=n("attn"), b=n("dx1"), out=gr("o_w"), trans_a=True, accumulate=acc)
        call("flash_attn_bwd", (n("dqkv"),), q=n("qkv+0"), k=n(f"qkv+{qn}"), v=n(f"qkv+{qn + kn}"), o=n("attn"),
             dout=n("dattn"), lse=n("lse"), dq=n("dqkv+0"), dk=n(f"dqkv+{qn}"), dv=n(f"dqkv+{qn + kn}"), mask=g.mask)
        call("rope_inplace", (n("dqkv"),), x=n("dqkv"), backward=True, position_ids=g.pos)
        if g.bias:
            call("colsum", (), a=n("dqkv"), out=gr("qkv_b"), accumulate=acc)
        call("gemm", (n("dn1"),), a=n("dqkv"), b=p("qkv_w"), trans_b=True)
        call("gemm", (), a=n("n1"), b=n("dqkv"), out=gr("qkv_w"), trans_a=True, accumulate=acc)
        call("rmsnorm_bwd", (f"l{i - 1}.dx2" if i else "demb",), dy=n("dn1"), x=layer_in(i), w=p("ln1"), rstd=n("rstd1"),
             dw=gr("ln1"), dres=n("dx1"), accumulate_dw=acc)
    call("embedding_bwd", (), dout="demb", dtable="g.embed")
    return E


def expected_counts(L, tied, fused, bias, recompute):
    """Calls per op kind of one forward_loss + backward, counted from decoder_engine.py independently of schedule()."""
    f = 2 if recompute else 1                                      # layer forwards run twice with recompute
    c = dict(embedding_fwd=1, embedding_bwd=1, ce_fwd=1, ce_bwd_=1, rmsnorm_fwd=2 * L * f + 1, rmsnorm_bwd=2 * L + 1,
             rope_inplace=L * f + L, flash_attn_fwd=L * f, flash_attn_bwd=L)
    if fused:
        c.update(gemm=3 * L * f + 1 + 7 * L + 2, gemm_swiglu=L * f, gemm_swiglu_bwd=L)
    else:
        c.update(gemm=4 * L * f + 1 + 8 * L + 2, swiglu_fwd=L * f, swiglu_bwd=L)
    if bias:
        c["colsum"] = L
    return c


class Schedule:
    """Matches op calls one by one against schedule()."""

    def __init__(self, calls):
        self.calls = list(calls)
        self.i = 0

    def peek(self):
        return self.calls[self.i] if self.i < len(self.calls) else None

    def next(self, op, got):
        if self.i >= len(self.calls):
            raise AssertionError(f"call {self.i} {op}{got}: the schedule has only {len(self.calls)} calls")
        e = self.calls[self.i]
        if e.op != op or e.args != got:
            diff = {k: (e.args.get(k), got.get(k)) for k in set(e.args) | set(got) if e.args.get(k) != got.get(k)}
            raise AssertionError(f"call {self.i}: expected {e.op} with {e.args}, got {op} with {got}; "
                                 f"differs in (expected, got): {diff}")
        self.i += 1
        return e

    def done(self):
        assert self.i == len(self.calls), f"{len(self.calls) - self.i} scheduled calls never made, first: " \
                                          f"{self.calls[self.i].op} {self.calls[self.i].args}"


def same_bits(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


# ----------------------------------------------------------------------------------------------------------
# CPU: label resolution and the schedule matcher
# ----------------------------------------------------------------------------------------------------------
def test_labels_resolve_views_to_their_buffer():
    B, S, nh, kvh, d = 2, 32, 12, 2, 128
    qn, kn = nh * d, kvh * d
    qkv = torch.zeros(B * S, qn + 2 * kn, dtype=BF16)
    lab = Labels()
    lab.add(qkv, "l0.qkv")
    q4 = qkv.view(B, S, -1)
    assert lab.name(qkv) == "l0.qkv" and lab.name(q4) == "l0.qkv"
    assert lab.name(q4[:, :, :qn].unflatten(2, (nh, d))) == "l0.qkv+0"
    assert lab.name(q4[:, :, qn:qn + kn].unflatten(2, (kvh, d))) == f"l0.qkv+{qn}"
    assert lab.name(q4[:, :, qn + kn:].unflatten(2, (kvh, d))) == f"l0.qkv+{qn + kn}"
    # views of one flat buffer: the smallest labelled range wins, a transposed view keeps its name
    flat = torch.zeros(1000, dtype=BF16)
    lab.add(flat, "flat")
    lab.add(flat[0:100].view(10, 10), "p.a")
    lab.add(flat[104:204], "p.b")
    assert lab.name(flat[0:100].view(10, 10).t()) == "p.a"
    assert lab.name(flat[104:204]) == "p.b" and lab.name(flat[110:120]) == "p.b+6"
    assert lab.name(flat[90:110]) == "flat+90"                     # straddles p.a and p.b
    assert lab.name(torch.zeros(4)) == "?" and lab.name(None) is None
    # in place: the same range renamed
    logits = torch.zeros(8, 16, dtype=BF16)
    lab.add(logits, "logits")
    lab.add(logits, "dlogits")
    assert lab.name(logits) == "dlogits" and sum(e[2] == "logits" for e in lab.entries) == 0


GEOMS = [Geometry(L, 14, 2, 64, tied, fused, bias, rc) for L in (1, 2) for tied in (False, True) for fused in (False, True)
         for bias in (False, True) for rc in (False, True)]


@pytest.mark.parametrize("g", GEOMS, ids=lambda g: f"L{g.L}-tied{int(g.tied)}-fused{int(g.fused)}-bias{int(g.bias)}-rc{int(g.recompute)}")
def test_schedule_counts_match_the_engine(g):
    got = Counter(c.op for c in schedule(g, acc=False))
    assert dict(got) == expected_counts(g.L, g.tied, g.fused, g.bias, g.recompute)
    assert all(c.args["accumulate"] for c in schedule(g, acc=True) if c.op == "gemm" and c.args["out"])


def test_schedule_matcher_rejects_wiring_faults():
    g = Geometry(2, 14, 2, 64, True, True, True, True, pos=True, mask=True)
    calls = schedule(g, acc=True)
    s = Schedule(calls)
    for c in calls:
        s.next(c.op, dict(c.args))
    s.done()
    with pytest.raises(AssertionError, match="only"):
        s.next("gemm", {})
    k = next(j for j, c in enumerate(calls) if c.args.get("out") == "g.l1.gu_w")

    def replay(j, op, args):
        s = Schedule(calls)
        for c in calls[:j]:
            s.next(c.op, dict(c.args))
        s.next(op, args)

    with pytest.raises(AssertionError, match=r"differs in .*'a': \('l1.n2', 'l1.n1'\)"):   # n1 where the gate|up dW expects n2
        replay(k, "gemm", {**calls[k].args, "a": "l1.n1"})
    with pytest.raises(AssertionError, match=r"differs in .*'accumulate': \(True, False\)"):  # written, not accumulated
        replay(k, "gemm", {**calls[k].args, "accumulate": False})
    j = next(j for j, c in enumerate(calls) if c.op == "rmsnorm_bwd" and c.args["w"] == "p.l0.ln2")
    with pytest.raises(AssertionError, match=r"differs in .*'dres': \('l0.dx2', 'l0.dx1'\)"):   # ln2 gets the wrong dres
        replay(j, "rmsnorm_bwd", {**calls[j].args, "dres": "l0.dx1"})
    j = next(j for j, c in enumerate(calls) if c.op == "rope_inplace" and c.args["backward"])
    with pytest.raises(AssertionError, match=r"differs in .*'backward': \(True, False\)"):
        replay(j, "rope_inplace", {**calls[j].args, "backward": False})
    j = next(j for j, c in enumerate(calls) if c.op == "flash_attn_bwd")
    with pytest.raises(AssertionError, match=r"differs in .*'dk'"):   # dk and dv swapped
        replay(j, "flash_attn_bwd", {**calls[j].args, "dk": calls[j].args["dv"], "dv": calls[j].args["dk"]})
    j = next(j for j, c in enumerate(calls) if c.recomputed)
    n_fwd = sum(1 for c in calls if c.recomputed and c.key.startswith("l1."))
    assert calls[j + n_fwd].op == "gemm_swiglu_bwd"
    with pytest.raises(AssertionError, match="expected rmsnorm_fwd"):  # the recomputed forward skipped
        replay(j, calls[j + n_fwd].op, dict(calls[j + n_fwd].args))
    s = Schedule(calls)
    for c in calls[:-1]:
        s.next(c.op, dict(c.args))
    with pytest.raises(AssertionError, match="never made"):          # the embedding scatter missing
        s.done()


# ----------------------------------------------------------------------------------------------------------
# The checker
# ----------------------------------------------------------------------------------------------------------
OPS = tuple(FIELDS)


class EngineChecker:
    """Wraps every ops.* function in OPS.  Each call is matched against the schedule, run on NaN-filled outputs where the
    engine lets the op allocate them, checked against fp64 of its operands, and its outputs labelled."""

    def __init__(self, eng, geom, monkeypatch):
        from paddlenlp_b200 import ops as o

        self.eng, self.geom, self.o = eng, geom, o
        self.orig = {k: getattr(o, k) for k in OPS}
        for k in OPS:
            monkeypatch.setattr(o, k, getattr(self, k))
        self.count = Counter()
        self.worst = {}
        self.c_need = dict(gemm=0.0, head_dX=0.0, head_dW=0.0, fp32_dW=0.0)
        self.sms = sm_count()
        self.tables_checked = False

    # -- per micro-batch --
    def start(self, mb, S, ids, labels, pos, mask, grad_scale):
        self.mb, self.S, self.ids, self.lab, self.pos, self.mask, self.gs = mb, S, ids, labels, pos, mask, grad_scale
        self.labels = Labels()
        eng = self.eng
        for name in eng.p:
            self.labels.add(eng.p[name], f"p.{name}")
            self.labels.add(eng.g[name], f"g.{name}")
        if self.geom.bias:
            for i in range(eng.L):
                b = eng._bias(i)                                  # the fp32 bias copy the qkv GEMM reads
                assert torch.equal(b, eng.p[f"l{i}.qkv_b"].float())
                self.labels.add(b, f"p.l{i}.qkv_b.f32")
        self.sched = Schedule(schedule(self.geom, acc=mb > 0))
        self.snap = {}
        self.ce = None

    def finish(self):
        self.sched.done()
        self.labels = self.snap = self.ce = None

    # -- helpers --
    def _enter(self, op, **fields):
        got = {k: (self.labels.name(v) if v is None or torch.is_tensor(v) else v) for k, v in fields.items()}
        e = self.sched.next(op, got)
        e.what = f"{op}({', '.join(f'{k}={v}' for k, v in got.items() if v not in (None, False))}) mb {self.mb}"
        return e

    def _produced(self, e, *outs):
        """Recompute: the op's outputs bit-identical to the forward's (checked before the numerics, so that the message says
        which).  Then label the outputs."""
        if e.recomputed:
            for name, a, b in zip(e.outs, outs, self.snap[e.key]):
                assert same_bits(a, b), f"{e.what}: recomputed {name} is not bit-identical to the forward's " \
                                        f"({int((a != b).sum())} elements differ)"
        elif self.geom.recompute and e.key is not None:
            self.snap[e.key] = tuple(t.clone() for t in outs)

    def _label(self, e, *outs):
        for name, t in zip(e.outs, outs):
            self.labels.add(t, name)

    def _done(self, e, ratio):
        self.count[e.op] += 1
        self.worst[e.op] = max(self.worst.get(e.op, 0.0), ratio)

    def _nan(self, *shape, dtype=BF16):
        return torch.full(shape, NAN, dtype=dtype, device=DEV)

    # -- forward ops --
    def embedding_fwd(self, ids, table, out=None):
        e = self._enter("embedding_fwd", table=table, out=out)
        assert torch.equal(ids, self.ids), f"{e.what}: ids are not the batch's"
        y = self._nan(ids.numel(), table.shape[1])
        self.orig["embedding_fwd"](ids, table, out=y)
        assert same_bits(y, table[ids]), f"{e.what}: != table[ids]"
        self._done(e, 0.0)
        self._label(e, y)
        return y

    def rmsnorm_fwd(self, x, w, eps, out=None, rstd=None):
        e = self._enter("rmsnorm_fwd", x=x, w=w, out=out, rstd=rstd)
        assert eps == self.eng.cfg.rms_norm_eps
        h = x.shape[-1]
        rows = x.numel() // h
        y, r = torch.full_like(x, NAN), self._nan(rows, dtype=F32)
        self.orig["rmsnorm_fwd"](x, w, eps, out=y, rstd=r)
        self._produced(e, y, r)
        xd = x.reshape(rows, h).double()
        rref = torch.rsqrt(xd.pow(2).mean(-1) + eps)
        rel = ((r.double() - rref).abs() / rref).nan_to_num(math.inf).max().item()
        assert rel <= 1e-5, f"{e.what}: rstd relative error {rel:.2e}"
        ref = R.rms_norm(xd, w.double(), eps, "bf16")
        assert_within_ulps(y.view(rows, h), ref, ulps=2, max_frac=0.01, what=e.what)
        ulps = ((y.view(rows, h).float() - ref.float()).abs() / (2 * bf16_ulp(ref))).max().item()
        self._done(e, max(rel / 1e-5, ulps))
        self._label(e, y, r)
        return y, r

    def gemm(self, a, b, out=None, *, trans_a=False, trans_b=False, accumulate=False, bias=None, residual=None, max_ctas=0):
        e = self._enter("gemm", a=a, b=b, out=out, bias=bias, residual=residual, trans_a=trans_a, trans_b=trans_b,
                        accumulate=accumulate)
        assert max_ctas == 0
        A, B = (a.t() if trans_a else a), (b.t() if trans_b else b)
        dst = self._nan(A.shape[0], B.shape[1]) if out is None else out
        old = dst.clone() if accumulate else None
        self.orig["gemm"](a, b, out=dst, trans_a=trans_a, trans_b=trans_b, accumulate=accumulate, bias=bias,
                          residual=residual)
        self._produced(e, dst)
        head = "dlogits" in (e.args["a"], e.args["b"])
        if dst.dtype == F32:
            st = assert_gemm_f32_close(dst, A, B, c_old=old, c=ENGINE_GEMM_C32, what=e.what)
            assert st["bf16_rejected"], f"{e.what}: the check cannot tell this fp32 gradient from its bf16 rounding"
        else:
            st = assert_gemm_close(dst, A, B, bias=bias, c_old=old, residual=residual,
                                   c=ENGINE_GEMM_C if head else GEMM_C, what=e.what)
        role = "fp32_dW" if dst.dtype == F32 else ("head_dW" if trans_a else "head_dX") if head else "gemm"
        self.c_need[role] = max(self.c_need[role], st["c_need"])
        self._done(e, st["ratio"])
        self._label(e, dst)
        return dst

    def rope_inplace(self, x, cos, sin, seq_len, num_heads, head_dim, position_ids=None, backward=False):
        e = self._enter("rope_inplace", x=x, backward=backward, position_ids=position_ids is not None)
        eng = self.eng
        assert (num_heads, head_dim, seq_len, x.shape[0]) == (eng.nh + eng.kvh, eng.d, self.S, self.ids.numel()), e.what
        if not self.tables_checked:                               # the tables are the reference's fp32 formula
            c2, s2 = self.o.rope_tables(eng.d, cos.shape[0], float(eng.cfg.rope_theta), DEV,
                                        max_position_embeddings=int(eng.cfg.max_position_embeddings))
            assert torch.equal(cos, c2) and torch.equal(sin, s2), "RoPE tables differ from rope_tables()"
            self.tables_checked = True
        if position_ids is not None:
            assert self.pos is not None and torch.equal(position_ids, self.pos), f"{e.what}: position_ids"
        before = x.clone()
        self.orig["rope_inplace"](x, cos, sin, seq_len, num_heads, head_dim, position_ids=position_ids, backward=backward)
        self._produced(e, x)
        T, H, d = x.shape[0], num_heads, head_dim
        pos = position_ids.long() if position_ids is not None else torch.arange(T, device=DEV) % seq_len
        c, s = cos.double()[pos][:, None, :], sin.double()[pos][:, None, :]
        if backward:
            s = -s
        qk = before[:, :H * d].double().view(T, H, d)
        x1, x2 = qk[..., :d // 2], qk[..., d // 2:]
        ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
        w = assert_rows_close(x[:, :H * d].reshape(T * H, d), ref.view(T * H, d), ROW_TOL, what=e.what)
        assert same_bits(x[:, H * d:], before[:, H * d:]), f"{e.what}: the v columns changed"
        self._done(e, w / ROW_TOL)
        self._label(e, x)
        return x

    def _check_mask(self, e, mask_start):
        if mask_start is None:
            assert self.mask is None, f"{e.what}: the batch has a mask"
        else:
            assert self.mask is not None and torch.equal(mask_start, self.mask), f"{e.what}: mask is not the canonical one"

    def flash_attn_fwd(self, q, k, v, softmax_scale=None, out=None, mask_start=None):
        e = self._enter("flash_attn_fwd", q=q, k=k, v=v, out=out, mask=mask_start is not None)
        self._check_mask(e, mask_start)
        assert softmax_scale is None
        B, S, nh, d = q.shape
        o = self._nan(B, S, nh, d)
        _, lse = self.orig["flash_attn_fwd"](q, k, v, None, out=o, mask_start=mask_start)
        self._produced(e, o, lse)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = reference(q, k, v, None, mask_start, 1.0 / math.sqrt(d))
            rep = check_forward(o, lse, ref, e.what)
        del ref
        self._done(e, max(rep["o"]["ratio"], rep["lse"]["ratio"]))
        self._label(e, o, lse)
        return o, lse

    def gemm_swiglu(self, x, w_gate_up, gate_up=None, out=None, store_gate_up=True):
        e = self._enter("gemm_swiglu", x=x, w=w_gate_up, gate_up=gate_up, out=out)
        assert store_gate_up
        M, I = x.shape[0], w_gate_up.shape[1] // 2
        gu, m = self._nan(M, 2 * I), self._nan(M, I)
        self.orig["gemm_swiglu"](x, w_gate_up, gate_up=gu, out=m)
        self._produced(e, gu, m)
        st = assert_gemm_close(gu, x, w_gate_up, what=e.what + " gate|up")
        self.c_need["gemm"] = max(self.c_need["gemm"], st["c_need"])
        gd, ud = gu[:, :I].double(), gu[:, I:].double()
        ref = gd * torch.sigmoid(gd) * ud                         # SwiGLU of the kernel's own (checked) gate|up
        del gd, ud
        sm = check_bound(m, ref, (BF16_REL + 2.0 ** -20) * ref.abs(), e.what + " m")     # one rounding + fp32 SFU
        del ref
        self._done(e, max(st["ratio"], sm["ratio"]))
        self._label(e, gu, m)
        return gu, m

    def swiglu_fwd(self, gate_up, out=None):
        e = self._enter("swiglu_fwd", gate_up=gate_up, out=out)
        M, I = gate_up.shape[0], gate_up.shape[1] // 2
        m = self._nan(M, I)
        self.orig["swiglu_fwd"](gate_up, out=m)
        self._produced(e, m)
        gd, ud = gate_up[:, :I].double(), gate_up[:, I:].double()
        w = assert_rows_close(m, gd * torch.sigmoid(gd) * ud, ROW_TOL, what=e.what)
        self._done(e, w / ROW_TOL)
        self._label(e, m)
        return m

    # -- criterion --
    def ce_fwd(self, logits, labels, ignore_index=-100):
        e = self._enter("ce_fwd", logits=logits)
        assert ignore_index == -100 and torch.equal(labels, self.lab), f"{e.what}: labels are not the batch's"
        loss_out, loss_tok, lse = self.orig["ce_fwd"](logits, labels, ignore_index)
        T = logits.shape[0]
        lse_ref = torch.empty(T, dtype=F64, device=DEV)
        lt_ref = torch.empty(T, dtype=F64, device=DEV)
        keep = labels != ignore_index
        for r0 in range(0, T, CE_ROWS):
            Ld = logits[r0:r0 + CE_ROWS].double()
            lse_ref[r0:r0 + CE_ROWS] = torch.logsumexp(Ld, -1)
            lab = labels[r0:r0 + CE_ROWS].clamp_min(0)
            picked = Ld.gather(1, lab[:, None])[:, 0]
            lt_ref[r0:r0 + CE_ROWS] = torch.where(keep[r0:r0 + CE_ROWS], lse_ref[r0:r0 + CE_ROWS] - picked, 0.0)
            del Ld
        tol = 2e-5 * (1 + lse_ref.abs())
        r1 = ((lse.double() - lse_ref).abs() / tol).nan_to_num(math.inf)
        r2 = ((loss_tok.double() - lt_ref).abs() / tol).nan_to_num(math.inf)
        assert r1.max().item() <= 1, f"{e.what}: lse row {int(r1.argmax())} off by {r1.max().item():.2f} x its bound"
        assert r2.max().item() <= 1, f"{e.what}: loss row {int(r2.argmax())} off by {r2.max().item():.2f} x its bound"
        cnt = int(keep.sum())
        assert cnt > 0 and bool((lt_ref[keep] > 0).all()) and bool((loss_tok[keep] > 0).all())
        mean_ref = lt_ref[keep].sum().item() / cnt
        assert loss_out[1].item() == cnt, f"{e.what}: count {loss_out[1].item()} != {cnt}"
        assert abs(loss_out[0].item() - mean_ref) <= 1e-5 * mean_ref, f"{e.what}: mean {loss_out[0].item()} vs {mean_ref}"
        self.ce = (lse_ref, cnt)
        self._done(e, max(r1.max().item(), r2.max().item()))
        self._label(e, loss_out, loss_tok, lse)
        return loss_out, loss_tok, lse

    def ce_bwd_(self, logits, labels, loss_tok, lse, loss_out, grad_scale=1.0, grad_scale_dev=None):
        e = self._enter("ce_bwd_", logits=logits, loss_tok=loss_tok, lse=lse, loss_out=loss_out)
        assert torch.equal(labels, self.lab) and grad_scale == self.gs and grad_scale_dev is None, e.what
        L0 = logits.clone()
        self.orig["ce_bwd_"](logits, labels, loss_tok, lse, loss_out, grad_scale, grad_scale_dev)
        lse_ref, cnt = self.ce
        worst = 0.0
        for r0 in range(0, logits.shape[0], CE_ROWS):
            p = torch.exp(L0[r0:r0 + CE_ROWS].double() - lse_ref[r0:r0 + CE_ROWS, None])
            lab = labels[r0:r0 + CE_ROWS]
            rows = (lab >= 0).nonzero()[:, 0]
            p[rows, lab[rows]] -= 1.0
            p *= torch.where(lab != -100, grad_scale / cnt, 0.0)[:, None]     # ignored rows: exactly zero
            worst = max(worst, assert_rows_close(logits[r0:r0 + CE_ROWS], p, ROW_TOL, what=f"{e.what} rows {r0}.."))
            del p
        del L0
        self._done(e, worst / ROW_TOL)
        self._label(e, logits)
        return logits

    # -- backward ops --
    def gemm_swiglu_bwd(self, dy, w_down, gate_up, dgate_up=None):
        e = self._enter("gemm_swiglu_bwd", dy=dy, w_down=w_down, gate_up=gate_up, dgate_up=dgate_up)
        M, I = dy.shape[0], w_down.shape[0]
        dgu = self._nan(M, 2 * I)
        self.orig["gemm_swiglu_bwd"](dy, w_down, gate_up, dgate_up=dgu)
        # the kernel's contract: the same bits as the dX GEMM followed by the swiglu_bwd kernel
        dm = self._nan(M, I)
        self.orig["gemm"](dy, w_down, out=dm, trans_b=True)
        st = assert_gemm_close(dm, dy, w_down.t(), what=e.what + " dX")
        self.c_need["gemm"] = max(self.c_need["gemm"], st["c_need"])
        assert same_bits(dgu, self.orig["swiglu_bwd"](gate_up, dm)), f"{e.what}: != gemm + swiglu_bwd"
        w = self._swiglu_bwd_rows(gate_up, dm, dgu, e.what)
        self._done(e, max(st["ratio"], w / ROW_TOL))
        self._label(e, dgu)
        return dgu

    def _swiglu_bwd_rows(self, gate_up, dm, dgu, what):
        I = dm.shape[1]
        gd, ud, dmd = gate_up[:, :I].double(), gate_up[:, I:].double(), dm.double()
        sg = torch.sigmoid(gd)
        w1 = assert_rows_close(dgu[:, :I], dmd * ud * sg * (1 + gd * (1 - sg)), ROW_TOL, what=what + " d(gate)")
        w2 = assert_rows_close(dgu[:, I:], dmd * gd * sg, ROW_TOL, what=what + " d(up)")
        return max(w1, w2)

    def swiglu_bwd(self, gate_up, dout, dgate_up=None):
        e = self._enter("swiglu_bwd", gate_up=gate_up, dout=dout, dgate_up=dgate_up)
        dgu = torch.full_like(gate_up, NAN)
        self.orig["swiglu_bwd"](gate_up, dout, dgate_up=dgu)
        w = self._swiglu_bwd_rows(gate_up, dout, dgu, e.what)
        self._done(e, w / ROW_TOL)
        self._label(e, dgu)
        return dgu

    def flash_attn_bwd(self, q, k, v, o, dout, lse, dq, dk, dv, softmax_scale=None, mask_start=None):
        base = dq._base
        assert base is not None and dk._base is base and dv._base is base, "dq, dk, dv are not views of one buffer"
        assert base.is_contiguous() and tuple(base.shape) == (q.shape[0] * q.shape[1], self.eng.qkv_n)
        base.fill_(NAN)
        nxt = self.sched.peek()
        self.labels.add(base, nxt.outs[0] if nxt is not None and nxt.op == "flash_attn_bwd" else "?")
        e = self._enter("flash_attn_bwd", q=q, k=k, v=v, o=o, dout=dout, lse=lse, dq=dq, dk=dk, dv=dv,
                        mask=mask_start is not None)
        self._check_mask(e, mask_start)
        assert softmax_scale is None
        self.orig["flash_attn_bwd"](q, k, v, o, dout, lse, dq, dk, dv, None, mask_start=mask_start)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = reference(q, k, v, dout, mask_start, 1.0 / math.sqrt(q.shape[-1]), o, lse)
            rep = check_backward(dq, dk, dv, ref, e.what)
        del ref
        self._done(e, max(r["ratio"] for r in rep.values()))
        return dq, dk, dv

    def rmsnorm_bwd(self, dy, x, w, rstd, dw, dres=None, accumulate_dw=True, dx=None):
        e = self._enter("rmsnorm_bwd", dy=dy, x=x, w=w, rstd=rstd, dw=dw, dres=dres, accumulate_dw=accumulate_dw, dx=dx)
        old = dw.clone() if accumulate_dw else None
        dxo = torch.full_like(x, NAN)
        self.orig["rmsnorm_bwd"](dy, x, w, rstd, dw, dres=dres, accumulate_dw=accumulate_dw, dx=dxo)
        h = x.shape[-1]
        rows = x.numel() // h
        rs = rstd.double()[:, None]
        xh = x.reshape(rows, h).double() * rs
        dyd = dy.reshape(rows, h).double()
        terms = dyd * xh.float().to(BF16).double()               # dw sums dy * bf16(x * rstd), the forward's rounded x-hat
        st = assert_colsum_close(dw, terms, old, parts=min(rows, 2 * self.sms), what=f"{e.what} dw")
        del terms
        if dw.dtype == F32:
            assert st["bf16_rejected"], f"{e.what}: the check cannot tell this fp32 dw from its bf16 rounding"
        gg = dyd * w.double()
        dx_ref = rs * (gg - xh * (gg * xh).mean(-1, keepdim=True))
        del gg, xh, dyd
        if dres is not None:
            dx_ref += dres.reshape(rows, h).double()
        wx = assert_rows_close(dxo.reshape(rows, h), dx_ref, ROW_TOL, what=f"{e.what} dx")
        self._done(e, max(st["ratio"], wx / ROW_TOL))
        self._label(e, dxo)
        return dxo

    def colsum(self, a, out, accumulate=True):
        e = self._enter("colsum", a=a, out=out, accumulate=accumulate)
        old = out.clone() if accumulate else None
        self.orig["colsum"](a, out, accumulate=accumulate)
        st = assert_colsum_close(out, a, old, parts=min(a.shape[0], 64), what=e.what)
        if out.dtype == F32:
            assert st["bf16_rejected"], f"{e.what}: the check cannot tell this fp32 gradient from its bf16 rounding"
        self._done(e, st["ratio"])
        return out

    def embedding_bwd(self, ids, dout, dtable):
        e = self._enter("embedding_bwd", dout=dout, dtable=dtable)
        assert torch.equal(ids, self.ids), f"{e.what}: ids are not the batch's"
        old = dtable.clone()
        self.orig["embedding_bwd"](ids, dout, dtable)
        st = assert_scatter_close(dtable, old, ids.reshape(-1), dout.reshape(-1, dtable.shape[1]), what=e.what)
        if dtable.dtype == F32:
            assert st["bf16_rejected"], f"{e.what}: the check cannot tell this fp32 gradient from its bf16 rounding"
        self._done(e, st["ratio"])
        return dtable


# ----------------------------------------------------------------------------------------------------------
# GPU: the cases
# ----------------------------------------------------------------------------------------------------------
def make_config(family, preset, L, recompute=False, **kw):
    import paddlenlp_b200.transformers as T

    cls = T.LlamaConfig if family == "llama" else T.Qwen2Config
    return getattr(cls, preset)(num_hidden_layers=L, recompute=recompute, **kw)


def positions_from_mask(ms):
    """position_ids restarting at every document of canonical start rows ms [B, S] (a document = a run of equal rows)."""
    B, S = ms.shape
    idx = torch.arange(S).expand(B, S)
    new = torch.ones(B, S, dtype=torch.bool)
    new[:, 1:] = ms[:, 1:] != ms[:, :-1]
    start = torch.where(new, idx, torch.zeros_like(idx)).cummax(1).values
    return (idx - start).to(torch.int64)


def make_batch(cfg, B, S, seed, sft):
    """Token ids and next-token labels; sft: packed documents of the SFT pipeline (start rows, position_ids restarting per
    document, label -100 on the padding)."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, cfg.vocab_size, (B, S + 1), generator=g)
    ids, lab = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    raw = pos = ms = None
    if sft:
        raw, ms = pipeline_mask(S, B, seed, greedy=False, front=FRONT, empty_rows=(B - 1,))
        raw = raw.reshape(B, S)
        pos = positions_from_mask(ms.reshape(B, S))
        lab[raw == 0] = -100
    return ids, lab, pos, raw, ms


def run_engine(cfg, B, S, monkeypatch, *, seed, fp32=False, sft=False, micro_batches=2, sabotage=None):
    """Two micro-batches of forward_loss + backward(grad_scale=0.5) under the checker.  sabotage(eng, ops, monkeypatch)
    installs a fault before the checker wraps the ops, so the checker sees the faulty function as the kernel."""
    from paddlenlp_b200 import ops as o
    from paddlenlp_b200.transformers.decoder_engine import DecoderEngine

    eng = DecoderEngine(cfg, device=DEV)
    eng.init_weights(seed)
    if eng.qkv_bias:
        for i in range(eng.L):
            eng.p[f"l{i}.qkv_b"].normal_(0, 0.02)
        eng.params_changed()
    if fp32:
        eng.set_master_grad(True)
    eng.flat_grads.fill_(NAN)                  # a view that is accumulated into instead of written shows up
    eng.clear_grad()
    geom = Geometry(cfg.num_hidden_layers, cfg.num_attention_heads, cfg.num_key_value_heads,
                    cfg.hidden_size // cfg.num_attention_heads, bool(cfg.tie_word_embeddings),
                    cfg.intermediate_size % 64 == 0, cfg.model_type == "qwen2", bool(cfg.recompute), pos=sft, mask=sft)
    if sabotage is not None:
        sabotage(eng, o, monkeypatch)
    chk = EngineChecker(eng, geom, monkeypatch)
    for mb in range(micro_batches):
        ids, lab, pos, raw, ms = make_batch(cfg, B, S, seed * 10 + mb, sft)
        chk.start(mb, S, ids.to(DEV).view(-1), lab.to(DEV).view(-1), None if pos is None else pos.to(DEV).int().view(-1),
                  None if ms is None else ms.to(DEV).int().contiguous(), 0.5)
        eng.forward_loss(ids.to(DEV), lab.to(DEV), position_ids=pos, attn_mask_startend_row_indices=raw)
        eng.backward(grad_scale=0.5)
        chk.finish()
    monkeypatch.undo()
    return eng, geom, chk


CASES = {                      # id: (family, preset, B, S, options)
    "llama3_2_1b": ("llama", "llama3_2_1b", 1, 4096, {}),
    "llama3_2_3b": ("llama", "llama3_2_3b", 1, 4096, {}),
    "llama3_8b": ("llama", "llama3_8b", 1, 4096, {}),
    "qwen2_0_5b": ("qwen2", "qwen2_0_5b", 2, 2048, {}),
    "qwen2_1_5b": ("qwen2", "qwen2_1_5b", 2, 2048, {}),
    "qwen2_7b": ("qwen2", "qwen2_7b", 2, 2048, {}),
    "llama3_2_3b-tied": ("llama", "llama3_2_3b", 1, 4096, dict(tie_word_embeddings=True)),
    "llama3_2_3b-recompute": ("llama", "llama3_2_3b", 1, 4096, dict(recompute=True)),
    "qwen2_0_5b-recompute": ("qwen2", "qwen2_0_5b", 2, 2048, dict(recompute=True)),
    "qwen2_1_5b-sft": ("qwen2", "qwen2_1_5b", 4, 2048, dict(sft=True)),
    "qwen2_1_5b-unfused_swiglu": ("qwen2", "qwen2_1_5b", 2, 2048, dict(intermediate_size=8968)),
    "qwen2_1_5b-fp32-untied": ("qwen2", "qwen2_1_5b", 4, 2048, dict(fp32=True)),
    "qwen2_1_5b-fp32-tied": ("qwen2", "qwen2_1_5b", 4, 2048, dict(fp32=True, tie_word_embeddings=True)),
    "llama3_2_1b-fp32": ("llama", "llama3_2_1b", 1, 4096, dict(fp32=True)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_engine_call_by_call(case, monkeypatch, fp64_reference):
    """Two decoder layers of the preset at its real vocabulary, two micro-batches (fresh, then accumulated): every op call
    checked against fp64 and against the schedule, exact call counts, every gradient view finite at the end."""
    family, preset, B, S, opt = CASES[case]
    opt = dict(opt)
    fp32, sft = opt.pop("fp32", False), opt.pop("sft", False)
    cfg = make_config(family, preset, 2, **opt)
    seed = 7 + list(CASES).index(case)
    eng, g, chk = run_engine(cfg, B, S, monkeypatch, seed=seed, fp32=fp32, sft=sft)
    if case.endswith("unfused_swiglu"):
        assert not g.fused
    per_mb = expected_counts(g.L, g.tied, g.fused, g.bias, g.recompute)
    print(f"\n[engine {case} L={g.L} B={B} S={S} tied={int(g.tied)} fused_swiglu={int(g.fused)} recompute={int(g.recompute)} "
          f"grads={'fp32' if fp32 else 'bf16'}] calls {dict(chk.count)} | worst err/bound "
          f"{ {k: round(v, 3) for k, v in chk.worst.items()} } | c_need {({k: f'{v:.2e}' for k, v in chk.c_need.items()})}")
    assert dict(chk.count) == {k: 2 * v for k, v in per_mb.items()}
    assert max(chk.worst.values()) <= 1.0
    for name, v in eng.g.items():
        assert bool(torch.isfinite(v).all()), f"gradient {name} not fully written"


# ----------------------------------------------------------------------------------------------------------
# GPU: the checker raises on a sabotaged step
# ----------------------------------------------------------------------------------------------------------
def _small(recompute=False):
    return make_config("qwen2", "qwen2_0_5b", 1, recompute=recompute)


def _wrap(o, monkeypatch, name, fn):
    orig = getattr(o, name)
    monkeypatch.setattr(o, name, lambda *a, **k: fn(orig, *a, **k))


def _no_accumulate(eng, o, monkeypatch):
    def gemm(orig, a, b, out=None, **kw):
        kw["accumulate"] = False                           # every dW GEMM of micro-batch 1 overwrites its gradient
        return orig(a, b, out=out, **kw)
    _wrap(o, monkeypatch, "gemm", gemm)


def _rope_forward_sign(eng, o, monkeypatch):
    def rope(orig, *a, backward=False, **k):
        return orig(*a, backward=False, **k)
    _wrap(o, monkeypatch, "rope_inplace", rope)


def _n1_for_n2(eng, o, monkeypatch):
    """The engine's saved activations with n1 in n2's place: the gate|up dW GEMM gets (n1, dgu), which the kernel computes
    correctly, so only the schedule can tell."""
    layer_bwd = eng._layer_bwd

    def swapped(i, dx2, saved, *a, **k):
        s = list(saved)                                    # (x, rstd1, n1, qkv, attn2, lse, x1, rstd2, n2, gu, m)
        s[8] = s[2]
        return layer_bwd(i, dx2, tuple(s), *a, **k)
    monkeypatch.setattr(eng, "_layer_bwd", swapped)


def _drop_token_row(eng, o, monkeypatch):
    def emb_bwd(orig, ids, dout, dtable):
        ids = ids.clone()
        uniq, counts = torch.unique(ids, return_counts=True)
        once = uniq[counts == 1]
        t = int(torch.isin(ids, once).nonzero()[0])        # a token whose row no other token adds to
        ids[t] = -1                                        # skipped by the scatter
        return orig(ids, dout, dtable)
    _wrap(o, monkeypatch, "embedding_bwd", emb_bwd)


def _perturb_recomputed_row(eng, o, monkeypatch):
    calls = [0]

    def rms(orig, x, w, eps, out=None, rstd=None):
        y, r = orig(x, w, eps, out=out, rstd=rstd)
        calls[0] += 1
        if calls[0] == 4:                                  # L = 1: ln1, ln2, final norm, then ln1 recomputed
            y.view(torch.int16)[5] += 1                    # one row one ulp off
        return y, r
    _wrap(o, monkeypatch, "rmsnorm_fwd", rms)


SABOTAGES = {
    "dW written on micro-batch 1": (_no_accumulate, False, "gemm"),
    "RoPE backward with the forward sign": (_rope_forward_sign, False, "rope_inplace"),
    "n1 where the gate|up dW expects n2": (_n1_for_n2, False, "l0.n2"),
    "one token row dropped from the embedding scatter": (_drop_token_row, False, "embedding_bwd"),
    "recomputed activation row one ulp off": (_perturb_recomputed_row, True, "recomputed l0.n1 is not bit-identical"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SABOTAGES))
def test_checker_catches_sabotage(name, monkeypatch, fp64_reference):
    """Qwen2-0.5B width, one layer, 1 x 1024 tokens: the checker raises on the sabotaged step, naming the op."""
    fn, recompute, match = SABOTAGES[name]
    with pytest.raises(AssertionError, match=match):
        run_engine(_small(recompute), 1, 1024, monkeypatch, seed=3, sabotage=fn)
