"""The data-parallel gradient exchange on the GPU.

DataParallel all-reduces the flat gradient buffer range by range on a side stream while the last micro-batch's backward is
still running: DecoderEngine.backward reports each range through grad_ready_hook(lo, hi) the moment flat_grads[lo:hi] is
final.  Single-process training never arms the hook, and a range reported one op too early would have every rank
all-reduce a partial gradient.

A. One process: a recorder on grad_ready_hook clones flat_grads[lo:hi] on the current stream at each report, so the copy
   holds the bits at that point of the stream.  After backward every copy must equal the final bits of its range, and the
   ranges must tile the buffer in the order head (untied only), layer L-1 ... 0, embedding, norm/bias tail.  The gradient
   buffer is NaN before the first micro-batch.  Cases: two layers of every preset at its real vocabulary
   (test_engine_call_by_call_gpu.CASES: tied and untied, Qwen2's q/k/v bias, recompute, unfused SwiGLU, SFT start rows with
   position_ids, fp32 gradients), with the hook armed on a fresh micro-batch and on micro-batch 2 of 2 (accumulating).
   Sabotage tests move a report before the op that finishes its range and require the check to name that range.

B. Two ranks on one GPU over gloo, and C. the same over NCCL with one GPU per rank: tests/data_parallel_worker.py (its
   docstring lists the checks).  The ranks run under torch.distributed.run in a session of their own, which is killed
   whole when the run ends, fails or times out.
"""
import json
import math
import os
import signal
import socket
import subprocess
import sys

import pytest
import torch

from test_engine_call_by_call_gpu import CASES, make_batch, make_config, same_bits

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ----------------------------------------------------------------------------------------------------------
# A. every reported range is final
# ----------------------------------------------------------------------------------------------------------
def _align8(n):
    return (n + 7) // 8 * 8


def expected_ranges(eng):
    """[(name, lo, hi)] in report order, from the layout: head, l{L-1} .. l0 (a layer's four matrices), embed, tail."""
    def span(first, last):
        o, shp = eng._offsets[last]
        return eng._offsets[first][0], o + _align8(math.prod(shp))

    out = [] if eng.tied else [("head",) + span("head", "head")]
    out += [(f"l{i}",) + span(f"l{i}.qkv_w", f"l{i}.down_w") for i in reversed(range(eng.L))]
    out += [("embed",) + span("embed", "embed"), ("tail", eng.decay_end, eng.numel)]
    return out


class Recorder:
    """grad_ready_hook that clones the reported range on the current stream."""

    def __init__(self, eng):
        self.eng, self.calls = eng, []

    def __call__(self, lo, hi):
        self.calls.append((lo, hi, self.eng.flat_grads[lo:hi].clone()))


def check_ranges(eng, rec):
    torch.cuda.synchronize()
    assert eng.grad_ready_hook is None, "the hook is still armed after backward"
    want = expected_ranges(eng)
    names = {(lo, hi): n for n, lo, hi in want}
    for lo, hi, snap in rec.calls:
        fin = eng.flat_grads[lo:hi]
        if not same_bits(snap, fin):
            iv = torch.int32 if fin.element_size() == 4 else torch.int16
            n = int((snap.view(iv) != fin.view(iv)).sum())
            raise AssertionError(f"range {names.get((lo, hi), '?')} [{lo}, {hi}) was reported before it was final: "
                                 f"{n} of {hi - lo} elements changed after the report")
    got = [(lo, hi) for lo, hi, _ in rec.calls]
    assert got == [(lo, hi) for _, lo, hi in want], \
        f"reported {[names.get(r, r) for r in got]}, expected {[n for n, _, _ in want]}"
    pos = 0
    for lo, hi in sorted(got):
        assert lo == pos and hi > lo, f"ranges do not tile the buffer at {pos}: {sorted(got)}"
        pos = hi
    assert pos == eng.numel
    return [names[r] for r in got]


def build_engine(cfg, seed, fp32):
    from paddlenlp_b200.transformers.decoder_engine import DecoderEngine

    eng = DecoderEngine(cfg, device=DEV)
    eng.init_weights(seed)
    if eng.qkv_bias:
        for i in range(eng.L):
            eng.p[f"l{i}.qkv_b"].normal_(0, 0.02)
        eng.params_changed()
    if fp32:
        eng.set_master_grad(True)
    return eng


def hooked_step(eng, cfg, B, S, seed, sft, micro_batches):
    """NaN gradients, then `micro_batches` forward_loss + backward(grad_scale=1/micro_batches); the hook is armed for the
    last one only, as DataParallel does outside no_sync()."""
    eng.flat_grads.fill_(float("nan"))
    eng.clear_grad()
    rec = Recorder(eng)
    for mb in range(micro_batches):
        ids, lab, pos, raw, _ = make_batch(cfg, B, S, seed * 10 + mb, sft)
        eng.forward_loss(ids.to(DEV), lab.to(DEV), position_ids=pos, attn_mask_startend_row_indices=raw)
        if mb == micro_batches - 1:
            eng.grad_ready_hook = rec
        eng.backward(grad_scale=1.0 / micro_batches)
    return rec


@pytest.mark.parametrize("case", list(CASES))
def test_reported_ranges_are_final(case):
    family, preset, B, S, opt = CASES[case]
    opt = dict(opt)
    fp32, sft = opt.pop("fp32", False), opt.pop("sft", False)
    cfg = make_config(family, preset, 2, **opt)
    seed = 31 + list(CASES).index(case)
    eng = build_engine(cfg, seed, fp32)
    for mbs in (1, 2):
        rec = hooked_step(eng, cfg, B, S, seed, sft, mbs)
        order = check_ranges(eng, rec)
        assert all(bool(torch.isfinite(s).all()) for _, _, s in rec.calls), "a reported range holds unwritten elements"
        print(f"\n[ranges {case} {'fresh' if mbs == 1 else 'micro-batch 2 of 2'} grads={'fp32' if fp32 else 'bf16'}] "
              f"{len(order)} ranges final when reported, tiling {eng.numel} elements: {', '.join(order)}")


def _layer_early(eng, rec, monkeypatch):
    layer_bwd = eng._layer_bwd

    def early(i, *a, **k):
        rec(*eng._range(f"l{i}.qkv_w", f"l{i}.down_w"))
        return layer_bwd(i, *a, **k)
    monkeypatch.setattr(eng, "_layer_bwd", early)


def _head_early(eng, rec, monkeypatch):
    from paddlenlp_b200 import ops as o

    gemm = o.gemm

    def early(a, b, out=None, **k):
        if out is not None and out.data_ptr() == eng.g["head"].data_ptr():
            rec(*eng._range("head", "head"))
        return gemm(a, b, out=out, **k)
    monkeypatch.setattr(o, "gemm", early)


def _embed_early(eng, rec, monkeypatch):
    from paddlenlp_b200 import ops as o

    emb_bwd = o.embedding_bwd

    def early(ids, dout, dtable):
        rec(*eng._range("embed", "embed"))
        return emb_bwd(ids, dout, dtable)
    monkeypatch.setattr(o, "embedding_bwd", early)


RANGE_SABOTAGES = {                 # name: (fault, tied, message)
    "each layer reported before its _layer_bwd": (_layer_early, False, r"range l1 \["),
    "head reported before the head dW GEMM": (_head_early, False, r"range head \["),
    "tied embed reported before embedding_bwd": (_embed_early, True, r"range embed \["),
}


@pytest.mark.parametrize("name", list(RANGE_SABOTAGES))
@pytest.mark.parametrize("micro_batches", [1, 2])
def test_range_check_catches_early_reports(name, micro_batches, monkeypatch):
    """Qwen2-0.5B width, two layers, 1 x 1024 tokens: a report moved before the op that finishes its range fails the check,
    which names the range."""
    fault, tied, match = RANGE_SABOTAGES[name]
    cfg = make_config("qwen2", "qwen2_0_5b", 2, tie_word_embeddings=tied)
    eng = build_engine(cfg, 5, False)
    rec = Recorder(eng)
    fault(eng, rec, monkeypatch)
    eng.flat_grads.fill_(float("nan"))
    eng.clear_grad()
    for mb in range(micro_batches):
        ids, lab, _, _, _ = make_batch(cfg, 1, 1024, 50 + mb, False)
        eng.forward_loss(ids.to(DEV), lab.to(DEV))
        rec.calls.clear()                           # the fault reports in every backward; only the hooked one counts
        if mb == micro_batches - 1:
            eng.grad_ready_hook = rec
        eng.backward(grad_scale=1.0 / micro_batches)
    with pytest.raises(AssertionError, match=match):
        check_ranges(eng, rec)


# ----------------------------------------------------------------------------------------------------------
# B / C. two ranks
# ----------------------------------------------------------------------------------------------------------
def free_port():
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def launch(backend, out_dir, sabotage, timeout=600):
    """Both ranks of tests/data_parallel_worker.py under torch.distributed.run, in a new session: whatever happens, the
    whole process group is killed before this returns, so no rank outlives the test."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(HERE, "data_parallel_worker.py"), "--backend", backend,
           "--out", str(out_dir)] + (["--sabotage"] if sabotage else [])
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PYTHONUNBUFFERED="1")
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, cwd=ROOT,
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out, _ = p.communicate()
        raise AssertionError(f"the two ranks did not finish in {timeout} s:\n{out[-6000:]}")
    finally:
        try:
            os.killpg(p.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    return p.returncode, out


def run_two_ranks(backend, tmp_path, sabotage):
    rc, out = launch(backend, tmp_path, sabotage)
    reports = [json.loads(ln.split(" ", 1)[1]) for ln in out.splitlines() if ln.startswith("DPREPORT ")]
    for r in reports:
        print(f"\n[{backend}] " + json.dumps(r))
    assert rc == 0, out[-8000:]
    parts = [r["part"] for r in reports]
    assert parts[0] == "start" and parts[-1] == "done", parts
    engine = [r for r in reports if r["part"] == "engine"]
    assert len(engine) == 6 and all(r["reduce_calls"] >= (2 if r["overlap"] else 1) for r in engine)
    assert all(r["reduce_calls"] == 1 for r in engine if not r["overlap"])
    assert len([r for r in reports if r["part"] == "trainer"]) == 3
    if sabotage:
        caught = {r["name"] for r in reports if r["part"] == "sabotage"}
        assert caught == {"sync_gradients reduces the whole buffer again", "hook armed under no_sync",
                          "grad_scale left at 1"}, caught
    return reports


def test_two_ranks_gloo_one_gpu(tmp_path):
    """Both ranks on cuda:0, gloo all-reducing the CUDA gradient buffer; with the worker's sabotage runs."""
    run_two_ranks("gloo", tmp_path, sabotage=True)


def test_two_ranks_nccl(tmp_path):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"NCCL needs one GPU per rank: {n} visible, 2 needed (the gloo test covers two ranks on one GPU)")
    run_two_ranks("nccl", tmp_path, sabotage=False)
