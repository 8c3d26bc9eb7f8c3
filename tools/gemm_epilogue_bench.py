"""GEMM epilogue cost at the bench.py pre-training shapes (Llama-3.2-3B, one 4096-token micro-batch).

For every GEMM of the step whose epilogue reads or writes more than the output tile (accumulate into the gradient buffer,
residual add, gate|up + SwiGLU, down-proj dX + SwiGLU backward), time it against the plain GEMM (mode 0) at the same shape and
operand layout.  The extra bytes of the epilogue at 3.35 TB/s give the time it should add.  Each variant runs back to back
over rotating operand sets larger than L2; rounds alternate the variants; the median and the min-max spread of the per-call
times are printed with the card's name, power limit and SM clock.

    python tools/gemm_epilogue_bench.py [--rounds 5] [--iters 10] [--json OUT]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import ops  # noqa: E402

DEV = "cuda:0"
BF = torch.bfloat16
T, H, I, QKV, V = 4096, 3072, 8192, 5120, 128256
HBM = 3.35e12
L2_BYTES = 50 << 20


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def rnd(*shape, scale=0.05, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(BF)


def sets_for(nbytes):
    """Number of operand sets whose total exceeds twice the L2."""
    return max(1, -(-2 * L2_BYTES // nbytes))


def cases():
    """(name, build) where build() returns (real, plain, extra_bytes) callables taking an iteration index."""
    out = []

    def dw(name, M, N):   # weight gradient, accumulated: op(X^T) dY into G[M, N]
        def build():
            n = sets_for(2 * T * (M + N))
            xs = [rnd(T, M, seed=s) for s in range(n)]
            dys = [rnd(T, N, seed=100 + s) for s in range(n)]
            g = rnd(M, N, seed=7)
            real = lambda i: ops.gemm(xs[i % n], dys[i % n], g, trans_a=True, accumulate=True)
            plain = lambda i: ops.gemm(xs[i % n], dys[i % n], g, trans_a=True)
            return real, plain, 2 * M * N
        out.append((name, build))

    def res(name, K):     # forward projection + residual: [T, K] x [K, H] + R
        def build():
            n = sets_for(2 * T * (K + H))
            xs = [rnd(T, K, seed=s) for s in range(n)]
            rs = [rnd(T, H, seed=100 + s) for s in range(n)]
            w = rnd(K, H, seed=7)
            y = torch.empty(T, H, dtype=BF, device=DEV)
            real = lambda i: ops.gemm(xs[i % n], w, y, residual=rs[i % n])
            plain = lambda i: ops.gemm(xs[i % n], w, y)
            return real, plain, 2 * T * H
        out.append((name, build))

    res("o_proj_residual", H)
    res("down_proj_residual", I)

    def swiglu_fwd():
        n = sets_for(2 * T * H)
        xs = [rnd(T, H, seed=s) for s in range(n)]
        w = rnd(H, 2 * I, seed=7)
        gu = torch.empty(T, 2 * I, dtype=BF, device=DEV)
        m = torch.empty(T, I, dtype=BF, device=DEV)
        real = lambda i: ops.gemm_swiglu(xs[i % n], w, gu, m)
        plain = lambda i: ops.gemm(xs[i % n], w, gu)
        return real, plain, 2 * T * I
    out.append(("gate_up_swiglu", swiglu_fwd))

    def swiglu_bwd():
        n = sets_for(2 * T * (H + 2 * I))
        dys = [rnd(T, H, seed=s) for s in range(n)]
        gus = [rnd(T, 2 * I, scale=1.0, seed=100 + s) for s in range(n)]
        w = rnd(I, H, seed=7)
        dgu = torch.empty(T, 2 * I, dtype=BF, device=DEV)
        dm = torch.empty(T, I, dtype=BF, device=DEV)
        real = lambda i: ops.gemm_swiglu_bwd(dys[i % n], w, gus[i % n], dgu)
        plain = lambda i: ops.gemm(dys[i % n], w, dm, trans_b=True)
        return real, plain, 2 * T * 2 * I + (2 * T * 2 * I - 2 * T * I)   # reads gate|up, writes 2I columns instead of I
    out.append(("down_dx_swiglu_bwd", swiglu_bwd))

    def logits():         # the plain GEMM with the head dW's FLOPs, for comparison with dw_head
        n = sets_for(2 * T * H)
        xs = [rnd(T, H, seed=s) for s in range(n)]
        w = rnd(H, V, seed=7)
        y = torch.empty(T, V, dtype=BF, device=DEV)
        f = lambda i: ops.gemm(xs[i % n], w, y)
        return f, f, 0
    out.append(("logits_mode0", logits))

    dw("dw_qkv", H, QKV)
    dw("dw_o", H, H)
    dw("dw_gate_up", H, 2 * I)
    dw("dw_down", I, H)
    dw("dw_head", H, V)
    return out


def time_per_call(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print("card (name, power limit, SM clock, max SM clock):", card())
    rows = []
    for name, build in cases():
        real, plain, extra = build()
        for f in (real, plain):
            for i in range(3):
                f(i)
        torch.cuda.synchronize()
        tr, tp = [], []
        for _ in range(a.rounds):
            tr.append(time_per_call(real, a.iters))
            tp.append(time_per_call(plain, a.iters))
        mr, mp = statistics.median(tr), statistics.median(tp)
        budget = mp + extra / HBM * 1e3
        row = dict(gemm=name, ms=round(mr, 4), ms_range=[round(min(tr), 4), round(max(tr), 4)], mode0_ms=round(mp, 4),
                   mode0_range=[round(min(tp), 4), round(max(tp), 4)], extra_mb=round(extra / 1e6, 1),
                   mode0_plus_bytes_ms=round(budget, 4), over_budget_pct=round(100 * (mr / budget - 1), 2))
        rows.append(row)
        print(json.dumps(row), flush=True)
        del real, plain
        torch.cuda.empty_cache()
    print("card at the end:", card())
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
