"""Where the wgmma GEMM's time goes at the bench.py pre-training shapes (Llama-3.2-3B, one 4096-token micro-batch).

1. A K sweep of the plain GEMM (mode 0) at M = 4096, N = 3072 and N = 16384, K = 1024 ... 16384, for the operand majors the step
   uses: forward (A K-major, B MN-major), dX (both K-major), dW (both MN-major; there M = 3072 and K is the token count).
   Every CTA of the persistent grid runs ceil(tiles / CTAs) tiles one after the other, so kernel time over that count is the
   time per tile.  A least-squares line  t_tile = a + b * k_blocks  gives the fixed cost per tile a (epilogue, pipeline fill,
   and the launch divided by the tiles per CTA) and the steady-state mainloop rate: SMs * 2 * 128 * 256 * 64 FLOP / b.
2. The GEMMs of one layer and of the head in the epilogue modes the step runs them in, time and TFLOP/s each, and their sum
   weighted by launches per step (28 layers x 8 micro-batches = 224, head 8): one number for the step's GEMM budget.

Each GEMM runs back to back over rotating operand sets larger than L2; rounds alternate the libraries; the median and the
min-max spread of the per-call times are printed with the card's name, power limit and SM clock at the start and the end.

    python tools/gemm_mainloop_bench.py [--baseline-lib [NAME=]OTHER/libb200nlp.so ...] [--rounds 5] [--iters 10] [--json OUT]

--baseline-lib (repeatable) loads another build of the library (for example the previous commit's) and times it alternately
with this tree's, round by round, in the same process.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
from ctypes import c_char_p, c_int

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import _lib  # noqa: E402

DEV = "cuda:0"
BF = torch.bfloat16
T, H, I, QKV, V = 4096, 3072, 8192, 5120, 128256
LAYER_LAUNCHES, HEAD_LAUNCHES = 28 * 8, 8
L2_BYTES = 50 << 20
BM, BN, BK = 128, 256, 64


class Lib:
    """The three GEMM entry points of one build of libb200nlp.so, called on torch tensors."""

    def __init__(self, path):
        self.lib = ctypes.CDLL(path)
        for name in ("b200_gemm_bf16_ex", "b200_gemm_swiglu_bf16", "b200_gemm_swiglu_bwd_bf16"):
            fn = getattr(self.lib, name)
            fn.argtypes = _lib._SIGNATURES[name]
            fn.restype = c_int
        self.lib.b200_last_error.restype = c_char_p

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"rc={rc}: {self.lib.b200_last_error().decode()}")

    def gemm(self, a, b, out, trans_a=False, trans_b=False, accumulate=False, residual=None):
        K, M = a.shape if trans_a else a.shape[::-1]
        N = b.shape[0] if trans_b else b.shape[1]
        self._check(self.lib.b200_gemm_bf16_ex(
            _lib.ptr(a), _lib.ptr(b), _lib.ptr(out), None, _lib.ptr(residual), M, N, K, a.stride(0), b.stride(0), out.stride(0),
            residual.stride(0) if residual is not None else 0, int(trans_a), int(not trans_b), int(accumulate), 0,
            _lib.stream_ptr()))

    def gemm_swiglu(self, x, w, gu, m):
        M, K = x.shape
        self._check(self.lib.b200_gemm_swiglu_bf16(_lib.ptr(x), _lib.ptr(w), _lib.ptr(gu), _lib.ptr(m), M, m.shape[1], K,
                                                   x.stride(0), w.stride(0), gu.stride(0), m.stride(0), _lib.stream_ptr()))

    def gemm_swiglu_bwd(self, dy, w, gu, dgu):
        M, K = dy.shape
        self._check(self.lib.b200_gemm_swiglu_bwd_bf16(_lib.ptr(dy), _lib.ptr(w), _lib.ptr(gu), _lib.ptr(dgu), M, w.shape[0], K,
                                                       dy.stride(0), w.stride(0), gu.stride(0), dgu.stride(0), _lib.stream_ptr()))


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
    return max(2, -(-2 * L2_BYTES // nbytes))


def plain(M, N, K, trans_a, trans_b):
    """call(lib, i) for the mode-0 GEMM over rotating operands."""
    n = sets_for(2 * K * (M + N))
    a = [rnd(*((K, M) if trans_a else (M, K)), seed=s) for s in range(n)]
    b = [rnd(*((N, K) if trans_b else (K, N)), seed=100 + s) for s in range(n)]
    out = torch.empty(M, N, dtype=BF, device=DEV)
    return lambda lib, i: lib.gemm(a[i % n], b[i % n], out, trans_a, trans_b)


def step_gemms():
    """(name, launches per step, FLOPs, build) of the step's GEMMs; build() returns call(lib, i)."""
    out = []

    def add(name, launches, M, N, K, build):
        out.append((name, launches, 2.0 * M * N * K, build))

    def fwd(name, launches, N, K, residual):      # [T, K] x [K, N] (+ residual)
        def build():
            n = sets_for(2 * T * (K + N))
            xs = [rnd(T, K, seed=s) for s in range(n)]
            rs = [rnd(T, N, seed=100 + s) for s in range(n)] if residual else None
            w = rnd(K, N, seed=7)
            y = torch.empty(T, N, dtype=BF, device=DEV)
            return lambda lib, i: lib.gemm(xs[i % n], w, y, residual=rs[i % n] if residual else None)
        add(name, launches, T, N, K, build)

    def dx(name, launches, N, K):                 # dY [T, K] x W[N, K]^T
        def build():
            n = sets_for(2 * T * K)
            dys = [rnd(T, K, seed=s) for s in range(n)]
            w = rnd(N, K, seed=7)
            y = torch.empty(T, N, dtype=BF, device=DEV)
            return lambda lib, i: lib.gemm(dys[i % n], w, y, trans_b=True)
        add(name, launches, T, N, K, build)

    def dw(name, launches, M, N):                 # G[M, N] += X[T, M]^T dY[T, N]
        def build():
            n = sets_for(2 * T * (M + N))
            xs = [rnd(T, M, seed=s) for s in range(n)]
            dys = [rnd(T, N, seed=100 + s) for s in range(n)]
            g = rnd(M, N, seed=7)
            return lambda lib, i: lib.gemm(xs[i % n], dys[i % n], g, trans_a=True, accumulate=True)
        add(name, launches, M, N, T, build)

    def swiglu_fwd():
        n = sets_for(2 * T * H)
        xs = [rnd(T, H, seed=s) for s in range(n)]
        w = rnd(H, 2 * I, seed=7)
        gu = torch.empty(T, 2 * I, dtype=BF, device=DEV)
        m = torch.empty(T, I, dtype=BF, device=DEV)
        return lambda lib, i: lib.gemm_swiglu(xs[i % n], w, gu, m)

    def swiglu_bwd():
        n = sets_for(2 * T * (H + 2 * I))
        dys = [rnd(T, H, seed=s) for s in range(n)]
        gus = [rnd(T, 2 * I, scale=1.0, seed=100 + s) for s in range(n)]
        w = rnd(I, H, seed=7)
        dgu = torch.empty(T, 2 * I, dtype=BF, device=DEV)
        return lambda lib, i: lib.gemm_swiglu_bwd(dys[i % n], w, gus[i % n], dgu)

    L, HD = LAYER_LAUNCHES, HEAD_LAUNCHES
    fwd("qkv", L, QKV, H, False)
    fwd("o + residual", L, H, H, True)
    add("gate|up + SwiGLU", L, T, 2 * I, H, swiglu_fwd)
    fwd("down + residual", L, H, I, True)
    fwd("head (logits)", HD, V, H, False)
    dx("dX head", HD, H, V)
    dx("dX qkv", L, H, QKV)
    dx("dX o", L, H, H)
    dx("dX gate|up", L, H, 2 * I)
    add("dX down + SwiGLU backward", L, T, I, H, swiglu_bwd)
    dw("dW qkv", L, H, QKV)
    dw("dW o", L, H, H)
    dw("dW gate|up", L, H, 2 * I)
    dw("dW down", L, I, H)
    dw("dW head", HD, H, V)
    return out


def time_per_call(fn, lib, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(lib, i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(fn, libs, rounds, iters):
    """{lib name: (median ms, min, max)}; rounds alternate the libraries."""
    for lib in libs.values():
        for i in range(3):
            fn(lib, i)
    torch.cuda.synchronize()
    ts = {k: [] for k in libs}
    for _ in range(rounds):
        for k, lib in libs.items():
            ts[k].append(time_per_call(fn, lib, iters))
    return {k: (statistics.median(v), min(v), max(v)) for k, v in ts.items()}


def fit(kbs, ts):
    """Least-squares t = a + b * kb."""
    n = len(kbs)
    mx, my = sum(kbs) / n, sum(ts) / n
    b = sum((x - mx) * (y - my) for x, y in zip(kbs, ts)) / sum((x - mx) ** 2 for x in kbs)
    return my - b * mx, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", action="append", default=[])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    libs = {"tree": Lib(_lib.LIB_PATH)}
    for i, spec in enumerate(a.baseline_lib):
        name, _, path = spec.rpartition("=")
        libs[name or ("baseline" if i == 0 else f"baseline{i}")] = Lib(os.path.abspath(path))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    result = dict(card_start=card(), sms=sms, sweep=[], step=[])
    print("card (name, power limit, SM clock, max SM clock):", result["card_start"], flush=True)

    # 1. K sweep
    ks = [1024, 2048, 4096, 8192, 16384]
    for major, M, ta, tb in (("forward (A K-major, B MN-major)", T, False, False), ("dX (A K-major, B K-major)", T, False, True),
                             ("dW (A MN-major, B MN-major)", H, True, False)):
        for N in (3072, 16384):
            tiles = (M // BM) * (N // BN)
            per_cta = -(-tiles // sms)
            t_tile = {k: [] for k in libs}
            spread = {k: 0.0 for k in libs}
            for K in ks:
                fn = plain(M, N, K, ta, tb)
                r = measure(fn, libs, a.rounds, a.iters)
                for k in libs:
                    t_tile[k].append(r[k][0] * 1e3 / per_cta)
                    spread[k] = max(spread[k], (r[k][2] - r[k][1]) / r[k][0])
                del fn
                torch.cuda.empty_cache()
            for k in libs:
                ic, sl = fit([K // BK for K in ks], t_tile[k])
                row = dict(lib=k, sweep=major, M=M, N=N, tiles=tiles, tiles_per_cta=per_cta, K=ks,
                           us_per_tile=[round(t, 3) for t in t_tile[k]], intercept_us=round(ic, 3),
                           intercept_kblocks=round(ic / sl, 2), us_per_kblock=round(sl, 4),
                           slope_tflops=round(sms * 2.0 * BM * BN * BK / sl / 1e6, 1), max_spread_pct=round(100 * spread[k], 2))
                result["sweep"].append(row)
                print(json.dumps(row), flush=True)

    # 2. the step's GEMMs
    total = {k: 0.0 for k in libs}
    for name, launches, flops, build in step_gemms():
        fn = build()
        r = measure(fn, libs, a.rounds, a.iters)
        for k in libs:
            med, lo, hi = r[k]
            total[k] += med * launches
            row = dict(lib=k, gemm=name, launches=launches, ms=round(med, 4), ms_range=[round(lo, 4), round(hi, 4)],
                       tflops=round(flops / med / 1e9, 1))
            result["step"].append(row)
            print(json.dumps(row), flush=True)
        del fn
        torch.cuda.empty_cache()
    result["step_gemm_ms"] = {k: round(v, 1) for k, v in total.items()}
    print("GEMM time per step, sum of median x launches (ms):", json.dumps(result["step_gemm_ms"]), flush=True)
    result["card_end"] = card()
    print("card at the end:", result["card_end"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
