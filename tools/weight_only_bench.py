"""The W8 GEMM (ops.weight_only_linear: int8 weights, per-channel scales) against the bf16 GEMM it replaces (ops.gemm_skinny,
the split-K kernel of the decode step, at M <= 128; ops.gemm above) at the Llama-3-8B and Llama-3.2-3B layer shapes.

Each kernel is timed as replays of a CUDA graph of `iters` calls, as the decode step runs it (an eager loop measures the
host's launch rate at these sizes).  Rounds alternate between the two kernels so that clock and neighbour drift hit both
alike.  Reports the time per call, the
achieved bytes/s over the bytes each kernel must move (weights + activations + output; the decode sizes are bound by them) and
TFLOP/s at M = 8192, with the card's name and power limit read in the same run.

    python tools/weight_only_bench.py [--rows 1 8 64 128 8192] [--rounds 5] [--iters 50]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import ops  # noqa: E402
from tools.serve_bench import card  # noqa: E402

MODELS = {"llama3-8b": dict(h=4096, nh=32, kvh=8, d=128, I=14336), "llama3.2-3b": dict(h=3072, nh=24, kvh=8, d=128, I=8192)}


def shapes(p):
    """(K, N) of qkv, o, ffn1 (gate|up) and ffn2 in [in, out] layout."""
    return {"qkv": (p["h"], (p["nh"] + 2 * p["kvh"]) * p["d"]), "o": (p["nh"] * p["d"], p["h"]), "ffn1": (p["h"], 2 * p["I"]),
            "ffn2": (p["I"], p["h"])}


def graph_of(fn, iters):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()                                     # warm-up outside capture: attributes, workspaces
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    return g


def timed(g, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1, 8, 64, 128, 8192])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    g = torch.Generator(device="cuda").manual_seed(0)
    results = []
    for model, p in MODELS.items():
        for name, (K, N) in shapes(p).items():
            w = (0.02 * torch.randn(K, N, generator=g, device="cuda")).to(torch.bfloat16)
            q, s = ops.weight_quantize(w)
            for M in a.rows:
                x = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
                out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
                w8 = lambda: ops.weight_only_linear(x, q, weight_scale=s, out=out)                       # noqa: E731
                if M <= ops.SKINNY_M:
                    bf = lambda: ops.gemm_skinny(x, w, out=out)                                           # noqa: E731
                else:
                    bf = lambda: ops.gemm(x, w, out=out)                                                  # noqa: E731
                g8, gb = graph_of(w8, a.iters), graph_of(bf, a.iters)
                t8, tb = [], []
                for _ in range(a.rounds):
                    t8.append(timed(g8, a.iters))
                    tb.append(timed(gb, a.iters))
                ms8, msb = min(t8), min(tb)
                act = M * K * 2 + M * N * 2
                r = dict(model=model, gemm=name, M=M, K=K, N=N, w8_us=ms8 * 1e3, bf16_us=msb * 1e3, speedup=msb / ms8,
                         w8_gbs=(N * K + N * 2 + act) / (ms8 / 1e3) / 1e9, bf16_gbs=(N * K * 2 + act) / (msb / 1e3) / 1e9,
                         w8_spread=max(t8) / ms8 - 1, bf16_spread=max(tb) / msb - 1)
                if M >= 4096:
                    r["w8_tflops"] = 2 * M * N * K / (ms8 / 1e3) / 1e12
                    r["bf16_tflops"] = 2 * M * N * K / (msb / 1e3) / 1e12
                results.append(r)
                print(json.dumps(r), flush=True)
                del g8, gb
            del w, q, s
    print(json.dumps(dict(card(), results=len(results))), flush=True)


if __name__ == "__main__":
    main()
