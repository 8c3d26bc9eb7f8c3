"""Micro-benchmarks of the decode-step kernels (CUDA events, L2-cold via a 256 MB flush between iterations)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import ops  # noqa: E402

dev = "cuda:0"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=20, cold=True):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        if cold:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters * 1e3   # us


def main():
    B, h, I, nh, kvh, d, V = 64, 4096, 14336, 32, 8, 128, 128256
    x = torch.randn(B, h, device=dev).to(torch.bfloat16)
    r = torch.randn(B, h, device=dev).to(torch.bfloat16)
    w = torch.ones(h, device=dev, dtype=torch.bfloat16)
    print(json.dumps(dict(op="add_rmsnorm[64x4096]", us=timeit(lambda: ops.add_rmsnorm(x, r, w, 1e-5)))))
    print(json.dumps(dict(op="rmsnorm_fwd[64x4096]", us=timeit(lambda: ops.rmsnorm_fwd(x, w, 1e-5)))))
    gu = torch.randn(B, 2 * I, device=dev).to(torch.bfloat16)
    print(json.dumps(dict(op="swiglu_fwd[64x14336]", us=timeit(lambda: ops.swiglu_fwd(gu)))))
    for name, K, N, tb in (("qkv", h, 6144, True), ("o", h, h, False), ("ffn1", h, 2 * I, False), ("ffn2", I, h, False), ("head", h, V, False)):
        a = torch.randn(B, K, device=dev).to(torch.bfloat16)
        wt = torch.randn((N, K) if tb else (K, N), device=dev).to(torch.bfloat16)
        for split in (0, 1):
            us = timeit(lambda: ops.gemm_skinny(a, wt, trans_b=tb, split_k=split))
            print(json.dumps(dict(op=f"gemm_skinny[{name} 64x{N}x{K}] split={split}", us=us, gbs=K * N * 2 / us / 1e3)))
        us = timeit(lambda: ops.gemm(a, wt, trans_b=tb))
        print(json.dumps(dict(op=f"gemm [{name}]", us=us, gbs=K * N * 2 / us / 1e3)))
    max_len = 2048
    cache = torch.randn(2, B, kvh, max_len, d, device=dev).to(torch.bfloat16)
    qkv = torch.randn(B, (nh + 2 * kvh) * d, device=dev).to(torch.bfloat16)
    for t in (128, 512, 1024, 2047):
        lens = torch.full((B,), t, dtype=torch.int32, device=dev)
        for impl, splits in (("simt", 0), ("tc", 0), ("tc", 1), ("tc", 2), ("tc", 4)):
            us = timeit(lambda: ops.decode_attention(qkv, cache, lens, nh, kvh, d, impl=impl, num_splits=splits))
            print(json.dumps(dict(op=f"decode_attention[{impl} splits={splits} t={t}]", us=us,
                                  gbs=2 * B * kvh * (t + 1) * d * 2 / us / 1e3)))
    cos, sin = ops.rope_tables(d, max_len, 500000.0, dev)
    lens = torch.full((B,), 100, dtype=torch.int32, device=dev)
    print(json.dumps(dict(op="decode_rope_append", us=timeit(lambda: ops.decode_rope_append(qkv, cache, cos, sin, lens, nh, kvh, d)))))


if __name__ == "__main__":
    main()
