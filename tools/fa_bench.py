"""Time both flash-attention forward kernels (b200_set_fa_fwd_impl 2 = wgmma, 1 = mma.sync) and both backward kernels
(b200_set_fa_bwd_impl, the same numbering) on an H100.

Shapes (B, S, q heads, kv heads, head_dim): the two benchmarked models, Llama-3.2-3B (1 x 4096, 24 / 8 heads) and the
Qwen2-1.5B SFT micro-batch (4 x 2048, 12 / 2 heads), then the Llama-3-8B and Qwen2-7B layouts, all at head_dim 128; then the
head_dim 64 models: Llama-3.2-1B (1 x 4096, 32 / 8), a Qwen2-0.5B SFT micro-batch (4 x 2048, 14 / 2) and TinyLlama
(1 x 2048, 32 / 4).  The four kernels are timed alternately in one process (REPEATS rounds each), so clock and neighbour
drift hit all alike; each line gives the median and the spread (min, max), and the impl 1 / impl 2 time ratio of the forward
and of the backward.
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import _lib, ops  # noqa: E402

REPEATS = 5
SHAPES = [(1, 4096, 24, 8, 128), (4, 2048, 12, 2, 128), (1, 4096, 32, 8, 128), (2, 4096, 32, 8, 128), (1, 2048, 28, 4, 128),
          (1, 4096, 32, 8, 64), (4, 2048, 14, 2, 64), (1, 2048, 32, 4, 64)]


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.splitlines()[0].split(",")))) if r.returncode == 0 else {}


def summary(ts):
    return dict(median_ms=statistics.median(ts), min_ms=min(ts), max_ms=max(ts))


def main():
    dev = "cuda:0"
    lib = _lib.load()
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    old_fwd = lib.b200_set_fa_fwd_impl(2)
    old_impl = lib.b200_set_fa_bwd_impl(2)
    for (B, S, nh, kvh, d) in SHAPES:
        ld = (nh + 2 * kvh) * d
        qkv = torch.randn(B, S, ld, device=dev).to(torch.bfloat16)
        q = qkv[:, :, : nh * d].view(B, S, nh, d)
        k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
        v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
        out, lse = ops.flash_attn_fwd(q, k, v)
        dout = torch.randn_like(out)
        dqkv = torch.empty_like(qkv)
        dq = dqkv[:, :, : nh * d].view(B, S, nh, d)
        dk = dqkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
        dv = dqkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
        t_f = {1: [], 2: []}
        t_b = {1: [], 2: []}
        for _ in range(REPEATS):
            for impl in (2, 1):
                lib.b200_set_fa_fwd_impl(impl)
                t_f[impl].append(timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out)))
            lib.b200_set_fa_fwd_impl(2)
            for impl in (2, 1):
                lib.b200_set_fa_bwd_impl(impl)
                t_b[impl].append(timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv)))
        lib.b200_set_fa_bwd_impl(2)
        fl_f = 4.0 * B * nh * S * S * d / 2        # causal
        fl_b = 2.5 * fl_f
        rec = dict(shape=[B, S, nh, kvh], head_dim=d)
        for kind, ts, fl in (("fwd", t_f, fl_f), ("bwd", t_b, fl_b)):
            for impl in (2, 1):
                sm = summary(ts[impl])
                rec[f"{kind}_impl{impl}"] = dict(sm, tflops=fl / sm["median_ms"] / 1e9)
            rec[f"{kind}_impl1_over_impl2"] = rec[f"{kind}_impl1"]["median_ms"] / rec[f"{kind}_impl2"]["median_ms"]
        print(json.dumps(rec), flush=True)
    lib.b200_set_fa_bwd_impl(old_impl)
    # FlashMask (packed samples): Qwen2-7B SFT row of 2048 tokens holding documents of 700 / 900 / 448 tokens; useful flops only
    B, S, nh, kvh, d = 4, 2048, 28, 4, 128
    docs = [700, 900, 448]
    ms = torch.empty(S, dtype=torch.int32)
    pos, useful = 0, 0
    for n in docs:
        ms[pos:pos + n] = pos + n
        pos += n
        useful += n * n
    ms = ms[None].expand(B, S).contiguous().to(dev)
    ld = (nh + 2 * kvh) * d
    qkv = torch.randn(B, S, ld, device=dev).to(torch.bfloat16)
    q = qkv[:, :, : nh * d].view(B, S, nh, d)
    k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    out, lse = ops.flash_attn_fwd(q, k, v, mask_start=ms)
    dout = torch.randn_like(out)
    dq, dk, dv = torch.empty_like(out), torch.empty(B, S, kvh, d, device=dev, dtype=torch.bfloat16), torch.empty(B, S, kvh, d, device=dev, dtype=torch.bfloat16)
    t_f = {1: [], 2: []}
    for _ in range(REPEATS):
        for impl in (2, 1):
            lib.b200_set_fa_fwd_impl(impl)
            t_f[impl].append(timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out, mask_start=ms)))
    lib.b200_set_fa_fwd_impl(2)
    t_b = timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, mask_start=ms))
    t_fc = timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out))
    t_bc = timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv))
    fl = 4.0 * B * nh * useful * d / 2
    rec = dict(flashmask_docs=docs, shape=[B, S, nh, kvh])
    for impl in (2, 1):
        sm = summary(t_f[impl])
        rec[f"fwd_impl{impl}"] = dict(sm, useful_tflops=fl / sm["median_ms"] / 1e9)
    rec["fwd_impl1_over_impl2"] = rec["fwd_impl1"]["median_ms"] / rec["fwd_impl2"]["median_ms"]
    rec.update(bwd_ms=t_b, plain_causal_fwd_ms=t_fc, plain_causal_bwd_ms=t_bc, useful_bwd_tflops=2.5 * fl / t_b / 1e9)
    print(json.dumps(rec), flush=True)
    lib.b200_set_fa_fwd_impl(old_fwd)


if __name__ == "__main__":
    main()
