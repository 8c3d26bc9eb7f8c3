"""Time the flash-attention forward/backward at the Llama-3-8B attention shape on an H100."""
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import ops  # noqa: E402


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


def main():
    dev = "cuda:0"
    for (B, S, nh, kvh) in [(1, 4096, 32, 8), (2, 4096, 32, 8), (1, 2048, 28, 4)]:
        d = 128
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
        t_f = timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out))
        t_b = timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv))
        fl_f = 4.0 * B * nh * S * S * d / 2        # causal
        fl_b = 2.5 * fl_f
        rec = dict(shape=[B, S, nh, kvh], fwd_ms=t_f, fwd_tflops=fl_f / t_f / 1e9, bwd_ms=t_b, bwd_tflops=fl_b / t_b / 1e9)
        try:
            from flash_attn import flash_attn_func

            qq, kk, vv = (t.contiguous().requires_grad_(True) for t in (q, k, v))
            t_ff = timeit(lambda: flash_attn_func(qq, kk, vv, causal=True))
            o2 = flash_attn_func(qq, kk, vv, causal=True)
            t_fb = timeit(lambda: torch.autograd.grad(o2, (qq, kk, vv), dout, retain_graph=True))
            rec.update(fa2_fwd_ms=t_ff, fa2_bwd_ms=t_fb, fa2_fwd_tflops=fl_f / t_ff / 1e9, fa2_bwd_tflops=fl_b / t_fb / 1e9)
        except Exception as e:  # library comparison only
            rec["fa2_error"] = str(e)[:200]
        print(json.dumps(rec), flush=True)
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
    t_f = timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out, mask_start=ms))
    t_b = timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, mask_start=ms))
    t_fc = timeit(lambda: ops.flash_attn_fwd(q, k, v, out=out))
    t_bc = timeit(lambda: ops.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv))
    fl = 4.0 * B * nh * useful * d / 2
    print(json.dumps(dict(flashmask_docs=docs, shape=[B, S, nh, kvh], fwd_ms=t_f, bwd_ms=t_b, plain_causal_fwd_ms=t_fc,
                          plain_causal_bwd_ms=t_bc, useful_fwd_tflops=fl / t_f / 1e9, useful_bwd_tflops=2.5 * fl / t_b / 1e9)), flush=True)


if __name__ == "__main__":
    main()
