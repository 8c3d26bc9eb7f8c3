"""bf16 against fp32 gradients (amp_master_grad) on an H100, in one process.

1. The weight-gradient GEMMs of one Llama-3.2-3B layer (T = 4096 tokens of one micro-batch, h = 3072, I = 8192, GQA 24/8) and
   of the untied head (h x V, V = 128 256), each in bf16 and in fp32 output, overwrite and accumulate:
       bf16 accumulate   C = bf16(C_old + acc)       (reads and writes 2 B per element)
       fp32 accumulate   C += acc by TMA reduce-add  (reads and writes 4 B per element, in L2)
   The forms alternate over ROUNDS rounds; median and (min, max) in ms per call.
2. grad_sqnorm and AdamW over the whole model's flat buffers with bf16 and with fp32 gradients.
3. The Llama-3.2-3B pre-training step of bench.py (8 x 4096 tokens per step, micro-batch 1, clip + AdamW), bf16 and fp32
   gradients alternating over STEP_ROUNDS rounds (a fresh model per round): tokens/s, step ms and max_memory_allocated.
4. The GPU name, power limit and SM clock, before and after.

    python tools/master_grad_bench.py [--rounds N] [--step-rounds N] [--steps K] [--warmup W] [--tied] [--out FILE]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200 import _lib, ops  # noqa: E402

BF16, F32 = torch.bfloat16, torch.float32
T_TOK, V, H, I, QKV = 4096, 128256, 3072, 8192, (24 + 2 * 8) * 128
SEQ, PER_GPU_BATCH = 4096, 8


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.splitlines()[0].split(",")))) if r.returncode == 0 else {}


def timeit(fn, iters, warm=3):
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


def summary(ts):
    return dict(median=statistics.median(ts), min=min(ts), max=max(ts))


def gemms(rounds):
    """dW = X^T dY for each weight of one layer and the untied head: [K = T, M] x [K = T, N] -> [M, N]."""
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * s).to(BF16)

    shapes = {"qkv": (H, QKV), "o": (H, H), "gate_up": (H, 2 * I), "down": (I, H), "head": (H, V)}
    res = {}
    for name, (M, N) in shapes.items():
        x, dy = rnd(T_TOK, M), rnd(T_TOK, N, s=1e-2)
        c16, c32 = torch.zeros(M, N, dtype=BF16, device=dev), torch.zeros(M, N, dtype=F32, device=dev)
        forms = {
            "bf16_overwrite": lambda: ops.gemm(x, dy, out=c16, trans_a=True),
            "fp32_overwrite": lambda: ops.gemm(x, dy, out=c32, trans_a=True),
            "bf16_accumulate": lambda: ops.gemm(x, dy, out=c16, trans_a=True, accumulate=True),
            "fp32_accumulate": lambda: ops.gemm(x, dy, out=c32, trans_a=True, accumulate=True),
        }
        ts = {k: [] for k in forms}
        iters = 5 if name == "head" else 20
        for _ in range(rounds):
            for k, fn in forms.items():
                ts[k].append(timeit(fn, iters))
        res[name] = {k + "_ms": summary(v) for k, v in ts.items()}
        res[name]["tflops_fp32_accumulate"] = 2 * T_TOK * M * N / (res[name]["fp32_accumulate_ms"]["median"] * 1e9)
        res[name]["fp32_over_bf16_accumulate"] = (res[name]["fp32_accumulate_ms"]["median"] /
                                                  res[name]["bf16_accumulate_ms"]["median"])
        print(json.dumps({"gemm": name, "M": M, "N": N, "K": T_TOK, **res[name]}), flush=True)
        del x, dy, c16, c32
        torch.cuda.empty_cache()
    return res


def optimizer(rounds, n):
    """grad_sqnorm + AdamW over n elements, bf16 and fp32 gradients."""
    dev = "cuda:0"
    p = torch.zeros(n, dtype=BF16, device=dev)
    master, m, v = (torch.zeros(n, dtype=F32, device=dev) for _ in range(3))
    sq = torch.zeros(1, dtype=F32, device=dev)
    res = {}
    for gdt in (BF16, F32):
        grads = torch.full((n,), 1e-3, dtype=gdt, device=dev)
        ts_sq, ts_ad = [], []
        for _ in range(rounds):
            ts_sq.append(timeit(lambda: ops.grad_sqnorm(grads, out=sq), 10))
            ts_ad.append(timeit(lambda: ops.adamw_step(p, grads, master, m, v, sq, decay_end=n, lr=1e-5, beta1=0.9,
                                                       beta2=0.999, eps=1e-8, weight_decay=0.01, step=1), 10))
        key = "bf16" if gdt == BF16 else "fp32"
        res[key] = dict(sqnorm_ms=summary(ts_sq), adamw_ms=summary(ts_ad))
        del grads
        torch.cuda.empty_cache()
    print(json.dumps({"optimizer": res, "elements": n}), flush=True)
    del p, master, m, v
    torch.cuda.empty_cache()
    return res


def pretrain_step(master_grad, tied, steps, warmup):
    """bench.py's resident step (data already on the device) for a fresh Llama-3.2-3B.
    Returns (tokens/s, step ms, peak allocated GiB, parameters)."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.optimizer import AdamW, ClipGradByGlobalNorm, LinearAnnealingWithWarmupDecay

    dev = torch.device("cuda", 0)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = T.LlamaForCausalLM(T.LlamaConfig.llama3_2_3b(tie_word_embeddings=tied))
    if master_grad:
        model.set_master_grad(True)
    eng = model.engine
    sched = LinearAnnealingWithWarmupDecay(3e-5, 3e-6, warmup_step=30, decay_step=10000)
    opt = AdamW(learning_rate=sched.get_lr, beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.01,
                grad_clip=ClipGradByGlobalNorm(1.0), multi_precision=True, engine=eng)
    g = torch.Generator().manual_seed(1234)
    tok = torch.randint(0, eng.V, (warmup + steps, PER_GPU_BATCH, SEQ + 1), generator=g)
    ids, lab = tok[:, :, :-1].contiguous().to(dev), tok[:, :, 1:].contiguous().to(dev)
    del tok

    def step(i):
        for mb in range(PER_GPU_BATCH):
            eng.forward_loss(ids[i, mb:mb + 1], lab[i, mb:mb + 1])
            eng.backward(1.0 / PER_GPU_BATCH)
        opt.step(); sched.step(); opt.clear_grad()

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    nparam = eng.num_parameters()
    assert eng.flat_grads.dtype == (F32 if master_grad else BF16)
    del model, eng, opt, ids, lab
    gc.collect()
    torch.cuda.empty_cache()
    return PER_GPU_BATCH * SEQ / (ms / 1e3), ms, peak, nparam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the GEMM and optimizer timings")
    ap.add_argument("--step-rounds", type=int, default=2, help="alternating rounds of the pre-training step")
    ap.add_argument("--steps", type=int, default=3, help="timed steps per round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tied", action="store_true", help="tie the input and output embeddings (the released layout)")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _lib.call("b200_device_check")
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    res = dict(gpu=info, gemm=gemms(args.rounds))
    import paddlenlp_b200.transformers as T

    cfg = T.LlamaConfig.llama3_2_3b(tie_word_embeddings=args.tied)
    nelem = (cfg.vocab_size * cfg.hidden_size * (1 if args.tied else 2) + cfg.num_hidden_layers *
             (cfg.hidden_size * (QKV + H + 3 * I) + 2 * cfg.hidden_size) + cfg.hidden_size) // 8 * 8
    res["optimizer"] = optimizer(args.rounds, nelem)
    runs = {"bf16": [], "fp32": []}
    for _ in range(args.step_rounds):
        for name in ("bf16", "fp32"):
            tps, ms, peak, nparam = pretrain_step(name == "fp32", args.tied, args.steps, args.warmup)
            runs[name].append((tps, ms, peak, nparam))
            print(json.dumps(dict(step=name + "_gradients", tied=args.tied, tokens_per_s=tps, step_ms=ms, peak_alloc_gib=peak,
                                  params=nparam)), flush=True)
    res["pretrain"] = {k: dict(tokens_per_s=summary([r[0] for r in v]), step_ms=summary([r[1] for r in v]),
                               peak_alloc_gib=max(r[2] for r in v), params=v[0][3]) for k, v in runs.items()}
    p = res["pretrain"]
    p["fp32_over_bf16_step_ms"] = p["fp32"]["step_ms"]["median"] / p["bf16"]["step_ms"]["median"]
    p["extra_peak_gib"] = p["fp32"]["peak_alloc_gib"] - p["bf16"]["peak_alloc_gib"]
    res["gpu_after"] = gpu_info()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=2)


if __name__ == "__main__":
    main()
