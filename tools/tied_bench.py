"""Tied against untied input / output embeddings on an H100, in one process.

1. The lm-head GEMMs at the Llama-3.2-3B training shape (T = 4096 tokens, V = 128 256, h = 3072) and the decode-step head
   (M = 64 rows), each in its untied and its tied operand form:
       logits   untied gemm(hf, head)                            tied gemm(hf, E, trans_b)       E [V, h] K-major B
       dX       untied gemm(dlogits, head, trans_b)              tied gemm(dlogits, E)           E MN-major B
       dW       untied gemm(hf, dlogits, trans_a) -> [h, V]      tied gemm(dlogits, hf, trans_a) -> [V, h], accumulate
       decode   untied _mm(hn, head)                             tied _mm(hn, E, trans_b)
   The two forms alternate over REPEATS rounds so clock and neighbour drift hit both alike; median and (min, max).
2. The Llama-3.2-3B pre-training step of bench.py (8 x 4096 tokens per step, micro-batch 1, AdamW), untied and tied,
   alternating over STEP_ROUNDS rounds (a fresh model per round: both do not fit one card at once): tokens/s and the
   peak allocated memory (GiB, the unit bench.py reports).
3. The GPU name, power limit and SM clock.

    python tools/tied_bench.py [--rounds N] [--step-rounds N] [--steps K] [--out FILE]
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

BF16 = torch.bfloat16
T_TOK, V, H, DECODE_M = 4096, 128256, 3072, 64
SEQ, PER_GPU_BATCH = 4096, 8


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.splitlines()[0].split(",")))) if r.returncode == 0 else {}


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


def summary(ts):
    return dict(median=statistics.median(ts), min=min(ts), max=max(ts))


def gemms(rounds):
    from paddlenlp_b200.experimental.transformers.fused_transformer_layers import FusedMultiTransformerBase

    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * s).to(BF16)

    hf, dl = rnd(T_TOK, H), rnd(T_TOK, V, s=1e-3)
    head, E = rnd(H, V, s=0.02), rnd(V, H, s=0.02)
    g_head, g_E = torch.zeros(H, V, dtype=BF16, device=dev), torch.zeros(V, H, dtype=BF16, device=dev)
    hn = rnd(DECODE_M, H)
    # FusedMultiTransformerBase._mm at M <= SKINNY_M and N = V (>= 100 column tiles): the persistent GEMM, cta_group 1
    assert DECODE_M <= FusedMultiTransformerBase.SKINNY_M and V >= 100 * 256

    def mm(a, w, trans_b=False):
        return ops.gemm(a, w, trans_b=trans_b, cta_group=1)

    cases = {
        "logits": (lambda: ops.gemm(hf, head), lambda: ops.gemm(hf, E, trans_b=True)),
        "dX": (lambda: ops.gemm(dl, head, trans_b=True), lambda: ops.gemm(dl, E)),
        "dW": (lambda: ops.gemm(hf, dl, out=g_head, trans_a=True, accumulate=True),
               lambda: ops.gemm(dl, hf, out=g_E, trans_a=True, accumulate=True)),
        "decode_head_m64": (lambda: mm(hn, head), lambda: mm(hn, E, trans_b=True)),
    }
    res = {}
    for name, (fu, ft) in cases.items():
        tu, tt = [], []
        iters = 200 if name.startswith("decode") else 10
        for _ in range(rounds):
            tu.append(timeit(fu, iters))
            tt.append(timeit(ft, iters))
        su, st = summary(tu), summary(tt)
        res[name] = dict(untied_ms=su, tied_ms=st, tied_over_untied=st["median"] / su["median"])
        print(json.dumps({"gemm": name, **res[name]}), flush=True)
    del hf, dl, head, E, g_head, g_E, hn
    torch.cuda.empty_cache()
    return res


def pretrain_step(tied, steps, warmup):
    """bench.py's resident step (data already on the device) for a fresh Llama-3.2-3B.
    Returns (tokens/s, peak allocated GiB, parameters)."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.optimizer import AdamW, ClipGradByGlobalNorm, LinearAnnealingWithWarmupDecay

    dev = torch.device("cuda", 0)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = T.LlamaForCausalLM(T.LlamaConfig.llama3_2_3b(tie_word_embeddings=tied))
    eng = model.engine
    sched = LinearAnnealingWithWarmupDecay(3e-5, 3e-6, warmup_step=30, decay_step=10000)
    opt = AdamW(learning_rate=sched.get_lr, beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.01,
                grad_clip=ClipGradByGlobalNorm(1.0), multi_precision=True, engine=eng)
    g = torch.Generator().manual_seed(1234)
    tok = torch.randint(0, eng.V, (warmup + steps, PER_GPU_BATCH, SEQ + 1), generator=g)
    ids, lab = tok[:, :, :-1].contiguous().to(dev), tok[:, :, 1:].contiguous().to(dev)
    del tok

    def step(i):
        for m in range(PER_GPU_BATCH):
            eng.forward_loss(ids[i, m:m + 1], lab[i, m:m + 1])
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
    tps = PER_GPU_BATCH * SEQ * steps / (e0.elapsed_time(e1) / 1e3)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30          # GiB, as bench.py reports it
    nparam = eng.num_parameters()
    del model, eng, opt, ids, lab
    gc.collect()
    torch.cuda.empty_cache()
    return tps, peak, nparam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the GEMM timings")
    ap.add_argument("--step-rounds", type=int, default=3, help="alternating rounds of the pre-training step")
    ap.add_argument("--steps", type=int, default=3, help="timed steps per round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _lib.call("b200_device_check")
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    res = dict(gpu=info, gemm=gemms(args.rounds))
    runs = {"untied": [], "tied": []}
    for _ in range(args.step_rounds):
        for name in ("untied", "tied"):
            tps, peak, nparam = pretrain_step(name == "tied", args.steps, args.warmup)
            runs[name].append((tps, peak, nparam))
            print(json.dumps(dict(step=name, tokens_per_s=tps, peak_alloc_gib=peak, params=nparam)), flush=True)
    res["pretrain"] = {k: dict(tokens_per_s=summary([r[0] for r in v]), peak_alloc_gib=max(r[1] for r in v), params=v[0][2])
                       for k, v in runs.items()}
    res["pretrain"]["tied_over_untied_tokens_per_s"] = (res["pretrain"]["tied"]["tokens_per_s"]["median"] /
                                                        res["pretrain"]["untied"]["tokens_per_s"]["median"])
    res["pretrain"]["peak_saving_gib"] = res["pretrain"]["untied"]["peak_alloc_gib"] - res["pretrain"]["tied"]["peak_alloc_gib"]
    res["gpu_after"] = gpu_info()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=2)


if __name__ == "__main__":
    main()
