"""Serving benchmark of continuous batching on the paged KV cache: one seeded stream of requests of mixed lengths (prompts
U{32..512}, outputs U{32..1920}; greedy, EOS disabled so every request runs to its drawn length), served three ways in one
process from the same cache bytes:
  (a) static batching: generate(block_attn=True, append_attn=True) in batches of 64, each padded to its longest prompt and run
      to its longest max_length;
  (b) continuous_generate with max_batch_size 64;
  (c) continuous_generate with larger max_batch_size (128, 256).
The modes alternate, round after round (--rounds), so that a drift of the shared host or card shows up in every mode alike.
Reports per mode and round useful generated tokens/s (each request's own max_length), total time, steps, pre-emptions, peak
blocks and the mean decode-only step (host clock, the per-step header read included), next to the decode step of
tools/gen_bench.py --block-attn at batch 64, with the card name and power limit.  Nothing about speed is asserted here.

    python tools/serve_bench.py --preset llama3_2_1b
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel  # noqa: E402
from tools import gen_bench  # noqa: E402

STATIC_BATCH = 64


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card name from torch is still reported
        q = f"nvidia-smi unavailable: {e}"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def make_requests(n, vocab, seed, prompt_range, out_range):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n):
        p = int(torch.randint(prompt_range[0], prompt_range[1] + 1, (1,), generator=g))
        m = int(torch.randint(out_range[0], out_range[1] + 1, (1,), generator=g))
        reqs.append((torch.randint(1, vocab, (p,), generator=g), m))
    return reqs


def static(m, reqs, max_prompt, max_out):
    """Batches of STATIC_BATCH in queue order, right-padded to the longest prompt and run to the longest max_length."""
    caches = m.allocate_block_caches(STATIC_BATCH, max_prompt + max_out)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, len(reqs), STATIC_BATCH):
        batch = reqs[i:i + STATIC_BATCH]
        S = max(ids.numel() for ids, _ in batch)
        ids = torch.zeros(len(batch), S, dtype=torch.int64)
        for b, (p, _) in enumerate(batch):
            ids[b, :p.numel()] = p
        lens = torch.tensor([p.numel() for p, _ in batch], dtype=torch.int32)
        m.generate(ids.cuda(), seq_len_encoder=lens.cuda(), max_length=max(n for _, n in batch), eos_token_id=-1,
                   cache_kvs=caches, sync_interval=0)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    num_blocks = caches[0].shape[0]
    del caches
    return dict(mode="static", batch=STATIC_BATCH, seconds=dt, num_blocks=num_blocks)


def continuous(m, reqs, max_batch_size, num_blocks):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs, stats = m.continuous_generate(reqs, max_batch_size=max_batch_size, num_blocks=num_blocks)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert [o.numel() for o in outs] == [n for _, n in reqs]
    return dict(mode="continuous", batch=max_batch_size, seconds=dt, num_blocks=num_blocks, ms_per_step=dt * 1e3 / stats["steps"],
                **stats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", choices=sorted(gen_bench.PRESETS), default="llama3_8b")
    ap.add_argument("--requests", type=int, default=512, help="a multiple of 64 (the static batch)")
    ap.add_argument("--prompt", type=int, nargs=2, default=[32, 512])
    ap.add_argument("--out", type=int, nargs=2, default=[32, 1920])
    ap.add_argument("--batches", type=int, nargs="+", default=[128, 256], help="max_batch_size of the larger runs (c)")
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--rounds", type=int, default=2, help="rounds of all modes, alternating")
    ap.add_argument("--quant-type", default="", choices=["", "weight_only_int8"], help="int8 layer weights (weight-only)")
    ap.add_argument("--cachekv-int8", action="store_true",
                    help="uint8 paged KV cache (static scales calibrated on the first requests' prompts), in the bf16 runs' "
                         "cache bytes: twice the pages")
    a = ap.parse_args()
    if a.requests % STATIC_BATCH:
        raise SystemExit(f"--requests must be a multiple of {STATIC_BATCH}")
    make = gen_bench.PRESETS[a.preset]
    cfg = make(num_hidden_layers=a.layers) if a.layers else make()
    m = LlamaForCausalLMInferenceModel(cfg, block_attn=True, append_attn=True, block_size=64, quant_type=a.quant_type,
                                       cachekv_int8_type="static" if a.cachekv_int8 else None)
    m.init_random(seed=42)
    reqs = make_requests(a.requests, cfg.vocab_size, a.seed, a.prompt, a.out)
    max_prompt, max_out = a.prompt[1], a.out[1]
    useful = sum(n for _, n in reqs)
    if a.cachekv_int8:
        calib = reqs[:16]
        S = max(p.numel() for p, _ in calib)
        ids = torch.zeros(len(calib), S, dtype=torch.int64)
        for b, (p, _) in enumerate(calib):
            ids[b, :p.numel()] = p
        m.calibrate_cache_scales(ids, torch.tensor([p.numel() for p, _ in calib], dtype=torch.int32))
    # the same cache bytes for every mode: the static batch's bf16 pages (twice as many uint8 pages)
    num_blocks = STATIC_BATCH * math.ceil((max_prompt + max_out) / m.block_size) * (2 if a.cachekv_int8 else 1)
    # warm-up: module loads and allocator pools of both paths
    warm = make_requests(8, cfg.vocab_size, 1, (16, 64), (8, 32))
    m.continuous_generate(warm, max_batch_size=4, num_blocks=64)
    static(m, make_requests(STATIC_BATCH, cfg.vocab_size, 2, (16, 64), (8, 16)), 64, 16)
    runs = []
    for rnd in range(a.rounds):
        runs += [static(m, reqs, max_prompt, max_out), continuous(m, reqs, STATIC_BATCH, num_blocks)]
        runs += [continuous(m, reqs, bsz, num_blocks) for bsz in a.batches]
        for r in runs[-2 - len(a.batches):]:
            r["round"] = rnd
            r["useful_tokens_per_s"] = useful / r["seconds"]
    del m
    torch.cuda.empty_cache()
    ref = gen_bench.run(batch=STATIC_BATCH, prompt=128, gen=256, block_attn=True, preset=a.preset, layers=a.layers,
                        quant_type=a.quant_type, cachekv_int8=a.cachekv_int8)
    print(json.dumps(dict(preset=a.preset, quant_type=a.quant_type, cachekv_int8=a.cachekv_int8, requests=a.requests, prompt=a.prompt, out=a.out, useful_tokens=useful, **card(),
                          runs=runs, gen_bench_block_attn=dict(batch=STATIC_BATCH, ms_per_step=ref["ms_per_step"])),
                     indent=1), flush=True)


if __name__ == "__main__":
    main()
