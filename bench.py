"""bench.py — tokens/s of a Llama-3 bf16 pre-training step on H100 80 GB (Llama-3.2-3B shapes; BASELINE.json configs[1] / configs[2]
used Llama-3-8B, whose full-parameter AdamW state alone is 128 GB).

    python bench.py [--gpus N --steps K --warmup W]                 # N = 1 (default) runs in-process
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W                      # one rank per GPU, NCCL
    python bench.py --impl reference ...                            # the reference's math on the host CPU (oracle port)

One "step" = one optimizer step over per-GPU batch 8 x seq 4096 synthetic tokens (8 micro-batches of 1 sequence with
gradient accumulation into the flat gradient buffer — the Trainer's gradient_accumulation_steps semantics,
trainer.py:1045-1091), including the data-parallel gradient all-reduce and the AdamW update; nothing is skipped.
Every step sees a FRESH random batch (drawn on the CPU from one seeded generator before the timed region).
Prints ONE JSON line (rank 0).  `value` has inputs resident in HBM; `e2e` runs the same step through the public
Trainer-facing API (model(input_ids, labels) -> loss.backward() -> optimizer.step()) with pinned-host inputs, the H2D
copies and a D2H read of the loss inside the timed region.

The same line also carries BASELINE.json configs[3] and configs[4] under `other_configs` (skip with --only-pretrain):
  sft     Qwen2-1.5B full-parameter SFT, seq 2048, through Trainer.train() (pure data parallel over the launched ranks)
  decode  Llama-3-8B generation, batch 64, prompt 128 -> +1920, FusedMultiTransformer KV-cache path (rank 0, N=1 only:
          the decode path does not shard — replicas only)
and `breakdown`: the in-step device time of every kernel family (CUDA events around each C-ABI call during one extra
step after the timed region; GEMM is additionally timed live INSIDE the timed region for `roofline`).
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SEQ = 4096
PER_GPU_BATCH = 8
METRIC = "tokens/sec Llama-3.2-3B seq4096 bf16 pretrain step (global, all GPUs)"


def load_peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return dict(bf16_burst=p["bf16_tflops"], bf16_sustained=p["bf16_tflops_sustained"], hbm=p["hbm_gbs"],
                    source="measured (MEASURED_PEAKS.json)")
    except Exception:
        return dict(bf16_burst=989.0, bf16_sustained=989.0, hbm=3350.0, source="H100 SXM data sheet (dense BF16, 700 W)")


class ClockSampler:
    """nvidia-smi clock / throttle-reason samples DURING the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu = gpu_index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i",
                                          str(self.gpu), "-lms", "200"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                                         text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, smax, reasons = [], [], set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); smax.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "samples": len(sm), "reasons": sorted(reasons)}


# ----------------------------------------------------------------------------------------------------------------
# CPU baseline (oracle port): one decoder layer fwd+bwd + lm_head/criterion fwd+bwd on a bounded token sample
# ----------------------------------------------------------------------------------------------------------------
def cpu_reference_sample(layer_tokens: int = 512, head_tokens: int = 128, attn_heads: int = 6, threads: int | None = None):
    """Times the oracle (oracle/llama_ref.py, bf16-rounding mode) on the host cores and extrapolates tokens/s of the
    full benchmark step (Llama-3.2-3B shapes):  tokens/s = 1 / (L * (t_layer/token + t_attn4096/token) + t_head/token)  where
      t_layer     = fwd+bwd of ONE full-width decoder layer on `layer_tokens` tokens (its own attention runs at that short
                    length: ~1 % of the layer's work),
      t_attn4096  = fwd+bwd of the causal GQA attention at the REAL sequence length 4096 on `attn_heads` of the q heads
                    (attn_heads/3 kv heads), scaled to all heads,
      t_head      = final norm + lm_head + criterion fwd+bwd on `head_tokens` tokens."""
    import torch

    from oracle import llama_ref as R

    # all PHYSICAL host cores, regardless of OMP_NUM_THREADS (torchrun exports OMP_NUM_THREADS=1; one thread per hardware thread
    # of a 2-way SMT host is slower for these GEMMs than one per core: measured 14.0 s vs ~3 s for the 512-token layer)
    if not threads:
        try:
            import psutil
            threads = psutil.cpu_count(logical=False) or os.cpu_count() or 1
        except Exception:
            threads = os.cpu_count() or 1
    torch.set_num_threads(threads)
    cores = torch.get_num_threads()
    cfg = R.llama3_2_3b()
    g = torch.Generator().manual_seed(0)
    h, I, d = cfg.hidden_size, cfg.intermediate_size, cfg.head_dim
    kvd = cfg.num_key_value_heads * d
    p = "llama.layers.0."
    cache = cpu_reference_sample.__dict__.setdefault("_weights", {})
    if not cache:
        def mat(*shape):
            return torch.empty(*shape).normal_(0.0, 0.02, generator=g)
        cache["w"] = {p + "self_attn.q_proj.weight": mat(h, h), p + "self_attn.k_proj.weight": mat(h, kvd),
                      p + "self_attn.v_proj.weight": mat(h, kvd), p + "self_attn.o_proj.weight": mat(h, h),
                      p + "mlp.gate_proj.weight": mat(h, I), p + "mlp.up_proj.weight": mat(h, I),
                      p + "mlp.down_proj.weight": mat(I, h), p + "input_layernorm.weight": torch.ones(h),
                      p + "post_attention_layernorm.weight": torch.ones(h)}
        cache["head"] = mat(h, cfg.vocab_size)
    w = {k: v.detach().requires_grad_(True) for k, v in cache["w"].items()}
    x = torch.randn(1, layer_tokens, h, generator=g).requires_grad_(True)
    cos, sin = R.rope_tables(d, layer_tokens, cfg.rope_theta)
    t0 = time.perf_counter()
    y = R.decoder_layer(x, w, p, cfg, cos, sin, "bf16")
    y.sum().backward()
    t_layer = time.perf_counter() - t0
    # attention at the real sequence length
    rep = cfg.num_attention_heads // cfg.num_key_value_heads
    akv = max(1, attn_heads // rep)
    q = torch.randn(1, SEQ, akv * rep, d, generator=g).requires_grad_(True)
    k = torch.randn(1, SEQ, akv, d, generator=g).requires_grad_(True)
    v = torch.randn(1, SEQ, akv, d, generator=g).requires_grad_(True)
    t0 = time.perf_counter()
    R.attention(q, k, v, "bf16").sum().backward()
    t_attn = (time.perf_counter() - t0) * (cfg.num_attention_heads / (akv * rep))
    del q, k, v
    head = cache["head"].detach().requires_grad_(True)
    hs = torch.randn(1, head_tokens, h, generator=g).requires_grad_(True)
    labels = torch.randint(0, cfg.vocab_size, (1, head_tokens), generator=g)
    t0 = time.perf_counter()
    logits = R.linear(R.rms_norm(hs, torch.ones(h), cfg.rms_norm_eps, "bf16"), head, None, "bf16")
    R.criterion(logits, labels).backward()
    t_head = time.perf_counter() - t0
    per_token = cfg.num_hidden_layers * (t_layer / layer_tokens + t_attn / SEQ) + t_head / head_tokens
    return dict(value=1.0 / per_token, unit="tokens/s", cores=cores, kind="port",
                sample=(f"oracle/llama_ref.py (torch CPU, bf16-rounding mode) fwd+bwd of ONE full-width decoder layer on "
                        f"{layer_tokens} tokens ({t_layer:.2f} s) + causal GQA attention fwd+bwd at seq {SEQ} on {akv * rep} of "
                        f"{cfg.num_attention_heads} q heads (scaled to all heads: {t_attn:.2f} s) + final-norm/lm_head/criterion "
                        f"on {head_tokens} tokens ({t_head:.2f} s); extrapolated x{cfg.num_hidden_layers} layers; optimizer step not included"),
                seconds=t_layer + t_attn * (akv * rep) / cfg.num_attention_heads + t_head)


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    vals = []
    for i in range(args.warmup + args.steps):
        r = cpu_reference_sample()
        if i >= args.warmup:
            vals.append(r)
    v = statistics.mean(x["value"] for x in vals)
    secs = statistics.mean(x["seconds"] for x in vals)
    base = dict(vals[-1]); base["value"] = v
    base.pop("seconds", None)
    out = {"impl": "reference", "metric": METRIC, "value": v, "unit": "tokens/s", "n_gpus": args.gpus, "steps": args.steps,
           "warmup": args.warmup, "ms_per_step": secs * 1e3, "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
           "config": {"workload": "Llama-3.2-3B bf16 pretrain step, per-GPU batch 8 x seq 4096",
                      "note": "reference arm = the reference's math on host CPU cores (PaddlePaddle is not installable "
                              "here); each step is a bounded sample, value extrapolated to the full model"},
           "cpu_baseline": base,
           "e2e": {"value": v, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(out), flush=True)


# ----------------------------------------------------------------------------------------------------------------
# native arm
# ----------------------------------------------------------------------------------------------------------------
# kernel family of every C-ABI entry point the training step calls (for `breakdown`)
FAMILY = {
    "b200_gemm_bf16_ex": "gemm (wgmma)", "b200_gemm_bf16": "gemm (wgmma)",
    "b200_gemm_swiglu_bf16": "gemm + swiglu epilogue (wgmma)", "b200_gemm_swiglu_bwd_bf16": "gemm + swiglu-bwd epilogue (wgmma)",
    "b200_fa_fwd_flashmask": "attention fwd (mma.sync)", "b200_fa_fwd": "attention fwd (mma.sync)",
    "b200_fa_bwd_flashmask": "attention bwd (mma.sync)", "b200_fa_bwd": "attention bwd (mma.sync)",
    "b200_rmsnorm_fwd": "rmsnorm", "b200_rmsnorm_bwd": "rmsnorm", "b200_rope_inplace": "rope",
    "b200_swiglu_fwd": "swiglu", "b200_swiglu_bwd": "swiglu", "b200_embedding_fwd": "embedding",
    "b200_embedding_bwd": "embedding", "b200_ce_fwd": "cross-entropy", "b200_ce_bwd": "cross-entropy",
    "b200_grad_sqnorm": "optimizer (|g|^2 + AdamW)", "b200_adamw_step": "optimizer (|g|^2 + AdamW)",
    "b200_colsum_bf16": "bias grad",
}


def free_device_memory():
    import gc

    import torch

    from paddlenlp_b200 import ops

    ops._workspaces.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def run_native(args):
    import torch
    import torch.distributed as dist

    import paddlenlp_b200.transformers as T
    from paddlenlp_b200 import _lib
    from paddlenlp_b200 import distributed as dist_env
    from paddlenlp_b200.optimizer import AdamW, ClipGradByGlobalNorm, LinearAnnealingWithWarmupDecay

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with: python -m torch.distributed.run --nproc-per-node N bench.py --gpus N ...")
    torch.cuda.set_device(local)
    dist_env.init_parallel_env("nccl")
    dev = torch.device("cuda", local)
    _lib.call("b200_device_check")

    cfg = T.LlamaConfig.llama3_2_3b(num_hidden_layers=args.layers) if args.layers else T.LlamaConfig.llama3_2_3b()
    model = T.LlamaForCausalLM(cfg)
    eng = model.engine
    dp = dist_env.DataParallel(model) if world > 1 else None
    sched = LinearAnnealingWithWarmupDecay(3e-5, 3e-6, warmup_step=30, decay_step=10000)   # llm/config/llama/pretrain_argument.json
    opt = AdamW(learning_rate=sched.get_lr, beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.01,
                grad_clip=ClipGradByGlobalNorm(1.0), multi_precision=True, engine=eng)
    opt.grad_scale = 1.0 / world
    mb = args.micro_batch
    accum = PER_GPU_BATCH // mb
    tokens_per_step = PER_GPU_BATCH * SEQ * world

    # synthetic data: a FRESH global batch for every step (warm-up, timed, breakdown and e2e steps all differ), drawn on the
    # CPU from one seeded generator; rank r owns rows r*8 .. r*8+7 of each global batch (SURVEY.md §8d)
    g = torch.Generator().manual_seed(1234)
    n_resident = args.warmup + args.steps + 1               # +1: the breakdown step
    n_e2e = args.steps + 1                                  # +1: one untimed step through the public API before its timed steps
    lo, hi = dist_env.shard_rows(PER_GPU_BATCH * world, rank, world)

    def draw(n):
        rows = []
        for _ in range(n):
            tok = torch.randint(0, cfg.vocab_size, (PER_GPU_BATCH * world, SEQ + 1), generator=g)
            rows.append(tok[lo:hi].clone())
        return torch.stack(rows)

    tok_res = draw(n_resident)
    dev_ids, dev_lab = tok_res[:, :, :-1].contiguous().to(dev), tok_res[:, :, 1:].contiguous().to(dev)
    tok_e2e = draw(n_e2e)
    host_ids = tok_e2e[:, :, :-1].contiguous().pin_memory()
    host_lab = tok_e2e[:, :, 1:].contiguous().pin_memory()
    del tok_res, tok_e2e
    l2_flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    step_losses = []        # device scalars of the first micro-batch of every resident step (read after the timed region)

    def step_resident(i):
        for m in range(accum):
            loss_out = eng.forward_loss(dev_ids[i, m * mb:(m + 1) * mb], dev_lab[i, m * mb:(m + 1) * mb])[0]
            if m == 0:
                step_losses.append(loss_out)
            if dp is not None and m == accum - 1:
                dp.prepare_backward()            # last micro-batch: finished gradient ranges are all-reduced during backward
            eng.backward(1.0 / accum)
        if dp is not None:
            dp.sync_gradients()
        opt.step(); sched.step(); opt.clear_grad()

    def step_e2e(i):
        """Public API path: pinned host batch -> H2D -> model(input_ids, labels) -> loss.backward() -> all-reduce ->
        optimizer.step(); the step's loss is read back to the host."""
        total = torch.zeros((), device=dev)
        for m in range(accum):
            ids = host_ids[i, m * mb:(m + 1) * mb].to(dev, non_blocking=True)
            lab = host_lab[i, m * mb:(m + 1) * mb].to(dev, non_blocking=True)
            ctx = dp.no_sync() if (dp is not None and m < accum - 1) else contextlib.nullcontext()
            with ctx:                            # trainer.py:1049-1075: accumulation micro-steps skip the exchange
                loss, _ = (dp or model)(input_ids=ids, labels=lab)
                loss = loss / accum
                loss.backward()
            total += loss.detach()
        if dp is not None:
            dp.sync_gradients()
        opt.step(); sched.step(); opt.clear_grad()
        return total.item()          # D2H of the step loss

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, k, first=0):
        """K steps bracketed by barrier + synchronize; device time by CUDA events; max over ranks."""
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(k):
            fn(first + i)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()

    for i in range(args.warmup):
        step_resident(i)
    l2_flush.zero_()

    # GEMM (dominant kernel family) timed live with CUDA events on the launching stream during the timed region
    gemm_events = []

    @contextlib.contextmanager
    def hook(name, a):
        if name in ("b200_gemm_bf16_ex", "b200_gemm_swiglu_bf16", "b200_gemm_swiglu_bwd_bf16"):
            if name == "b200_gemm_bf16_ex":
                M, N, K = int(a[5]), int(a[6]), int(a[7])
            elif name == "b200_gemm_swiglu_bf16":          # (X, W, GU, M_out, M, I, K, ...): N = 2 I
                M, N, K = int(a[4]), 2 * int(a[5]), int(a[6])
            else:                                          # (dY, Wdown, GU, DGU, M, I, K, ...): N = I
                M, N, K = int(a[4]), int(a[5]), int(a[6])
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            yield
            e1.record()
            gemm_events.append((e0, e1, 2.0 * M * N * K, (M, N, K)))
        else:
            yield

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = _lib.launch_count
    _lib.call_hook = hook if rank == 0 else None
    ms = timed(step_resident, args.steps, first=args.warmup)
    _lib.call_hook = None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, step_losses[args.warmup + args.steps - 1], model)
    launches = _lib.launch_count - launches0
    clocks = sampler.stop() if rank == 0 else None
    gemm_ms = sum(e0.elapsed_time(e1) for e0, e1, _, _ in gemm_events)
    gemm_flops = sum(f for _, _, f, _ in gemm_events)
    n_gemm = len(gemm_events)
    per_shape = {}
    for e0, e1, f, shp in gemm_events:
        r = per_shape.setdefault(shp, [0, 0.0, 0.0])
        r[0] += 1; r[1] += e0.elapsed_time(e1); r[2] += f
    gemm_events.clear()

    # one extra step with CUDA events around EVERY C-ABI call: in-step time of each kernel family (all ranks run it — the
    # gradient exchange is collective — rank 0 records)
    fam_events = []

    @contextlib.contextmanager
    def hook_all(name, a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        yield
        e1.record()
        fam_events.append((FAMILY.get(name, name), e0, e1))

    _lib.call_hook = hook_all if rank == 0 else None
    ms_bd = timed(step_resident, 1, first=args.warmup + args.steps)
    _lib.call_hook = None
    breakdown = None
    if rank == 0:
        fam = {}
        for name, e0, e1 in fam_events:
            r = fam.setdefault(name, [0, 0.0])
            r[0] += 1; r[1] += e0.elapsed_time(e1)
        covered = sum(v[1] for v in fam.values())
        breakdown = {"step_ms": ms_bd, "note": "one extra step, CUDA events around every C-ABI call (adds ~2 event records per call)",
                     "families": {k: {"calls": v[0], "ms": round(v[1], 3), "share": round(v[1] / ms_bd, 4)}
                                  for k, v in sorted(fam.items(), key=lambda kv: -kv[1][1])},
                     "uncovered_ms (launch gaps, torch fill/copy, NCCL)": round(ms_bd - covered, 3)}
    fam_events.clear()
    first_losses = [float(t[0]) for t in step_losses[:1] + step_losses[args.warmup:args.warmup + 1] + step_losses[-1:]]

    losses = []
    step_e2e(args.steps)                 # untimed: first call through the public-API path (autograd wrapper, pinned-buffer copies)
    ms_e2e = timed(lambda i: losses.append(step_e2e(i)), args.steps)

    peaks = load_peaks()
    ms_per_step = ms / args.steps
    value = tokens_per_step / (ms_per_step / 1e3)
    e2e_value = tokens_per_step / (ms_e2e / args.steps / 1e3)
    flops_per_token = model.get_algorithmic_flops_per_token(SEQ)
    tf_per_gpu = value / world * flops_per_token / 1e12
    gemm_tf = gemm_flops / (gemm_ms / 1e3) / 1e12 if gemm_ms > 0 else None
    hbm_peak_gb = torch.cuda.max_memory_allocated() / 2 ** 30
    out = None
    if rank == 0:
        out = {
            "metric": METRIC, "value": value, "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic",
            "config": {"workload": "Llama-3.2-3B bf16 pretrain step, per-GPU batch 8 x seq 4096",
                       "model": "Llama-3.2-3B" if not args.layers else f"Llama-3.2-3B width, {args.layers} layers (DEBUG, not the metric)",
                       "global_batch": PER_GPU_BATCH * world, "seq_len": SEQ, "micro_batch": mb, "grad_accum": accum,
                       "parallelism": f"dp{world}", "optimizer": "AdamW fp32 master + global-norm clip, in the timed step",
                       "batches": "a fresh uniform-random batch every step (seed 1234, drawn on the CPU before the timed region)",
                       "l2": "inputs (weights 7 GB, activations) exceed the 50 MB L2; a 192 MB flush precedes the timed region"},
            "clocks": clocks,
            "gpu_launches": launches,
            "hbm_peak_allocated_gb": hbm_peak_gb,
            "first_loss": first_losses[0] if first_losses else None,      # ~ ln(vocab) = 11.76 at the reference init
            "loss_trace": {"first_warmup_step": first_losses[0] if first_losses else None,
                           "first_timed_step": first_losses[1] if len(first_losses) > 1 else None,
                           "last_step": first_losses[-1] if first_losses else None, "ln_vocab": 11.7618},
            "model_tflops_per_gpu": tf_per_gpu,
            "clock_normalised": {"sm_mhz_over_max": (clocks["sm_mhz"] / clocks["sm_max_mhz"]) if clocks and clocks.get("sm_mhz") else None,
                                 "model_tflops_per_gpu_per_ghz": (tf_per_gpu / (clocks["sm_mhz"] / 1e3)) if clocks and clocks.get("sm_mhz") else None,
                                 "note": "compare runs on different boxes by TFLOP/s per GHz of median SM clock"},
            "mfu": {"algorithmic_gflop_per_token": flops_per_token / 1e9, "vs_nominal_989": tf_per_gpu / 989.0,
                    "vs_measured_burst": tf_per_gpu / peaks["bf16_burst"], "vs_measured_sustained": tf_per_gpu / peaks["bf16_sustained"]},
            "roofline": {"bound": "tensor", "kernel": "gemm_bf16_kernel (wgmma, all projection/lm_head GEMMs fwd+bwd)",
                         "achieved": gemm_tf, "peak": peaks["bf16_sustained"], "unit": "TFLOP/s",
                         "frac": (gemm_tf / peaks["bf16_sustained"]) if gemm_tf else None, "peak_source": peaks["source"] + ", sustained",
                         "launches_timed": n_gemm, "avg_launch_ms": gemm_ms / max(1, n_gemm), "share_of_step": gemm_ms / ms,
                         "algorithmic_flops_per_launch": gemm_flops / max(1, n_gemm),
                         "per_shape_MNK": {f"{k[0]}x{k[1]}x{k[2]}": {"launches": v[0], "ms_per_launch": round(v[1] / v[0], 4),
                                                                       "tflops": round(v[2] / (v[1] / 1e3) / 1e12, 1)}
                                           for k, v in sorted(per_shape.items(), key=lambda kv: -kv[1][1])}},
            "breakdown": breakdown,
            "e2e": {"value": e2e_value, "unit": "tokens/s", "h2d_bytes_per_step": int(PER_GPU_BATCH * SEQ * 8 * 2),
                    "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps, "untimed_warmup_steps": 1, "first_loss": losses[0] if losses else None,
                    "last_loss": losses[-1] if losses else None},
        }

    # ---- BASELINE.json configs[3] (Qwen2-7B SFT, all ranks) and configs[4] (decode, rank 0 at N=1) in the same process ----
    if not args.only_pretrain and not args.layers:
        others = {}
        del model, eng, opt, dp, dev_ids, dev_lab, host_ids, host_lab, l2_flush
        step_losses.clear()
        free_device_memory()
        try:
            from tools import sft_bench
            rec = sft_bench.run(steps=args.sft_steps, warmup=2, micro_batch=4, accum=2, zero_padding=False, quiet=True)
            if rank == 0:
                others["sft"] = rec
        except Exception as e:  # the extra configs must never take the headline number down with them
            if rank == 0:
                others["sft"] = {"error": f"{type(e).__name__}: {str(e)[:300]}"}
        free_device_memory()
        if world == 1:
            try:
                from tools import gen_bench
                others["decode"] = gen_bench.run()
            except Exception as e:
                others["decode"] = {"error": f"{type(e).__name__}: {str(e)[:300]}"}
            free_device_memory()
        if rank == 0:
            out["other_configs"] = others
            if isinstance(others.get("decode"), dict) and "decode_tokens_per_s" in others["decode"]:
                out["decode_tok_s"] = others["decode"]["decode_tokens_per_s"]
                out["decode_roofline_frac"] = others["decode"]["roofline_frac"]
            if isinstance(others.get("sft"), dict) and "tokens_per_s" in others["sft"]:
                out["sft_tok_s"] = others["sft"]["tokens_per_s"]

    if rank != 0:
        return
    if world == 1 and not args.no_cpu_baseline:
        try:
            cb = cpu_reference_sample()
            cb.pop("seconds", None)
            out["cpu_baseline"] = cb
        except Exception as e:  # the CPU column must never take the GPU number down with it
            out["cpu_baseline"] = {"error": str(e)[:200]}
    print(json.dumps(out), flush=True)


def dump_outputs(out_dir, loss, model, per_tensor=16384):
    """What the timed path leaves to its caller after its last step: that step's loss (first micro-batch) and the updated
    parameters, as a fixed seeded sample of `per_tensor` entries per tensor (float32, ~16 MB in all)."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().float().reshape(-1).cpu().numpy())
    g = torch.Generator().manual_seed(4321)
    samples = []
    for name, t in sorted(model.state_dict().items()):
        flat = t.detach().reshape(-1)
        idx = torch.randint(0, flat.numel(), (min(per_tensor, flat.numel()),), generator=g)
        samples.append(flat[idx.to(flat.device)].float().cpu())
    np.save(os.path.join(out_dir, "param_sample.npy"), torch.cat(samples).numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--micro-batch", type=int, default=1, choices=[1, 2, 4, 8])
    ap.add_argument("--layers", type=int, default=0, help="debug only: fewer layers (invalidates the metric)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--only-pretrain", action="store_true", help="skip the Qwen2-1.5B SFT and Llama-3-8B decode sub-benchmarks")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's loss and a fixed, seeded sample of the updated "
                         "parameters as DIR/<name>.npy (float32), to compare two builds output for output")
    ap.add_argument("--sft-steps", type=int, default=4)
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_native(args)
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
