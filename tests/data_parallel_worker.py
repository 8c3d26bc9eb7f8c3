"""Rank worker of tests/test_data_parallel_gpu.py, launched by torch.distributed.run with two processes.

    python -m torch.distributed.run --nproc-per-node 2 tests/data_parallel_worker.py --backend gloo --out DIR [--sabotage]

gloo: both ranks on cuda:0 (gloo all-reduces CUDA tensors through host memory).  nccl: one device per rank.  Every check
raises an AssertionError naming what differs; rank 0 prints one `DPREPORT <json>` line per finished part.  Cross-rank
comparisons go through a separate gloo group on host copies, so they add no call to the gradient exchange they observe.

Engine-level step (per variant, overlap on and off): two micro-batches per rank, the first under no_sync().  Every
all-reduce of the flat gradient buffer is logged as (offset, numel, phase), and the overlap hook is wrapped so that each rank
snapshots its local range before DataParallel hands it to the collective.  Checks: (1) every element reduced exactly once
per optimizer step and never during a no_sync micro-batch; with overlap every range goes out during backward and
sync_gradients() adds nothing, without it there is one call over the whole buffer.  (2) The exchanged buffer is
bit-identical across ranks and equals round(local_0 + local_1): a two-way sum rounds once, in any order.  (3) Half the
exchanged gradient matches the fp32 oracle's gradient of the global batch, per named tensor.

Trainer at world 2 (model not pre-wrapped, rank 1 initialised from another seed): (4) flat_params, master, exp_avg and
exp_avg_sq bit-identical across ranks after every step; (5) step 1 equals fp64 AdamW from rank 0's initial weights with
gradient = exchanged / world; (6) per-step sample indices disjoint across ranks, one epoch covering the dataset once; (7) the
logged loss is the mean of the ranks' step losses; (8) only rank 0 writes files, rng_state_2.pth holds both ranks' states,
and a world-2 resume from checkpoint-2 reproduces step 3's loss bit for bit.

--sabotage also runs three faults and requires the checks to raise on each: sync_gradients() reducing the whole buffer
again, the overlap hook armed under no_sync(), and the optimizer's grad_scale left at 1.
"""
import argparse
import contextlib
import json
import math
import os
import shutil
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import llama_ref as R  # noqa: E402
from oracle import optim_ref  # noqa: E402
from tied_oracle import tied_loss_and_grads  # noqa: E402

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
WORLD = 2
B, S, ACCUM = 2, 256, 2                    # rows per micro-batch, tokens per row, micro-batches per optimizer step
# family, tied embeddings, fp32 gradients (amp_master_grad)
VARIANTS = {"llama": ("llama", False, False), "qwen2-tied": ("qwen2", True, False), "llama-fp32": ("llama", False, True)}
# Relative Frobenius error of (exchanged / 2) against the fp32 oracle's mean gradient, per named tensor.  Measured on an H100
# 80GB HBM3 (700 W power limit): worst 1.57e-2 over the three variants (a layer-3 q/k projection or bias), bf16 and fp32
# gradients alike.  The bound is ~4x that; a layer missed or reduced twice by the exchange is off by ~50%.
ORACLE_REL = 0.06
LR, WD, MAX_GRAD_NORM = 1e-3, 0.01, 100.0   # the clip stays inactive, so step 1's moments scale with grad_scale


def same_bits(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def n_differ(a, b):
    iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return int((a.contiguous().view(iv) != b.contiguous().view(iv)).sum())


class Ctx:
    def __init__(self, rank, group):
        self.rank, self.group = rank, group

    def gather(self, t):
        """Host copies of `t` from every rank (rank order), moved as bytes: the check group is gloo on the host."""
        x = t.detach().contiguous().view(-1).cpu()
        raw = x.view(torch.uint8)
        parts = [torch.empty_like(raw) for _ in range(WORLD)]
        dist.all_gather(parts, raw, group=self.group)
        return [p.view(x.dtype) for p in parts]

    def gather_obj(self, obj):
        out = [None] * WORLD
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def barrier(self):
        dist.barrier(group=self.group)

    def report(self, **kw):
        if self.rank == 0:
            print("DPREPORT " + json.dumps(kw), flush=True)


# ----------------------------------------------------------------------------------------------------------
# All-reduce log
# ----------------------------------------------------------------------------------------------------------
class ReduceLog:
    """Wraps torch.distributed.all_reduce (which paddlenlp_b200.distributed and the Trainer call through the module) and
    logs (offset, numel, phase) of every call on a view of `flat`."""

    def __init__(self):
        self.flat, self.phase, self.entries = None, None, []
        self.orig = dist.all_reduce
        dist.all_reduce = self._all_reduce

    def _all_reduce(self, tensor, *a, **k):
        f = self.flat
        if f is not None and tensor.untyped_storage().data_ptr() == f.untyped_storage().data_ptr():
            self.entries.append((tensor.storage_offset() - f.storage_offset(), tensor.numel(), self.phase))
        return self.orig(tensor, *a, **k)


def check_reduces(entries, numel, overlap, hook_ranges):
    """(1): every element of the flat gradient buffer all-reduced exactly once per optimizer step, none during a no_sync
    micro-batch; with overlap one call per reported range during backward and none from sync_gradients(), without it one
    call over the whole buffer."""
    for off, n, phase in entries:
        assert "no_sync" not in phase, f"all-reduce of [{off}, {off + n}) during {phase}"
    cover = torch.zeros(numel, dtype=torch.int32)
    for off, n, _ in entries:
        cover[off:off + n] += 1
    if not bool((cover == 1).all()):
        i = int((cover != 1).nonzero()[0])
        raise AssertionError(f"element {i} all-reduced {int(cover[i])} times in one optimizer step (per element "
                             f"{int(cover.min())}..{int(cover.max())} times over {len(entries)} calls)")
    if overlap:
        late = [e for e in entries if e[2] == "sync_gradients"]
        assert not late, f"sync_gradients() issued {len(late)} further all-reduce(s) after an overlapped backward: {late[:3]}"
        got = [(off, off + n) for off, n, _ in entries]
        assert got == hook_ranges, f"the all-reduces {got} are not the reported ranges {hook_ranges}"
    else:
        assert entries == [(0, numel, "sync_gradients")], f"without overlap: expected one call over [0, {numel}), got {entries}"


# ----------------------------------------------------------------------------------------------------------
# Models and data
# ----------------------------------------------------------------------------------------------------------
def make_model(family, tied, rank):
    """dp_check-sized model (4 layers, h 512, vocab 1024).  Rank r > 0 draws its weights from another seed, so only a
    broadcast makes the ranks agree."""
    import paddlenlp_b200.transformers as T

    kw = dict(vocab_size=1024, hidden_size=512, intermediate_size=1376, num_hidden_layers=4, num_attention_heads=4,
              num_key_value_heads=2, max_position_embeddings=S, seq_length=S, tie_word_embeddings=tied)
    m = T.LlamaForCausalLM(T.LlamaConfig(**kw)) if family == "llama" else T.Qwen2ForCausalLM(T.Qwen2Config(**kw))
    if rank:
        m.engine.init_weights(42 + 1000 * rank)
    return m


def ref_config(cfg):
    return R.RefConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                       num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                       num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                       qkv_bias=cfg.model_type == "qwen2", model_type=cfg.model_type,
                       max_position_embeddings=cfg.max_position_embeddings)


def global_batch(seed):
    """Tokens [ACCUM * WORLD, B, S + 1]: micro-batch m of rank r is entry m * WORLD + r."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, 1024, (ACCUM * WORLD, B, S + 1), generator=g)


# ----------------------------------------------------------------------------------------------------------
# Engine-level step
# ----------------------------------------------------------------------------------------------------------
def engine_step(ctx, log, family, tied, fp32, overlap, seed, sabotage=None, oracle=True):
    from paddlenlp_b200 import distributed as D

    dev = torch.device("cuda", torch.cuda.current_device())
    model = make_model(family, tied, ctx.rank)
    dp = D.DataParallel(model, overlap=overlap)
    eng = model.engine
    if fp32:
        model.set_master_grad(True)
    snaps = []
    on_ready = dp._on_ready

    def record(lo, hi):                  # the local range, on the compute stream, before the collective is enqueued
        snaps.append((lo, hi, log.phase, eng.flat_grads[lo:hi].clone()))
        on_ready(lo, hi)

    dp._on_ready = record
    if sabotage == "hook armed under no_sync":
        dp.prepare_backward = lambda: setattr(eng, "grad_ready_hook", dp._on_ready)
    elif sabotage == "sync_gradients reduces the whole buffer again":
        sync = dp.sync_gradients

        def sync_twice():
            sync()
            dist.all_reduce(eng.flat_grads)
        dp.sync_gradients = sync_twice
    tok = global_batch(seed)
    log.flat, log.entries = eng.flat_grads, []
    eng.clear_grad()
    last = f"micro-batch {ACCUM - 1}"
    for mb in range(ACCUM):
        t = tok[mb * WORLD + ctx.rank].to(dev)
        ids, lab = t[:, :-1].contiguous(), t[:, 1:].contiguous()
        log.phase = f"micro-batch {mb}" + (" (no_sync)" if mb < ACCUM - 1 else "")
        with (dp.no_sync() if mb < ACCUM - 1 else contextlib.nullcontext()):
            loss, _ = dp(input_ids=ids, labels=lab)
            (loss / ACCUM).backward()
    local = None if overlap else eng.flat_grads.clone()
    log.phase = "sync_gradients"
    dp.sync_gradients()
    torch.cuda.synchronize()
    log.flat = None
    numel = eng.numel
    hook_ranges = [(lo, hi) for lo, hi, ph, _ in snaps if ph == last]
    entries = list(log.entries)

    # (1)
    check_reduces(entries, numel, overlap, hook_ranges)
    if overlap:
        local = torch.empty_like(eng.flat_grads)
        for lo, hi, ph, s in snaps:
            if ph == last:
                local[lo:hi] = s
    # (2)
    ex = ctx.gather(eng.flat_grads)
    assert same_bits(ex[0], ex[1]), f"the exchanged gradients differ across ranks in {n_differ(ex[0], ex[1])} elements"
    l0, l1 = ctx.gather(local)
    assert not same_bits(l0, l1), "both ranks computed the same local gradients: the check below would prove nothing"
    want = (l0.double() + l1.double()).to(l0.dtype)
    assert same_bits(ex[0], want), f"exchanged != round(local_0 + local_1) in {n_differ(ex[0], want)} of {numel} elements"
    # (3) rank 0: half the exchanged gradient against the oracle's mean over the global batch's micro-batches
    worst, worst_name = 0.0, None
    if oracle and ctx.rank == 0:
        rc = ref_config(model.config)
        w = {k: v.detach().float().clone() for k, v in eng.named_views().items()}
        ref = None
        for i in range(ACCUM * WORLD):
            t = tok[i].to(dev)
            fn = tied_loss_and_grads if tied else R.loss_and_grads
            _, _, gr = fn(t[:, :-1], t[:, 1:], w, rc, mode="fp32")
            ref = gr if ref is None else {k: ref[k] + gr[k] for k in ref}
        got = eng.named_views(grads=True)
        assert set(got) == set(ref), sorted(set(got) ^ set(ref))
        for k, r in ref.items():
            r = r.double() / (ACCUM * WORLD)
            rel = ((got[k].double() * (1.0 / WORLD) - r).norm() / r.norm()).item()
            if rel > worst:
                worst, worst_name = rel, k
        assert worst <= ORACLE_REL, f"exchanged / {WORLD} vs the oracle: {worst_name} relative error {worst:.3e} > {ORACLE_REL}"
    calls = len(entries)
    del dp, model, eng, snaps, local
    torch.cuda.empty_cache()
    return dict(reduce_calls=calls, elements=numel, bit_identical_across_ranks=True, equals_rounded_local_sum=True,
                oracle_worst_rel=worst, oracle_worst_tensor=worst_name,
                oracle_margin=(ORACLE_REL / worst) if worst else None)


# ----------------------------------------------------------------------------------------------------------
# Trainer at world 2
# ----------------------------------------------------------------------------------------------------------
class Toy(torch.utils.data.Dataset):
    """24 samples = 3 optimizer steps of 2 ranks x 2 micro-batches x 2 rows; records every index it serves."""

    def __init__(self, n=24):
        g = torch.Generator().manual_seed(7)
        self.tok = torch.randint(1, 1024, (n, S + 1), generator=g)
        self.seen = []

    def __len__(self):
        return self.tok.shape[0]

    def __getitem__(self, i):
        self.seen.append(int(i))
        return {"input_ids": self.tok[i, :-1].clone(), "labels": self.tok[i, 1:].clone()}


def run_trainer(ctx, family, tied, fp32, out_dir, max_steps, save_steps, resume=None):
    from paddlenlp_b200.trainer import Trainer, TrainingArguments
    from paddlenlp_b200.trainer.trainer import TrainerCallback
    from paddlenlp_b200.transformers import conversion_utils as cu

    model = make_model(family, tied, ctx.rank)
    eng = model.engine
    init_params = eng.flat_params.clone()
    args = TrainingArguments(output_dir=out_dir, per_device_train_batch_size=B, gradient_accumulation_steps=ACCUM,
                             max_steps=max_steps, learning_rate=LR, weight_decay=WD, max_grad_norm=MAX_GRAD_NORM,
                             lr_scheduler_type="constant", logging_steps=1, save_steps=save_steps, max_seq_length=S,
                             amp_master_grad=fp32)
    ds = Toy()
    rec = dict(diffs=[], indices=[], step1=None, writes=[], losses=[])

    class Probe(TrainerCallback):
        """Records only: a check that raised inside train() on one rank would leave the other in a collective."""

        def on_step_end(self, a, state, control, **kw):
            opt = tr.optimizer
            for name, t in (("flat_params", eng.flat_params), ("master", opt.master), ("exp_avg", opt.exp_avg),
                            ("exp_avg_sq", opt.exp_avg_sq)):
                p = ctx.gather(t)
                if not same_bits(p[0], p[1]):
                    rec["diffs"].append((state.global_step, name, n_differ(p[0], p[1])))
            if state.global_step == 1:
                rec["step1"] = dict(exchanged=eng.flat_grads.clone(), master=opt.master.clone(), m=opt.exp_avg.clone(),
                                    v=opt.exp_avg_sq.clone(), grad_scale=opt.grad_scale, lr=opt.get_lr())
            rec["indices"].append(ds.seen[-B * ACCUM:])
            ds.seen.clear()

    tr = Trainer(model=model, args=args, train_dataset=ds, callbacks=[Probe()])
    ts = tr.training_step

    def training_step(m, inputs):
        loss = ts(m, inputs)
        rec["losses"].append(loss)
        return loss
    tr.training_step = training_step
    save_sharded, save_pretrained, tsave = cu.save_sharded, model.save_pretrained, torch.save

    def w_sharded(sd, d, *a, **k):
        rec["writes"].append(a[0] if a else k.get("weights_name", cu.SAFE_WEIGHTS_NAME))
        return save_sharded(sd, d, *a, **k)

    def w_pretrained(d, *a, **k):
        rec["writes"].append("model")
        return save_pretrained(d, *a, **k)

    def w_save(obj, f, *a, **k):
        if isinstance(f, (str, os.PathLike)):          # all_gather_object pickles through torch.save into a buffer
            rec["writes"].append(os.path.basename(str(f)))
        return tsave(obj, f, *a, **k)
    cu.save_sharded, model.save_pretrained, torch.save = w_sharded, w_pretrained, w_save
    try:
        tr.train(resume_from_checkpoint=resume)
    finally:
        cu.save_sharded, torch.save = save_sharded, tsave
    rec["log"] = [h for h in tr.state.log_history if "loss" in h]
    rec["init_params"], rec["decay_end"], rec["numel"] = init_params, eng.decay_end, eng.numel
    rec["args"] = args
    return rec


def check_same_across_ranks(rec):
    """(4)"""
    assert not rec["diffs"], "parameters or optimizer state differ across ranks: " + \
        ", ".join(f"{name} after step {s} ({n} elements)" for s, name, n in rec["diffs"])


def check_step1(rec):
    """(5) rank 0: step 1 against fp64 AdamW from rank 0's initial weights, gradient = exchanged * (1 / world), clip
    coefficient from the exchanged norm.  Bounds of test_kernels_at_scale_gpu's AdamW test with zero moments."""
    s1, a = rec["step1"], rec["args"]
    dev = s1["master"].device
    numel = rec["numel"]
    g = s1["exchanged"].double()
    master0 = rec["init_params"].double()
    mask = torch.arange(numel, device=dev) < rec["decay_end"]
    b1, b2 = a.adam_beta1, a.adam_beta2
    pr, mr, vr, _ = optim_ref.adamw_step(master0, torch.zeros_like(g), torch.zeros_like(g), g, lr=s1["lr"], beta1=b1,
                                         beta2=b2, eps=a.adam_epsilon, weight_decay=a.weight_decay, step=1, decay_mask=mask,
                                         grad_scale=1.0 / WORLD, max_grad_norm=a.max_grad_norm)
    norm = (g * (1.0 / WORLD)).norm().item()
    assert norm < a.max_grad_norm, f"gradient norm {norm} reaches the clip: step 1 would not depend on grad_scale"
    geff = g * (1.0 / WORLD)
    m_mag = (1 - b1) * geff.abs()
    mb = 2.0 ** -18 * m_mag
    vb = 2.0 ** -15 * (1 - b2) * geff.pow(2)
    denom = vr.sqrt() / math.sqrt(1 - b2) + a.adam_epsilon
    upd_mag = s1["lr"] / (1 - b1) * m_mag / denom
    pb = 2.0 ** -22 * master0.abs() + 2.0 ** -14 * upd_mag
    worst = {}
    for name, got, ref, bound in (("exp_avg", s1["m"], mr, mb), ("exp_avg_sq", s1["v"], vr, vb), ("master", s1["master"], pr, pb)):
        err = (got.double() - ref).abs()
        ok = err <= bound
        if not bool(ok.all()):
            i = int(torch.where(ok, 0.0, (err / bound).nan_to_num(math.inf)).argmax())
            raise AssertionError(f"step 1 {name} vs fp64 AdamW with grad_scale 1/{WORLD}: {int((~ok).sum())} of {numel} "
                                 f"elements beyond their bound; worst at {i}: got {got[i].item():.9e} ref {ref[i].item():.9e} "
                                 f"bound {bound[i].item():.3e} (optimizer grad_scale {s1['grad_scale']})")
        worst[name] = float((err / bound.clamp_min(1e-300)).max())
    return dict(step1_worst_err_over_bound=worst, step1_grad_norm=norm)


def check_trainer(ctx, rec, out_dir):
    check_same_across_ranks(rec)
    res = check_step1(rec) if ctx.rank == 0 else {}
    # (6)
    idx = ctx.gather_obj(rec["indices"])
    seen = []
    for s, (i0, i1) in enumerate(zip(*idx), 1):
        assert len(i0) == len(i1) == B * ACCUM, (s, i0, i1)
        assert not set(i0) & set(i1), f"step {s}: ranks read the same samples {sorted(set(i0) & set(i1))}"
        seen += i0 + i1
    assert sorted(seen) == list(range(24)), f"one epoch did not read every sample once: {sorted(seen)}"
    # (7)
    dev = rec["losses"][0].device
    per_step = []
    for s in range(len(rec["log"])):
        t = torch.zeros((), dtype=F32, device=dev)
        for x in rec["losses"][s * ACCUM:(s + 1) * ACCUM]:
            t += x
        per_step.append(t.item())
    both = ctx.gather_obj(per_step)
    for s, h in enumerate(rec["log"]):
        mean = ((torch.tensor(both[0][s], dtype=F32) + torch.tensor(both[1][s], dtype=F32)) / WORLD).item()
        assert h["loss"] == round(mean, 8), f"step {s + 1}: logged loss {h['loss']} != mean of the ranks' losses {mean}"
    # (8)
    writes = ctx.gather_obj(rec["writes"])
    assert not writes[1], f"rank 1 wrote {writes[1]}"
    for need in ("model", "optimizer", "master_weights", "rng_state_2.pth"):
        assert any(need in w for w in writes[0]), f"rank 0 did not write {need}: {writes[0]}"
    ck = os.path.join(out_dir, "checkpoint-2")
    if ctx.rank == 0:
        rng = torch.load(os.path.join(ck, "rng_state_2.pth"), weights_only=False)
        assert isinstance(rng, list) and len(rng) == WORLD and all(set(r) >= {"python", "numpy", "cpu", "cuda"} for r in rng)
        assert not os.path.exists(os.path.join(ck, "rng_state.pth"))
    res.update(steps=len(rec["log"]), losses=[h["loss"] for h in rec["log"]])
    return res


def trainer_part(ctx, family, tied, fp32, out):
    out_dir = os.path.join(out, f"{family}-{int(tied)}-{int(fp32)}")
    rec = run_trainer(ctx, family, tied, fp32, out_dir, max_steps=3, save_steps=2)
    res = check_trainer(ctx, rec, out_dir)
    # world-2 resume from checkpoint-2: step 3's loss bit-equal to the uninterrupted run's
    res_dir = out_dir + "-resumed"
    if ctx.rank == 0:
        shutil.copytree(os.path.join(out_dir, "checkpoint-2"), os.path.join(res_dir, "checkpoint-2"))
    ctx.barrier()
    r2 = run_trainer(ctx, family, tied, fp32, res_dir, max_steps=3, save_steps=0,
                     resume=os.path.join(res_dir, "checkpoint-2"))
    check_same_across_ranks(r2)
    assert [h["global_step"] for h in r2["log"]] == [1, 2, 3], r2["log"]
    assert r2["log"][2]["loss"] == rec["log"][2]["loss"], \
        f"resumed step-3 loss {r2['log'][2]['loss']} != uninterrupted {rec['log'][2]['loss']}"
    assert r2["indices"][-1] == rec["indices"][-1], "the resumed run read other samples at step 3"
    res["resumed_step3_loss_bit_equal"] = True
    return res


# ----------------------------------------------------------------------------------------------------------
def expect_raise(ctx, name, fn, match):
    try:
        fn()
    except AssertionError as e:
        msg = str(e)
        assert match in msg, f"sabotage {name!r}: the check raised, but not on {match!r}: {msg}"
        ctx.report(part="sabotage", name=name, caught=msg[:300])
        return
    raise AssertionError(f"sabotage {name!r} was not caught")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", choices=("gloo", "nccl"), required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--sabotage", action="store_true")
    opt = ap.parse_args()
    from paddlenlp_b200 import distributed as D

    if opt.backend == "gloo":
        torch.cuda.set_device(0)           # before init: init_parallel_env would pick NCCL and LOCAL_RANK's device
    D.init_parallel_env(opt.backend)
    rank = D.get_rank()
    assert D.get_world_size() == WORLD
    ctx = Ctx(rank, dist.new_group(backend="gloo"))
    log = ReduceLog()
    ctx.report(part="start", backend=opt.backend, device=torch.cuda.get_device_name(), devices=[
        r for r in ctx.gather_obj(torch.cuda.current_device())])
    for v, (family, tied, fp32) in VARIANTS.items():
        for overlap in (True, False):
            r = engine_step(ctx, log, family, tied, fp32, overlap, seed=11)
            ctx.report(part="engine", variant=v, overlap=overlap, **r)
    if opt.sabotage:
        for name, match in (("sync_gradients reduces the whole buffer again", "times in one optimizer step"),
                            ("hook armed under no_sync", "during micro-batch 0 (no_sync)")):
            expect_raise(ctx, name, lambda: engine_step(ctx, log, "llama", False, False, True, seed=11, sabotage=name,
                                                        oracle=False), match)
            log.flat = None
            ctx.barrier()
    for v, (family, tied, fp32) in VARIANTS.items():
        r = trainer_part(ctx, family, tied, fp32, opt.out)
        ctx.report(part="trainer", variant=v, amp_master_grad=fp32, **r)
    if opt.sabotage:
        from paddlenlp_b200.optimizer import AdamW

        step = AdamW.step

        def step_scale_1(self):
            self.grad_scale = 1.0
            return step(self)
        AdamW.step = step_scale_1
        try:
            rec = run_trainer(ctx, "llama", False, False, os.path.join(opt.out, "scale1"), max_steps=1, save_steps=0)
        finally:
            AdamW.step = step
        if rank == 0:
            expect_raise(ctx, "grad_scale left at 1", lambda: check_step1(rec), "with grad_scale 1/2")
        ctx.barrier()
    ctx.barrier()
    ctx.report(part="done")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
