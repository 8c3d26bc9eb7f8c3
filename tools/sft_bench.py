"""Config 4: Qwen2-1.5B full-parameter SFT, bf16, seq 2048, through the Trainer API with synthetic instruction pairs
(Qwen2-7B, the BASELINE.json size, needs 122 GB of weights and AdamW state: more than one H100 holds).

    python tools/sft_bench.py [--steps 4 --micro-batch 4 --accum 2]           # 1 GPU
    python -m torch.distributed.run --nproc-per-node N tools/sft_bench.py     # pure data parallel

Synthetic data (SURVEY.md §8d): src_len ~ U{64..1024}, tgt_len ~ U{16..2048-src_len}, labels = [-100]*src + tgt shifted
by one (llm/utils/data.py:196-199), right-padded to 2048 with pad id / -100 (DataCollatorForSeq2Seq semantics).
tokens/s counts all 2048 positions (the reference's speed_metrics convention) and, separately, non-pad tokens."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import paddlenlp_b200.transformers as T  # noqa: E402
from paddlenlp_b200.trainer import Trainer, TrainingArguments  # noqa: E402

S = 2048


class SyntheticSFT(torch.utils.data.Dataset):
    def __init__(self, n, vocab, seed=1234):
        g = torch.Generator().manual_seed(seed)
        self.items = []
        for _ in range(n):
            src = int(torch.randint(64, 1025, (1,), generator=g))
            tgt = int(torch.randint(16, S - src + 1, (1,), generator=g))
            toks = torch.randint(1, vocab, (src + tgt,), generator=g)
            labels = torch.cat([torch.full((src,), -100), toks[src:]])
            ids, lab = toks[:-1], labels[1:]                       # shift by one
            pad = S - ids.numel()
            self.items.append((torch.cat([ids, torch.zeros(pad, dtype=torch.int64)]),
                               torch.cat([lab, torch.full((pad,), -100)]), src + tgt - 1))

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return {"input_ids": self.items[i][0], "labels": self.items[i][1]}


def run(steps=4, warmup=2, micro_batch=4, accum=2, layers=0, zero_padding=False, quiet=False):
    """Train `warmup + steps` optimizer steps through Trainer.train(); returns the record (rank 0) / None (other ranks)."""
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    args = TrainingArguments(output_dir="/tmp/sft_out", per_device_train_batch_size=micro_batch,
                             gradient_accumulation_steps=accum, max_steps=steps + warmup, learning_rate=3e-5,
                             weight_decay=0.01, warmup_steps=1, logging_steps=1, max_seq_length=S, lr_scheduler_type="linear")
    cfg = T.Qwen2Config.qwen2_1_5b(num_hidden_layers=layers) if layers else T.Qwen2Config.qwen2_1_5b()
    model = T.AutoModelForCausalLM.from_config(cfg, dtype="bfloat16")
    n = (steps + warmup) * micro_batch * accum * args.world_size
    collator = None
    if zero_padding:
        from paddlenlp_b200.data import DataCollatorForSeq2Seq
        from paddlenlp_b200.datasets import ZeroPaddingMapDataset

        raw = SyntheticSFT(3 * n, cfg.vocab_size)                    # ~2-3 samples fit one row
        recs = [{"input_ids": it[0][: it[2]].tolist(), "labels": it[1][: it[2]].tolist()} for it in raw.items]
        packed = ZeroPaddingMapDataset(recs, max_length=S, greedy_zero_padding=True)
        packed.new_data = packed.new_data[:n]
        assert len(packed) >= n, "not enough packed rows"
        real = [len(r["input_ids"]) for r in packed.new_data]
        ds = packed
        ds.items = [(None, None, r) for r in real]
        collator = DataCollatorForSeq2Seq(max_length=S, pad_token_id=0)
    else:
        ds = SyntheticSFT(n, cfg.vocab_size)
    trainer = Trainer(model=model, args=args, train_dataset=ds, data_collator=collator)
    if quiet:
        from paddlenlp_b200.trainer.trainer import PrinterCallback
        trainer.callbacks = [c for c in trainer.callbacks if not isinstance(c, PrinterCallback)]
    trainer.train()
    hist = trainer.state.log_history[warmup:]
    rec = None
    if args.process_index == 0:
        sps = sum(h["interval_samples_per_second"] for h in hist) / len(hist)
        nonpad = sum(it[2] for it in ds.items) / len(ds.items)
        rec = dict(workload="Qwen2-1.5B full-parameter SFT bf16 through Trainer.train(), synthetic instruction pairs "
                            "(BASELINE.json configs[3])",
                   model="Qwen2-1.5B" if not layers else f"Qwen2-1.5B width, {layers} layers", n_gpus=args.world_size,
                   seq_len=S, zero_padding=bool(zero_padding), micro_batch=micro_batch, grad_accum=accum, steps=steps,
                   global_batch=micro_batch * accum * args.world_size,
                   tokens_per_s=sps * S, nonpad_tokens_per_s=sps * nonpad, loss_first=hist[0]["loss"], loss_last=hist[-1]["loss"],
                   tflops_per_gpu=sps * S / args.world_size * model.get_algorithmic_flops_per_token(S) / 1e12,
                   timing="host wall clock between log steps (Trainer speed_metrics, logging_steps=1 => one loss read per step)",
                   mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    del trainer, model
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--micro-batch", type=int, default=4)
    ap.add_argument("--accum", type=int, default=2)
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--zero-padding", action="store_true",
                    help="pack samples into 2048-token rows (ZeroPaddingMapDataset + FlashMask), llm/run_finetune.py --zero_padding")
    a = ap.parse_args()
    rec = run(a.steps, a.warmup, a.micro_batch, a.accum, a.layers, a.zero_padding)
    if rec is not None:
        print(json.dumps(rec), flush=True)
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
