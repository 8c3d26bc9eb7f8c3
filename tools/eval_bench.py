"""Evaluation forward on one H100: the chunked fused path against the unfused one, at pre-training / SFT eval shapes.

    python tools/eval_bench.py --preset qwen2_1_5b --batch 8 --seq 2048
    python tools/eval_bench.py --preset llama3_2_3b --batch 2 --seq 4096

Times, with random weights, in alternating rounds after a warm-up of each:
  * eval      engine.forward_eval(predictions=True): head GEMM over row chunks + fused loss / arg-max row pass
  * eval_loss engine.forward_eval(predictions=False)
  * unfused   engine.forward_loss(keep_for_backward=False) + ops.argmax over the whole [T, V] logits
and reports each one's median time, eval tokens/s and peak allocated memory (torch.cuda.max_memory_allocated above the
weights), with the card name and power limit.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import paddlenlp_b200.transformers as T  # noqa: E402
from paddlenlp_b200 import ops  # noqa: E402
from paddlenlp_b200.transformers import decoder_engine  # noqa: E402

PRESETS = {"qwen2_1_5b": T.Qwen2Config.qwen2_1_5b, "llama3_2_3b": T.LlamaConfig.llama3_2_3b}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", choices=sorted(PRESETS), default="qwen2_1_5b")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seq", type=int, default=2048)
    ap.add_argument("--layers", type=int, default=0, help="override the layer count (0: the preset's)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    make = PRESETS[a.preset]
    cfg = make(num_hidden_layers=a.layers) if a.layers else make()
    Model = T.Qwen2ForCausalLM if a.preset.startswith("qwen2") else T.LlamaForCausalLM
    m = Model(cfg)
    eng = m.engine
    eng.init_weights(seed=42, on_host=False)
    g = torch.Generator().manual_seed(1234)
    B, S, V = a.batch, a.seq, cfg.vocab_size
    ids = torch.randint(0, V, (B, S), generator=g).cuda()
    labels = torch.randint(0, V, (B, S), generator=g).cuda()
    labels[:, : S // 4] = -100

    def eval_pred():
        return eng.forward_eval(ids, labels, predictions=True)

    def eval_loss():
        return eng.forward_eval(ids, labels, predictions=False)

    def unfused():
        loss_out, logits = eng.forward_loss(ids, labels, keep_for_backward=False)
        return loss_out, ops.argmax(logits.view(-1, V))

    paths = {"eval": eval_pred, "eval_loss": eval_loss, "unfused": unfused}
    # the three paths compute the same loss and predictions
    (l_e, p_e), (l_u, p_u) = eval_pred(), unfused()
    same = bool(torch.equal(l_e, l_u) and torch.equal(p_e.view(-1), p_u))
    peaks = {}
    for name, fn in paths.items():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del out
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n in paths}
    for _ in range(a.rounds):
        for name, fn in paths.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    T_ = B * S
    rows = max(hi - lo for lo, hi in eng._eval_chunks(T_))
    res = {"preset": a.preset, "batch": B, "seq": S, "layers": cfg.num_hidden_layers, "vocab": V, "card": _card(),
           "chunk_rows": rows, "chunk_bytes_limit": decoder_engine.EVAL_LOGITS_CHUNK_BYTES, "same_loss_and_preds": same,
           "expected_saving_gib": round((T_ - rows) * V * 2 / 2 ** 30, 3)}
    for name in paths:
        ms = statistics.median(times[name])
        res[name] = {"ms": round(ms, 3), "tokens_per_s": round(T_ / ms * 1e3, 1), "peak_gib": round(peaks[name] / 2 ** 30, 3),
                     "ms_all": [round(t, 3) for t in times[name]]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
