"""Probe: full-width Llama-3-8B layers (reduced depth) fwd+bwd timing on one H100, with extrapolation to 32 layers."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import paddlenlp_b200.transformers as T  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--model", default="llama")
    a = ap.parse_args()
    if a.model == "llama":
        cfg = T.LlamaConfig.llama3_8b(num_hidden_layers=a.layers)
        model = T.LlamaForCausalLM(cfg)
    else:
        cfg = T.Qwen2Config.qwen2_7b(num_hidden_layers=a.layers)
        model = T.Qwen2ForCausalLM(cfg)
    eng = model.engine
    g = torch.Generator().manual_seed(1234)
    tok = torch.randint(0, cfg.vocab_size, (a.batch, a.seq + 1), generator=g)
    ids, labels = tok[:, :-1].contiguous().cuda(), tok[:, 1:].contiguous().cuda()

    def fwd():
        return eng.forward_loss(ids, labels)

    def step():
        eng.forward_loss(ids, labels)
        eng.backward(1.0)

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tf = tb = 0.0
    t0 = time.time()
    for _ in range(a.iters):
        e[0].record()
        eng.forward_loss(ids, labels)
        e[1].record()
        eng.backward(1.0)
        e[2].record()
        torch.cuda.synchronize()
        tf += e[0].elapsed_time(e[1])
        tb += e[1].elapsed_time(e[2])
    wall = (time.time() - t0) / a.iters * 1e3
    tf /= a.iters
    tb /= a.iters
    loss = eng.forward_loss(ids, labels, keep_for_backward=False)[0][0].item()
    T_ = a.batch * a.seq
    rec = dict(model=a.model, layers=a.layers, tokens=T_, fwd_ms=tf, bwd_ms=tb, wall_ms=wall, loss=loss,
               mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(json.dumps(rec), flush=True)
    if a.layers >= 2:
        # second measurement with half the layers to separate per-layer cost from head/embedding cost
        pass


if __name__ == "__main__":
    main()
