"""The tied-embedding oracle shared by tests/test_tied_embeddings_cpu.py and tests/test_tied_embeddings_gpu.py (TEST
INFRASTRUCTURE ONLY, like oracle/).

It is oracle/llama_ref.py used unchanged, with the head bound to the embedding: `lm_head.weight` = E^T, a view of
E = `<model_type>.embed_tokens.weight`, so logits = hf @ E^T (llama/modeling.py:1924-1938, LlamaLMHead(transpose_y=True)) and
autograd sums the lookup's scatter and the head's term into the one matrix E.  The untied oracle stays byte-for-byte the one
every other test checks against; this module adds no arithmetic of its own.  It is pinned to HuggingFace with tied embeddings
by tests/golden/{llama,qwen2}_tiny_tied.pt (tools/make_tied_golden.py)."""
import os

import torch

from oracle import llama_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def embed_key(cfg) -> str:
    return f"{cfg.model_type}.embed_tokens.weight"


def bind_head(w, cfg):
    """The untied oracle's weight dict with `lm_head.weight` = E^T (a view: gradients flow into E)."""
    return {**{k: v for k, v in w.items() if k != "lm_head.weight"}, "lm_head.weight": w[embed_key(cfg)].t()}


def tied_forward(input_ids, w, cfg, mode="bf16", **kw):
    return R.model_forward(input_ids, bind_head(w, cfg), cfg, mode, **kw)


def tied_loss_and_grads(input_ids, labels, w, cfg, mode="bf16"):
    """Forward + autograd backward of the tied oracle: the gradient of E holds both terms.  A `lm_head.weight` in `w` is
    ignored."""
    wl = {k: v.clone().requires_grad_(True) for k, v in w.items() if k != "lm_head.weight"}
    logits = R.model_forward(input_ids, bind_head(wl, cfg), cfg, mode)
    loss = R.criterion(logits, labels)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in wl.items()}


def load_golden(name):
    """A tied fixture: (raw dict, RefConfig, fp32 weights without lm_head.weight)."""
    d = torch.load(os.path.join(GOLD, name), map_location="cpu", weights_only=False)
    c = dict(d["config"])
    assert c.pop("tie_word_embeddings") is True
    cfg = R.RefConfig(**c)
    w = {k: v.float() for k, v in d["weights"].items()}
    return d, cfg, w
