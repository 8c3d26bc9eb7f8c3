"""Generate the golden fixtures of tied input / output embeddings (outputs are committed).

    python tools/make_tied_golden.py        # writes tests/golden/{llama,qwen2}_tiny_tied.pt

Same recipe and file format as oracle/make_golden.py (HuggingFace Llama / Qwen2 as the numerical twin of the reference,
tests/transformers/llama/test_modeling.py:398-506), with `tie_word_embeddings=True`: the HF model's lm_head shares the
embedding matrix, so the weights carry no `lm_head.weight` and the embedding gradient holds both the lookup's scatter and
the head's `dlogits^T @ hidden` term (llama/modeling.py:1924-1938, LlamaLMHead(embedding_weights=..., transpose_y=True)).
tests/test_tied_embeddings_cpu.py checks the tied oracle (tests/tied_oracle.py) against these, with no transformers import
needed.  oracle/make_golden.py and the untied fixtures it wrote are left as they are: they pin the untied oracle every other
test uses, and a change to that recipe would change the yardstick of the untied path.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import llama_ref as R  # noqa: E402


def make(model_type: str, path: str):
    import transformers

    cfg = R.RefConfig(vocab_size=160, hidden_size=64, intermediate_size=176, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, rope_theta=500000.0 if model_type == "llama" else 1e6,
                      qkv_bias=(model_type == "qwen2"), model_type=model_type,
                      rms_norm_eps=1e-5 if model_type == "llama" else 1e-6, max_position_embeddings=64)
    w = R.init_weights(cfg, seed=2025, round_bf16=True)
    w.pop("lm_head.weight")
    g = torch.Generator().manual_seed(8)
    for k in w:
        if "norm" in k:
            w[k] = (1.0 + 0.1 * torch.randn(w[k].shape, generator=g)).to(torch.bfloat16).float()
        elif k.endswith("weight"):
            w[k] = (w[k] * 4.0).to(torch.bfloat16).float()        # non-degenerate logits
    hcfg = R.hf_config(cfg)
    hcfg.tie_word_embeddings = True
    cls = transformers.Qwen2ForCausalLM if model_type == "qwen2" else transformers.LlamaForCausalLM
    m = cls(hcfg).float().eval()
    res = m.load_state_dict(R.to_hf_state_dict(w, cfg), strict=False)
    assert not res.unexpected_keys and set(res.missing_keys) <= {"lm_head.weight"}, res
    m.tie_weights()
    assert m.lm_head.weight.data_ptr() == m.model.embed_tokens.weight.data_ptr(), "HF model did not tie its head"
    tok = torch.randint(0, cfg.vocab_size, (2, 33), generator=g)
    ids, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    labels[1, :5] = -100
    logits = m(input_ids=ids).logits
    loss = R.criterion(logits, labels)
    loss.backward()
    hf_grads = {k: v.grad.clone() for k, v in m.named_parameters()}   # the shared matrix is listed once (embed_tokens)
    grads = {}
    for k in w:
        hk = ("model." + k[len(cfg.model_type) + 1:]) if k.startswith(cfg.model_type + ".") else k
        gk = hf_grads[hk]
        grads[k] = gk.t().contiguous() if k.endswith("_proj.weight") else gk
    torch.save({"config": {**cfg.__dict__, "tie_word_embeddings": True},
                "weights": {k: v.to(torch.bfloat16) for k, v in w.items()}, "input_ids": ids,
                "labels": labels, "hf_logits_fp32": logits.detach(), "loss_fp32": loss.detach(),
                "grads_fp32": {k: v.to(torch.float32) for k, v in grads.items()},
                "generator": f"tools/make_tied_golden.py, transformers {transformers.__version__}, torch {torch.__version__}"},
               path)
    print(path, os.path.getsize(path), "bytes; loss", float(loss))


if __name__ == "__main__":
    out = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out, exist_ok=True)
    make("llama", os.path.join(out, "llama_tiny_tied.pt"))
    make("qwen2", os.path.join(out, "qwen2_tiny_tied.pt"))
