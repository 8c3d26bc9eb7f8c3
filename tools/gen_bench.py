"""Config 5: Llama-3-8B generation decode, 1xH100, batch 64, prompt 128 -> gen 1920 (FusedMultiTransformer KV-cache path).
`--preset llama3_2_1b` / `qwen2_0_5b` runs the same workload on the head_dim 64 models (tied embeddings, as released).

Reports prefill time, decode tokens/s = B * (gen - 1) / decode time, and the HBM roofline of the decode step
(weights 15.01 GB + KV read 8.39 MB * t per step; SURVEY.md §8d)."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import paddlenlp_b200.transformers as T  # noqa: E402
from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel  # noqa: E402


PRESETS = {"llama3_8b": T.LlamaConfig.llama3_8b, "llama3_2_1b": T.LlamaConfig.llama3_2_1b, "qwen2_0_5b": T.Qwen2Config.qwen2_0_5b}


def run(batch=64, prompt=128, gen=1920, layers=0, graph=True, pdl=True, block_attn=False, preset="llama3_8b", quant_type="",
        cachekv_int8=False):
    class A:
        pass
    a = A()
    a.batch, a.prompt, a.gen, a.layers, a.no_graph, a.no_pdl, a.block_attn = batch, prompt, gen, layers, not graph, not pdl, block_attn
    a.preset, a.quant_type, a.cachekv_int8 = preset, quant_type, cachekv_int8
    return _run(a)


def _run(a):
    make = PRESETS[a.preset]
    cfg = make(num_hidden_layers=a.layers) if a.layers else make()
    if a.cachekv_int8 and not a.block_attn:
        raise SystemExit("--cachekv-int8 needs --block-attn (the int8 cache is paged)")
    m = LlamaForCausalLMInferenceModel(cfg, block_attn=a.block_attn, quant_type=a.quant_type,
                                       cachekv_int8_type="static" if a.cachekv_int8 else None)
    m.init_random(seed=42)
    g = torch.Generator().manual_seed(1234)
    ids = torch.randint(0, cfg.vocab_size, (a.batch, a.prompt), generator=g).cuda()
    if a.cachekv_int8:
        m.calibrate_cache_scales(ids)                      # static scales from the benchmark's own prompts
    max_len = a.prompt + a.gen
    caches = m.allocate_caches(a.batch, max_len)
    # warm-up (kernel attributes, allocator)
    m.generate(ids, max_length=min(8, a.gen), eos_token_id=-1, cache_kvs=caches, use_cuda_graph=not a.no_graph, use_pdl=not a.no_pdl)
    torch.cuda.synchronize()
    # prefill alone
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    enc = torch.full((a.batch,), a.prompt, dtype=torch.int32, device="cuda")
    e0.record()
    m._prefill(ids, enc, caches)
    e1.record()
    torch.cuda.synchronize()
    prefill_ms = e0.elapsed_time(e1)
    e0.record()
    out, stop, dec = m.generate(ids, max_length=a.gen, eos_token_id=-1, cache_kvs=caches, use_cuda_graph=not a.no_graph,
                                sync_interval=0, use_pdl=not a.no_pdl)
    e1.record()
    torch.cuda.synchronize()
    total_ms = e0.elapsed_time(e1)
    decode_ms = total_ms - prefill_ms
    steps = a.gen - 1
    L = cfg.num_hidden_layers
    h, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    kvd = cfg.num_key_value_heads * (h // cfg.num_attention_heads)
    layer_params = L * (h * (h + 2 * kvd) + h * h + 3 * h * I)
    # int8 layer weights: one byte each plus a bf16 scale per output channel; embeddings and head stay bf16
    w_bytes = (layer_params + L * (h + 2 * kvd + h + 2 * I + h) * 2 if a.quant_type else layer_params * 2) + V * h * 2
    kv_per_tok = 2 * L * a.batch * kvd * (1 if a.cachekv_int8 else 2)
    mean_t = a.prompt + steps / 2.0
    bytes_per_step = w_bytes + kv_per_tok * mean_t
    # H100 SXM data-sheet HBM3 bandwidth unless a measured peak is supplied next to the repository
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0}
    ms_step = decode_ms / steps
    achieved = bytes_per_step / (ms_step / 1e3) / 1e9
    rec = dict(workload="Llama-3-8B generation decode, batch 64, prompt 128 -> +1920, FusedMultiTransformer KV-cache path "
                        "(BASELINE.json configs[4])" if (a.batch, a.prompt, a.gen, a.layers, a.preset) == (64, 128, 1920, 0, "llama3_8b")
               else f"{a.preset} decode, batch {a.batch}, prompt {a.prompt} -> +{a.gen}",
               batch=a.batch, prompt=a.prompt, gen=a.gen, layers=L, paged_kv=bool(a.block_attn), quant_type=a.quant_type,
               cachekv_int8_type="static" if a.cachekv_int8 else None,
               prefill_ms=prefill_ms, decode_ms=decode_ms,
               ms_per_step=ms_step,
               decode_tokens_per_s=a.batch * steps / (decode_ms / 1e3), bytes_per_step_gb=bytes_per_step / 1e9,
               achieved_gbs=achieved, hbm_peak_gbs=peaks["hbm_gbs"], roofline_frac=achieved / peaks["hbm_gbs"],
               graph=not a.no_graph, pdl=not a.no_pdl, mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30, last_tokens=out[0, -4:].tolist())
    del m, caches
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--gen", type=int, default=1920)
    ap.add_argument("--layers", type=int, default=0)
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-pdl", action="store_true")
    ap.add_argument("--preset", choices=sorted(PRESETS), default="llama3_8b")
    ap.add_argument("--block-attn", action="store_true", help="paged KV cache (FusedBlockMultiTransformer, 64-row blocks)")
    ap.add_argument("--quant-type", default="", choices=["", "weight_only_int8"],
                    help="weight_only_int8: int8 layer weights with per-channel scales (FusedMultiTransformerWeightOnly)")
    ap.add_argument("--cachekv-int8", action="store_true",
                    help="uint8 paged KV cache with static per-head scales calibrated on the benchmark's prompts (needs --block-attn)")
    a = ap.parse_args()
    print(json.dumps(_run(a)), flush=True)


if __name__ == "__main__":
    main()
