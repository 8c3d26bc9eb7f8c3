"""Weight-file plumbing for the decoder path: HF <-> Paddle name/layout conversion and sharded safetensors I/O.

Reference behaviour restated here:
* name map + transposes between HuggingFace (`model.layers.N...`, Linear weights `[out, in]`) and PaddleNLP
  (`llama.layers.N...` / `qwen2.layers.N...`, Linear weights `[in, out]`): `LlamaPretrainedModel._get_name_mappings`
  llama/modeling.py:1243-1274, `Qwen2PretrainedModel._get_name_mappings` qwen2/modeling.py (same table + q/k/v biases);
* on-disk layout: one `model.safetensors`, or `model-0000i-of-0000N.safetensors` shards plus
  `model.safetensors.index.json` = {"metadata": {"total_size": bytes}, "weight_map": {name: shard file}}
  (`shard_checkpoint` transformers/model_utils.py:562-640, names from utils/env.py:97-110).
"""
from __future__ import annotations

import json
import os
import re
from typing import Dict, Iterable, List, Tuple

import torch

SAFE_WEIGHTS_NAME = "model.safetensors"
SAFE_WEIGHTS_INDEX_NAME = "model.safetensors.index.json"
SAFE_OPTIMIZER_NAME = "optimizer.safetensors"
SAFE_OPTIMIZER_INDEX_NAME = "optimizer.safetensors.index.json"
SAFE_MASTER_WEIGHTS_NAME = "master_weights.safetensors"
SAFE_MASTER_WEIGHTS_INDEX_NAME = "master_weights.safetensors.index.json"

_TRANSPOSED = re.compile(r"(_proj\.weight|^lm_head\.weight)$")
_IGNORED = re.compile(r"self_attn\.rotary_emb\.inv_freq$")          # llama/modeling.py:1240


def _is_linear(name: str) -> bool:
    return bool(_TRANSPOSED.search(name))


def hf_to_paddle_state_dict(sd: Dict[str, torch.Tensor], model_type: str,
                            tie_word_embeddings: bool = False) -> Dict[str, torch.Tensor]:
    """`model.X` -> `<model_type>.X`, Linear weights transposed to `[in, out]`; `lm_head.weight` kept at top level.
    Tied embeddings (llama/modeling.py:1270-1271): the mapping has no lm_head, so a stray `lm_head.weight` is dropped.
    Untied: a tied-embedding checkpoint (no lm_head.weight) gets a separate head materialised from the embedding."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in sd.items():
        if _IGNORED.search(k) or (tie_word_embeddings and k == "lm_head.weight"):
            continue
        nk = (model_type + k[len("model"):]) if k.startswith("model.") else k
        out[nk] = v.t().contiguous() if _is_linear(nk) else v
    if not tie_word_embeddings and "lm_head.weight" not in out and f"{model_type}.embed_tokens.weight" in out:
        out["lm_head.weight"] = out[f"{model_type}.embed_tokens.weight"].t().contiguous()
    return out


def paddle_to_hf_state_dict(sd: Dict[str, torch.Tensor], model_type: str,
                            tie_word_embeddings: bool = False) -> Dict[str, torch.Tensor]:
    """Inverse of hf_to_paddle_state_dict; a tied model's state dict maps to one without `lm_head.weight`."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in sd.items():
        if tie_word_embeddings and k == "lm_head.weight":
            continue
        nk = ("model" + k[len(model_type):]) if k.startswith(model_type + ".") else k
        out[nk] = v.t().contiguous() if _is_linear(k) else v
    return out


def looks_like_hf(keys: Iterable[str]) -> bool:
    return any(k.startswith("model.") for k in keys)


# ----------------------------------------------------------------------------------------------------------
# sharded safetensors
# ----------------------------------------------------------------------------------------------------------
def parse_size(size) -> int:
    """"5GB" / "500MB" / int bytes (convert_file_size_to_int, transformers/model_utils.py)."""
    if isinstance(size, int):
        return size
    m = re.fullmatch(r"\s*(\d+(?:\.\d+)?)\s*([KMGT]i?B)\s*", str(size), re.IGNORECASE)
    if not m:
        raise ValueError(f"size must be an int or like '5GB', got {size!r}")
    unit = m.group(2).upper()
    base = 1024 if "I" in unit else 1000
    return int(float(m.group(1)) * base ** ("KMGT".index(unit[0]) + 1))


def plan_shards(sizes: List[Tuple[str, int]], max_shard_size) -> List[List[str]]:
    """Greedy in-order packing (shard_checkpoint: a new shard starts when the next tensor would overflow; a tensor larger
    than the limit gets a shard of its own)."""
    limit = parse_size(max_shard_size)
    shards: List[List[str]] = [[]]
    cur = 0
    for name, nbytes in sizes:
        if shards[-1] and cur + nbytes > limit:
            shards.append([])
            cur = 0
        shards[-1].append(name)
        cur += nbytes
    return shards


def _shard_name(base: str, i: int, n: int) -> str:
    stem, ext = os.path.splitext(base)
    return f"{stem}-{i + 1:05d}-of-{n:05d}{ext}"


def save_sharded(tensors: Dict[str, torch.Tensor], directory: str, weights_name: str = SAFE_WEIGHTS_NAME,
                 index_name: str = SAFE_WEIGHTS_INDEX_NAME, max_shard_size="5GB", always_index: bool = False) -> List[str]:
    """Writes `tensors` (any device; each is copied to the host when its shard is written, so peak host memory is one
    shard) and returns the list of files written.  A single shard is written as the bare `weights_name` (what
    `save_pretrained` / shard_checkpoint do, model_utils.py:562-640) unless `always_index`: the Trainer's unified checkpoint
    always writes `<stem>-00001-of-0000N<ext>` plus the index, and its loader requires the index
    (trainer/plugins/unified_checkpoint.py:301-423, select_model_weight_index)."""
    from safetensors.torch import save_file

    os.makedirs(directory, exist_ok=True)
    sizes = [(k, v.numel() * v.element_size()) for k, v in tensors.items()]
    shards = plan_shards(sizes, max_shard_size)
    for stale in os.listdir(directory):            # a previous save with a different shard count must not linger
        stem, ext = os.path.splitext(weights_name)
        if stale == weights_name or stale == index_name or re.fullmatch(re.escape(stem) + r"-\d{5}-of-\d{5}" + re.escape(ext), stale):
            os.remove(os.path.join(directory, stale))
    written = []
    if len(shards) == 1 and not always_index:
        save_file({k: tensors[k].detach().cpu().contiguous() for k in shards[0]}, os.path.join(directory, weights_name),
                  metadata={"format": "pt"})
        return [weights_name]
    weight_map = {}
    for i, names in enumerate(shards):
        fname = _shard_name(weights_name, i, len(shards))
        save_file({k: tensors[k].detach().cpu().contiguous() for k in names}, os.path.join(directory, fname),
                  metadata={"format": "pt"})
        written.append(fname)
        for k in names:
            weight_map[k] = fname
    index = {"metadata": {"total_size": sum(n for _, n in sizes)}, "weight_map": weight_map}
    with open(os.path.join(directory, index_name), "w", encoding="utf-8") as f:
        f.write(json.dumps(index, indent=2, sort_keys=True) + "\n")
    written.append(index_name)
    return written


def iter_sharded(directory: str, weights_name: str = SAFE_WEIGHTS_NAME, index_name: str = SAFE_WEIGHTS_INDEX_NAME):
    """Yields (name, host tensor) from a single-file or sharded safetensors checkpoint, one shard resident at a time."""
    from safetensors import safe_open

    single = os.path.join(directory, weights_name)
    index = os.path.join(directory, index_name)
    if os.path.isfile(index):
        with open(index, encoding="utf-8") as f:
            files = sorted(set(json.load(f)["weight_map"].values()))
    elif os.path.isfile(single):
        files = [weights_name]
    else:
        raise FileNotFoundError(f"no {weights_name} or {index_name} under {directory}")
    for fname in files:
        path = os.path.join(directory, fname)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"{index_name} lists {fname}, which is missing from {directory}")
        with safe_open(path, framework="pt", device="cpu") as f:
            for k in f.keys():
                yield k, f.get_tensor(k)


def list_keys(directory: str, weights_name: str = SAFE_WEIGHTS_NAME, index_name: str = SAFE_WEIGHTS_INDEX_NAME) -> List[str]:
    """Tensor names of a checkpoint without reading any tensor data."""
    from safetensors import safe_open

    index = os.path.join(directory, index_name)
    if os.path.isfile(index):
        with open(index, encoding="utf-8") as f:
            return list(json.load(f)["weight_map"])
    with safe_open(os.path.join(directory, weights_name), framework="pt", device="cpu") as f:
        return list(f.keys())


def load_sharded(directory: str, weights_name: str = SAFE_WEIGHTS_NAME, index_name: str = SAFE_WEIGHTS_INDEX_NAME):
    return dict(iter_sharded(directory, weights_name, index_name))


def has_safetensors(directory: str, weights_name: str = SAFE_WEIGHTS_NAME, index_name: str = SAFE_WEIGHTS_INDEX_NAME):
    return os.path.isfile(os.path.join(directory, weights_name)) or os.path.isfile(os.path.join(directory, index_name))
