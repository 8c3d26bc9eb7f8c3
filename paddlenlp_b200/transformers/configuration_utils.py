"""Minimal PretrainedConfig / LlmMetaConfig surface for the decoder hot path.

Mirrors paddlenlp/transformers/configuration_utils.py:317+ (PretrainedConfig: attribute bag with JSON round trip)
and :230-314 (LlmMetaConfig: runtime switches copied from TrainingArguments onto the model config).  Hub download,
sharded checkpoints and conversion are out of scope (SURVEY.md §2.1): configs are constructed, not fetched.
"""
from __future__ import annotations

import copy
import json
import os
from typing import Any, Dict

# Runtime switches the reference copies from TrainingArguments (configuration_utils.py:231-314).  They are accepted
# and stored; on this implementation every one of them maps onto the single native sm_90a path.
LLM_META_SWITCHES = {
    "use_flash_attention": True,
    "use_fused_rms_norm": True,
    "use_fused_rope": True,
    "use_fused_linear": False,
    "use_fused_dropout_add": False,
    "use_fast_layer_norm": False,
    "tensor_parallel_degree": 1,
    "pipeline_parallel_degree": 1,
    "sep_parallel_degree": 1,
    "context_parallel_degree": 1,
    "sequence_parallel": False,
    "recompute": False,
    "recompute_granularity": "full",
    "recompute_use_reentrant": False,
}


class PretrainedConfig:
    model_type: str = ""
    attribute_map: Dict[str, str] = {}

    def __init__(self, **kwargs):
        self.pad_token_id = kwargs.pop("pad_token_id", None)
        self.bos_token_id = kwargs.pop("bos_token_id", None)
        self.eos_token_id = kwargs.pop("eos_token_id", None)
        self.tie_word_embeddings = kwargs.pop("tie_word_embeddings", False)
        self.dtype = kwargs.pop("dtype", "bfloat16")
        self.return_dict = kwargs.pop("return_dict", False)
        self.output_hidden_states = kwargs.pop("output_hidden_states", False)
        self.output_attentions = kwargs.pop("output_attentions", False)
        for k, v in LLM_META_SWITCHES.items():
            setattr(self, k, kwargs.pop(k, v))
        for k, v in kwargs.items():
            setattr(self, k, v)
        for name, degree in (("tensor_parallel_degree", 1), ("pipeline_parallel_degree", 1), ("sep_parallel_degree", 1),
                             ("context_parallel_degree", 1)):
            if getattr(self, name) not in (1, -1, None):
                raise NotImplementedError(f"{name}={getattr(self, name)}: this build covers pure data parallelism only")

    def __getattr__(self, name):
        amap = type(self).attribute_map
        if name in amap:
            return getattr(self, amap[name])
        raise AttributeError(name)

    def to_dict(self) -> Dict[str, Any]:
        d = copy.deepcopy(self.__dict__)
        d["model_type"] = type(self).model_type
        return d

    def to_json_string(self) -> str:
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    def save_pretrained(self, save_directory: str):
        os.makedirs(save_directory, exist_ok=True)
        with open(os.path.join(save_directory, "config.json"), "w") as f:
            f.write(self.to_json_string())

    @classmethod
    def from_dict(cls, d: Dict[str, Any], **kwargs):
        d = dict(d)
        d.pop("model_type", None)
        d.update(kwargs)
        return cls(**d)

    @classmethod
    def from_pretrained(cls, path: str, **kwargs):
        cfg_file = os.path.join(path, "config.json") if os.path.isdir(path) else path
        if not os.path.exists(cfg_file):
            raise FileNotFoundError(f"{cfg_file}: model-hub download is out of scope; pass a local config.json")
        with open(cfg_file) as f:
            return cls.from_dict(json.load(f), **kwargs)

    def __repr__(self):
        return f"{type(self).__name__} {self.to_json_string()}"


class LlmMetaConfig:
    """set_llm_config(config, training_args): copy runtime switches (configuration_utils.py:312-314)."""

    @staticmethod
    def set_llm_config(config: PretrainedConfig, args) -> None:
        for k in LLM_META_SWITCHES:
            if hasattr(args, k):
                setattr(config, k, getattr(args, k))


def llmmetaclass(cls):
    """configuration_utils.py:294-310: class decorator that adds the LlmMetaConfig switches as dataclass fields of an
    arguments class (run_pretrain.py:60 `@llmmetaclass @dataclass class PreTrainingArguments(TrainingArguments)`).  The
    TrainingArguments of this build already carries the switches that have a meaning on the single native path; the decorator
    adds any missing one as a plain class attribute with its default so that `set_llm_config` finds it."""
    for k, v in LLM_META_SWITCHES.items():
        if not hasattr(cls, k):
            setattr(cls, k, v)
    return cls
