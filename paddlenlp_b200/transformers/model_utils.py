"""PretrainedModel base: the slice of paddlenlp/transformers/model_utils.py (:921 class, :1101 from_config-style
construction, :1140 recompute_enable) that the decoder hot path exercises.  Parameters are torch Parameters that
alias the engine's flat bf16 buffer; `.grad` aliases the flat gradient buffer, or, with fp32 gradients (set_master_grad),
`.main_grad` does and `.grad` is None."""
from __future__ import annotations

import json
import os
from typing import Dict

import torch
from torch import nn

from .decoder_engine import DecoderEngine


class _CausalLMLossFn(torch.autograd.Function):
    """Bridges `loss.backward()` (trainer.py:2243) to the engine's explicit backward."""

    @staticmethod
    def forward(ctx, anchor, engine, input_ids, labels, position_ids, ignore_index, mask_rows=None):
        loss_out, logits = engine.forward_loss(input_ids, labels, position_ids, ignore_index,
                                               attn_mask_startend_row_indices=mask_rows)
        ctx.engine = engine
        ctx.mark_non_differentiable(logits)
        return loss_out[0].clone(), logits

    @staticmethod
    def backward(ctx, gloss, _glogits):
        g = gloss.detach().to(torch.float32).reshape(1).contiguous()
        ctx.engine.backward(1.0, g)          # upstream scale stays on the device: no host sync
        return None, None, None, None, None, None, None


class _CausalLMLogitsFn(torch.autograd.Function):
    """Differentiable logits for a caller-side criterion: forward keeps the engine's activations, backward feeds d(logits)
    into the engine's explicit backward (gradients land in the flat gradient buffer, like the fused path)."""

    @staticmethod
    def forward(ctx, anchor, engine, input_ids, position_ids, mask_rows=None):
        logits = engine.forward_logits_train(input_ids, position_ids, attn_mask_startend_row_indices=mask_rows)
        ctx.engine = engine
        return logits

    @staticmethod
    def backward(ctx, glogits):
        ctx.engine.backward(1.0, None, dlogits=glogits)
        return None, None, None, None, None


class PretrainedModel(nn.Module):
    config_class = None
    base_model_prefix = ""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.training = True

    # -- construction -------------------------------------------------------------------------------
    def _build_engine(self, config, device=None):
        self.engine = DecoderEngine(config, device=device, prefix=self.base_model_prefix)
        self._anchor = nn.Parameter(torch.zeros(1, device=self.engine.device), requires_grad=True)
        self._named = {}
        grads = self.engine.named_views(grads=True)
        for name, view in self.engine.named_views().items():
            prm = nn.Parameter(view, requires_grad=True)
            prm.grad = grads[name]
            self._named[name] = prm
        seed = getattr(config, "seed", 42)
        self.engine.init_weights(seed)

    @classmethod
    def from_config(cls, config, dtype: str = "bfloat16", **kwargs):
        if dtype not in ("bfloat16", torch.bfloat16):
            raise NotImplementedError("the hot path computes in bf16 (AMP O2: parameters are created in bf16)")
        return cls(config, **kwargs)

    _from_config = from_config

    @classmethod
    def from_pretrained(cls, path, config=None, dtype="bfloat16", convert_from_hf=None, **kwargs):
        """Local directory with config.json and weights: `model.safetensors` / sharded `model-0000i-of-0000N.safetensors`
        + `model.safetensors.index.json` (the reference's unified on-disk layout, utils/env.py:97-98), or the legacy
        single `model_state.pt`.  Weights in HuggingFace naming/layout are detected (or forced with
        `convert_from_hf=True`) and converted on the fly (llama/modeling.py:1243-1274).  Hub download is out of scope."""
        from . import conversion_utils as cu

        if config is None:
            config = cls.config_class.from_pretrained(path)
        model = cls(config, **kwargs)
        if not os.path.isdir(path):
            return model
        legacy = os.path.join(path, "model_state.pt")
        if cu.has_safetensors(path):
            if convert_from_hf is None:
                convert_from_hf = cu.looks_like_hf(cu.list_keys(path))
            model._load_streaming(cu.iter_sharded(path), convert_from_hf)
        elif os.path.exists(legacy):
            model.set_state_dict(torch.load(legacy, map_location="cpu"))
        return model

    def _load_streaming(self, items, convert_from_hf: bool = False):
        """Copies (name, host tensor) pairs into the flat parameter buffer one tensor at a time."""
        from . import conversion_utils as cu

        views = self.engine.named_views()
        mt = self.engine.prefix
        seen = set()
        with torch.no_grad():
            for k, v in items:
                if convert_from_hf:
                    conv = cu.hf_to_paddle_state_dict({k: v}, mt, tie_word_embeddings=self.engine.tied)
                    if k != "lm_head.weight":
                        conv.pop("lm_head.weight", None)      # one tensor at a time: no head materialised from the embedding
                else:
                    conv = {k: v}
                for nk, nv in conv.items():
                    if nk not in views:
                        continue                      # rotary inv_freq buffers (llama/modeling.py:1240), a tied model's lm_head
                    if tuple(nv.shape) != tuple(views[nk].shape):
                        raise ValueError(f"{nk}: shape {tuple(nv.shape)} != {tuple(views[nk].shape)}")
                    views[nk].copy_(nv.to(device=self.engine.device, dtype=torch.bfloat16))
                    seen.add(nk)
        missing = [k for k in views if k not in seen]
        if missing:
            raise KeyError(f"checkpoint is missing {len(missing)} tensors, e.g. {missing[:3]}")
        self.engine.params_changed()

    def save_pretrained(self, save_directory: str, max_shard_size="5GB", safe_serialization: bool = True,
                        hf_format: bool = False, unified_checkpoint: bool = False):
        """config.json + safetensors shards + index (model_utils.py save_pretrained / shard_checkpoint :562-640).
        `hf_format=True` writes HuggingFace names and `[out, in]` Linear layouts instead of the Paddle ones.  A model with
        tied embeddings writes no `lm_head.weight`."""
        from . import conversion_utils as cu

        os.makedirs(save_directory, exist_ok=True)
        self.config.save_pretrained(save_directory)
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        if not safe_serialization:
            torch.save({k: v.cpu().contiguous() for k, v in sd.items()}, os.path.join(save_directory, "model_state.pt"))
            return
        if hf_format:
            sd = cu.paddle_to_hf_state_dict(sd, self.engine.prefix, tie_word_embeddings=self.engine.tied)
        # unified_checkpoint: always `model-0000i-of-0000N.safetensors` + index, even for one shard (the Trainer's layout)
        cu.save_sharded(sd, save_directory, max_shard_size=max_shard_size, always_index=unified_checkpoint)

    # -- parameters ---------------------------------------------------------------------------------
    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        for k, v in self._named.items():
            yield (prefix + k, v)

    def parameters(self, recurse: bool = True):
        for _, v in self.named_parameters():
            yield v

    def state_dict(self, *args, **kwargs) -> Dict[str, torch.Tensor]:
        return {k: v.detach() for k, v in self._named.items()}

    def set_state_dict(self, sd: Dict[str, torch.Tensor]):
        self.engine.load_state_dict(sd)

    load_state_dict = set_state_dict

    def num_parameters(self) -> int:
        return self.engine.num_parameters()

    def set_master_grad(self, enable: bool = True):
        """amp_master_grad: fp32 gradients (DecoderEngine.set_master_grad).  Each parameter then exposes its fp32 gradient
        view as `main_grad` and keeps `.grad = None`, the reference's convention (trainer.py:1139-1142); torch would refuse
        an fp32 `.grad` on a bf16 parameter anyway."""
        self.engine.set_master_grad(enable)
        grads = self.engine.named_views(grads=True)
        for name, prm in self._named.items():
            if enable:
                prm.grad = None
                prm.main_grad = grads[name]
            else:
                prm.grad = grads[name]
                if hasattr(prm, "main_grad"):
                    del prm.main_grad

    def recompute_enable(self):
        """model_utils.py:1140: activation recomputation — every decoder layer keeps only its input and is re-run in
        backward (llama/modeling.py:1706-1733, granularity "full")."""
        self.config.recompute = True
        self.engine.recompute = True

    def recompute_disable(self):
        self.config.recompute = False
        self.engine.recompute = False

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    # -- FLOP accounting ----------------------------------------------------------------------------
    def get_model_flops(self, batch_size=1, seq_length=None, **kwargs):
        """caculate_llm_flops (paddlenlp/transformers/utils.py:963-1003): MHA-sized, non-causal convention,
        x3 for fwd+bwd.  Kept for the reference's `interval_hardware_tflops_per_device` log key."""
        c = self.config
        s = seq_length or getattr(c, "seq_length", 2048)
        h, L, V, I = c.hidden_size, c.num_hidden_layers, c.vocab_size, c.intermediate_size
        flops_per_layer = 2 * s * h * h * 4 + 2 * s * s * h * 2 + 2 * s * h * I * 3
        return 3 * batch_size * (L * flops_per_layer + 2 * s * h * V)

    def get_algorithmic_flops_per_token(self, seq_length=None) -> float:
        """Honest count (SURVEY.md §8d): GQA-sized projections, causal attention, x3 for fwd+bwd."""
        c = self.config
        s = seq_length or getattr(c, "seq_length", 2048)
        h, L, V, I = c.hidden_size, c.num_hidden_layers, c.vocab_size, c.intermediate_size
        kvd = c.num_key_value_heads * (h // c.num_attention_heads)
        per_layer = 2 * (h * h + 2 * h * kvd + h * h + 3 * h * I) + 2 * s * h
        return 3.0 * (L * per_layer + 2 * h * V)
