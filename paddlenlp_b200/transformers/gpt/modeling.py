"""GPT-2 modeling classes for BASELINE.json configs[0] — the reference's own CPU-runnable plumbing case
(GPT-2-small forward + loss, batch 2 x seq 128, fp32, no custom kernels; SURVEY.md §3.5 / §8 row a15).

Surface of paddlenlp/transformers/gpt/modeling.py: GPTEmbeddings :715-774 (word + learned position), MultiHeadAttention
:183-445 (`_core_attention` :350-385: q * d^-0.5 @ k^T + triangular mask, softmax, @ v; q/k/v/out Linear with bias),
GPTDecoderLayer :567-712 (pre-LN, tanh-GELU MLP), final LayerNorm(eps 1e-5) :455, GPTLMHead :1461-1503 (tied to the word
embeddings), GPTPretrainingCriterion :1323-1363 (ignore_index defaults to 0; mean over loss > 0), GPTForCausalLM :1506-1620.
This path is plain fp32 torch by design: the reference runs it on the CPU through Paddle's CPU kernels, there is nothing
to accelerate and no GPU kernel is involved.  Linear weights keep Paddle's [in, out] layout and parameter names.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from ..model_outputs import CausalLMOutputWithCrossAttentions
from .configuration import GPTConfig

__all__ = ["GPTModel", "GPTForCausalLM", "GPTPretrainingCriterion", "GPTLMHeadModel"]


class _Linear(nn.Module):
    """paddle.nn.Linear: y = x @ W + b with W stored [in_features, out_features]."""

    def __init__(self, i, o):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(i, o))
        self.bias = nn.Parameter(torch.zeros(o))

    def forward(self, x):
        return x @ self.weight + self.bias


class MultiHeadAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = config.hidden_size
        self.num_heads, self.head_dim, self.scale_qk_coeff = config.num_attention_heads, h // config.num_attention_heads, config.scale_qk_coeff
        self.q_proj, self.k_proj, self.v_proj, self.out_proj = _Linear(h, h), _Linear(h, h), _Linear(h, h), _Linear(h, h)

    def forward(self, x):
        b, s, h = x.shape
        shp = (b, s, self.num_heads, self.head_dim)
        q, k, v = (p(x).view(shp).transpose(1, 2) for p in (self.q_proj, self.k_proj, self.v_proj))
        product = (q * ((self.scale_qk_coeff * self.head_dim) ** -0.5)) @ k.transpose(-1, -2)
        if self.scale_qk_coeff != 1.0:
            product = product * self.scale_qk_coeff
        mask = torch.full((s, s), torch.finfo(product.dtype).min, dtype=product.dtype, device=x.device).triu(1)
        weights = F.softmax(product + mask, dim=-1)
        out = (weights @ v).transpose(1, 2).reshape(b, s, h)
        return self.out_proj(out)


class GPTDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = config.hidden_size
        self.self_attn = MultiHeadAttention(config)
        self.linear1, self.linear2 = _Linear(h, config.intermediate_size), _Linear(config.intermediate_size, h)
        self.norm1, self.norm2 = nn.LayerNorm(h, eps=1e-5), nn.LayerNorm(h, eps=1e-5)

    def forward(self, x):
        x = x + self.self_attn(self.norm1(x))
        return x + self.linear2(F.gelu(self.linear1(self.norm2(x)), approximate="tanh"))


class _Decoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layers = nn.ModuleList([GPTDecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = nn.LayerNorm(config.hidden_size, eps=1e-5)

    def forward(self, x):
        for layer in self.layers:
            x = layer(x)
        return self.norm(x)


class _Embeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)

    def forward(self, input_ids, position_ids=None):
        if position_ids is None:
            position_ids = torch.arange(input_ids.shape[1], device=input_ids.device).unsqueeze(0).expand_as(input_ids)
        return self.word_embeddings(input_ids) + self.position_embeddings(position_ids)


class GPTModel(nn.Module):
    config_class = GPTConfig

    def __init__(self, config: GPTConfig):
        super().__init__()
        self.config = config
        self.embeddings = _Embeddings(config)
        self.decoder = _Decoder(config)
        std = config.initializer_range
        for name, p in self.named_parameters():                      # GPTPretrainedModel._init_weights: N(0, 0.02), LN = 1/0
            if name.endswith("bias"):
                nn.init.zeros_(p)
            elif "norm" in name:
                nn.init.ones_(p)
            else:
                nn.init.normal_(p, 0.0, std)

    def forward(self, input_ids, position_ids=None, attention_mask=None, **kw):
        if attention_mask is not None and attention_mask.dim() > 2:
            raise NotImplementedError("only the causal mask is implemented")
        return self.decoder(self.embeddings(input_ids, position_ids))


class GPTPretrainingCriterion(nn.Module):
    """gpt/modeling.py:1323-1363: fp32 CE, ignore_index = config.ignore_index (default 0), mean over loss > 0."""

    def __init__(self, config: GPTConfig):
        super().__init__()
        self.ignore_index = config.ignore_index

    def forward(self, prediction_scores, masked_lm_labels, loss_mask=None):
        per = F.cross_entropy(prediction_scores.float().reshape(-1, prediction_scores.shape[-1]), masked_lm_labels.reshape(-1),
                              reduction="none", ignore_index=self.ignore_index)
        if loss_mask is None:
            loss_mask = (per > 0).float()
        return (per * loss_mask.reshape(-1)).sum() / loss_mask.sum()


class GPTForCausalLM(nn.Module):
    config_class = GPTConfig

    def __init__(self, config: GPTConfig):
        super().__init__()
        self.config = config
        self.gpt = GPTModel(config)
        self.criterion = GPTPretrainingCriterion(config)

    @classmethod
    def from_config(cls, config, dtype="float32", **kw):
        return cls(config)

    def forward(self, input_ids=None, position_ids=None, attention_mask=None, labels=None, return_dict=False, **kw):
        hidden = self.gpt(input_ids, position_ids, attention_mask)
        logits = hidden @ self.gpt.embeddings.word_embeddings.weight.t()      # GPTLMHead: tied, transpose_y=True
        loss = self.criterion(logits, labels) if labels is not None else None
        if return_dict:
            return CausalLMOutputWithCrossAttentions(loss=loss, logits=logits)
        return (loss, logits) if loss is not None else (logits,)


GPTLMHeadModel = GPTForCausalLM
