"""Per-op plug-in seam of the Llama training path (reference: paddlenlp/transformers/llama/fusion_ops.py).

The reference lets a vendor back-end replace four ops behind fixed Python signatures — `fusion_rms_norm` (:128-144),
`fusion_rope` (:57-116), `fusion_flash_attention` (:147-267) and `swiglu` (llama/modeling.py:38-45).  This module keeps
those names, argument orders and error behaviour and forwards each one to a `torch.autograd.Function` whose forward and
backward are single C-ABI calls into libb200nlp.so (include/b200nlp.h).  The fused whole-block path
(`DecoderEngine`) bypasses this seam; the two are tested to agree.

Tensors are CUDA bf16; there is no CPU fallback (a missing extension raises `B200Error`).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from ... import ops

__all__ = ["fusion_rms_norm", "fusion_rope", "fusion_flash_attention", "swiglu", "LlamaRotaryEmbedding", "LlamaRMSNorm"]


# ----------------------------------------------------------------------------------------------------------
# RMSNorm  (fused_ln.fused_rms_norm, legacy/model_zoo/gpt-3/external_ops/fused_ln/layer_norm_cuda.cu:164-239)
# ----------------------------------------------------------------------------------------------------------
class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        xc = x.contiguous()
        y, rstd = ops.rmsnorm_fwd(xc, weight, eps)
        ctx.save_for_backward(xc, weight, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, rstd = ctx.saved_tensors
        dw = torch.empty_like(weight)
        dx = ops.rmsnorm_bwd(dy.contiguous(), x, weight, rstd, dw, accumulate_dw=False)
        return dx, dw, None


def fusion_rms_norm(hidden_states, weight, variance_epsilon, use_fast_ln=False):
    """y = w * bf16(x * rsqrt(mean(x^2) + eps)); fp32 statistics.  `use_fast_ln` selects an apex kernel variant in the
    reference (fusion_ops.py:144) with the same math; it is accepted and ignored."""
    return _RMSNormFn.apply(hidden_states, weight, float(variance_epsilon))


class LlamaRMSNorm(torch.nn.Module):
    """llama/modeling.py:352-386 with `use_fused_rms_norm` always on."""

    def __init__(self, config, device="cuda"):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.weight = torch.nn.Parameter(torch.ones(self.hidden_size, dtype=torch.bfloat16, device=device))
        self.variance_epsilon = config.rms_norm_eps
        self.config = config

    def forward(self, hidden_states):
        return fusion_rms_norm(hidden_states, self.weight, self.variance_epsilon,
                               getattr(self.config, "use_fast_layer_norm", False))


# ----------------------------------------------------------------------------------------------------------
# RoPE  (rotate-half convention; fusion_ops.py:107-115 passes use_neox_rotary_style=False)
# ----------------------------------------------------------------------------------------------------------
class LlamaRotaryEmbedding:
    """llama/modeling.py:402-439: cos/sin caches; here fp32 half tables [max_pos, d/2] on the device, computed on the
    host exactly as the reference does so that oracle and device share bits."""

    def __init__(self, dim, max_position_embeddings=2048, base=10000, device="cuda"):
        self.dim = dim
        self.max_position_embeddings = max_position_embeddings
        self.base = base
        self.cos_cached, self.sin_cached = ops.rope_tables(dim, max_position_embeddings, float(base), device)

    def __call__(self, x=None, seq_len=None):
        if seq_len is not None and seq_len > self.max_position_embeddings:
            raise ValueError(f"seq_len {seq_len} exceeds max_position_embeddings {self.max_position_embeddings}")
        return self.cos_cached, self.sin_cached


class _RopeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cos, sin, position_ids):
        b, s, heads, d = x.shape
        y = x.contiguous().clone()
        ops.rope_inplace(y.view(b * s, heads * d), cos, sin, s, heads, d, position_ids=position_ids)
        ctx.save_for_backward(cos, sin, position_ids if position_ids is not None else torch.empty(0))
        ctx.has_pos = position_ids is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        cos, sin, pos = ctx.saved_tensors
        b, s, heads, d = dy.shape
        dx = dy.contiguous().clone()
        ops.rope_inplace(dx.view(b * s, heads * d), cos, sin, s, heads, d, position_ids=pos if ctx.has_pos else None,
                         backward=True)
        return dx, None, None, None


def fusion_rope(query_states, key_states, value_states, hidden_states, position_ids, past_key_value, rotary_emb,
                context_parallel_degree=-1):
    """Rotate q and k ([b, s, heads, d]); returns (q, k).  Mirrors fusion_ops.py:57-116: no KV cache on the fused path,
    context parallelism is out of scope for the data-parallel path."""
    assert past_key_value is None, "fuse rotary not support cache kv for now"
    if context_parallel_degree > 1:
        raise NotImplementedError("context parallelism is outside the data-parallel hot path")
    _, seq_length, _, head_dim = query_states.shape
    cos, sin = rotary_emb(value_states, seq_len=seq_length)
    pos = None
    if position_ids is not None:
        pos = position_ids.to(torch.int32).contiguous().view(-1)
    q = _RopeFn.apply(query_states, cos, sin, pos)
    k = _RopeFn.apply(key_states, cos, sin, pos)
    return q, k


# ----------------------------------------------------------------------------------------------------------
# Flash attention  (F.scaled_dot_product_attention(q, k, v, attn_mask=None, is_causal=True), fusion_ops.py:240-246)
# ----------------------------------------------------------------------------------------------------------
class _FlashAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, mask_rows=None):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        o, lse = ops.flash_attn_fwd(q, k, v, scale, mask_start=mask_rows)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.scale = scale
        ctx.mask_rows = mask_rows
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        ops.flash_attn_bwd(q, k, v, o, do.contiguous(), lse, dq, dk, dv, ctx.scale, mask_start=ctx.mask_rows)
        return dq, dk, dv, None, None


def fusion_flash_attention(query_states, config, key_states, value_states, attention_mask, output_attentions, alibi=None,
                           attn_mask_startend_row_indices=None, sequence_parallel=False, reshard_layer=None,
                           npu_is_casual=False):
    """Causal GQA flash attention; q [b, s, nh, d], k/v [b, s, kvh, d] -> [b, s, nh*d] (or [b*s, nh*d] under
    `sequence_parallel`, fusion_ops.py:262-265).  The pre-training path passes attention_mask=None
    (llama/modeling.py:1679-1699 with a causal mask); packed SFT samples pass `attn_mask_startend_row_indices`
    (FlashMask); dense masks are outside the hot path and rejected."""
    bsz, q_len, num_heads, head_dim = query_states.shape
    if alibi is not None:
        raise NotImplementedError("alibi is not on the Llama-3 / Qwen2 path")
    if attention_mask is not None:
        raise NotImplementedError("dense attention masks are not built: causal, or causal + FlashMask start rows")
    if reshard_layer is not None:
        raise NotImplementedError("sep-parallel resharding is outside the data-parallel hot path")
    if output_attentions:
        raise ValueError("flash attention does not return attention weights (fusion_ops.py:209-212)")
    ops.check_head_dim(head_dim, "fusion_flash_attention")
    mask_rows = None
    if attn_mask_startend_row_indices is not None:
        # fusion_ops.py:218-231: F.flashmask_attention(..., startend_row_indices=idx.unsqueeze(-1), causal=True); idx is
        # [b, s] or [b, 1, s].  Canonical form for the kernels: every column visible at least to its own row.
        ops.check_mask_form(attn_mask_startend_row_indices.reshape(bsz, q_len))
        idx = attn_mask_startend_row_indices.reshape(bsz, q_len).to(device=query_states.device, dtype=torch.int32)
        own = torch.arange(1, q_len + 1, dtype=torch.int32, device=idx.device)
        mask_rows = torch.maximum(idx, own[None, :]).contiguous()
    out = _FlashAttnFn.apply(query_states, key_states, value_states, 1.0 / math.sqrt(head_dim), mask_rows)
    if sequence_parallel:
        return out.reshape(bsz * q_len, num_heads * head_dim)
    return out.reshape(bsz, q_len, num_heads * head_dim)


# ----------------------------------------------------------------------------------------------------------
# SwiGLU  (llama/modeling.py:38-45: silu(x) * y, or chunk(x, 2) when y is None)
# ----------------------------------------------------------------------------------------------------------
class _SwigluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        ctx.save_for_backward(gate_up)
        return ops.swiglu_fwd(gate_up)

    @staticmethod
    def backward(ctx, dout):
        (gate_up,) = ctx.saved_tensors
        return ops.swiglu_bwd(gate_up, dout.contiguous())


def swiglu(x, y: Optional[torch.Tensor] = None):
    if y is None:
        shp = x.shape
        out = _SwigluFn.apply(x.reshape(-1, shp[-1]).contiguous())
        return out.reshape(*shp[:-1], shp[-1] // 2)
    shp = x.shape
    gate_up = torch.cat([x.reshape(-1, shp[-1]), y.reshape(-1, shp[-1])], dim=-1)
    return _SwigluFn.apply(gate_up).reshape(shp)
