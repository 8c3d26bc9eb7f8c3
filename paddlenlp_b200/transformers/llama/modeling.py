"""Llama modeling classes — API surface of paddlenlp/transformers/llama/modeling.py on the native sm_90a engine.

    LlamaPretrainingCriterion   :1777-1825     LlamaModel        :1440-1774
    LlamaForCausalLM            :1924-2071     LlamaPretrainedModel :1235-1436

`LlamaForCausalLM.__call__(input_ids, position_ids=None, attention_mask=None, inputs_embeds=None, labels=None,
use_cache=False, past_key_values=None, output_attentions=None, output_hidden_states=None, return_dict=None)` returns
`(loss, logits)` / `logits` tuples or a CausalLMOutputWithCrossAttentions exactly like the reference (:2013-2071).
Labels are NOT shifted inside the model (the caller pre-shifts, llm/run_pretrain.py:245-255).
"""
from __future__ import annotations

from typing import Optional

import torch

from ... import ops
from ..model_outputs import BaseModelOutputWithPastAndCrossAttentions, CausalLMOutputWithCrossAttentions
from ..model_utils import PretrainedModel, _CausalLMLogitsFn, _CausalLMLossFn
from .configuration import LlamaConfig

__all__ = ["LlamaModel", "LlamaPretrainedModel", "LlamaForCausalLM", "LlamaPretrainingCriterion"]


class _CriterionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits2d, labels, ignore_index):
        loss_out, loss_tok, lse = ops.ce_fwd(logits2d, labels, ignore_index)
        ctx.save_for_backward(logits2d, labels, loss_tok, lse, loss_out)
        return loss_out[0].clone()

    @staticmethod
    def backward(ctx, gloss):
        logits2d, labels, loss_tok, lse, loss_out = ctx.saved_tensors
        d = logits2d.clone()
        ops.ce_bwd_(d, labels, loss_tok, lse, loss_out, 1.0, gloss.detach().float().reshape(1).contiguous())
        return d, None, None


class LlamaPretrainingCriterion(torch.nn.Module):
    """fp32 CE (reduction none, ignore_index) -> mean over positions with loss > 0 (modeling.py:1799-1825)."""

    def __init__(self, config=None, ignore_index: int = -100):
        super().__init__()
        self.config = config
        self.ignore_index = ignore_index

    def forward(self, prediction_scores: torch.Tensor, masked_lm_labels: torch.Tensor):
        V = prediction_scores.shape[-1]
        logits2d = prediction_scores.reshape(-1, V)
        labels = masked_lm_labels.to(device=logits2d.device, dtype=torch.int64).reshape(-1).contiguous()
        return _CriterionFn.apply(logits2d, labels, self.ignore_index)


def _check_unsupported(attention_mask, inputs_embeds, use_cache, past_key_values, output_attentions):
    if inputs_embeds is not None:
        raise NotImplementedError("inputs_embeds: the hot path starts from token ids")
    if past_key_values is not None or use_cache:
        raise NotImplementedError("KV-cache decoding is served by paddlenlp_b200.experimental (FusedMultiTransformer path)")
    if output_attentions:
        raise NotImplementedError("output_attentions: flash attention never materialises the attention matrix")
    if attention_mask is not None and attention_mask.dim() > 2:
        raise NotImplementedError("dense 3-D/4-D attention masks: pass attn_mask_startend_row_indices (FlashMask) for packed "
                                  "samples or a 2-D [batch, seq] padding mask")


def _mask_rows_from_padding_mask(attention_mask: torch.Tensor) -> torch.Tensor:
    """2-D `[batch, src_len]` padding mask (1 = attend, 0 = padding) -> FlashMask causal start rows.

    The reference expands it to `[b, 1, tgt, src]` and ANDs it with the causal mask (llama/modeling.py:1517-1552,
    qwen2/modeling.py:950-973): key column c is hidden from every query row when mask[b, c] == 0.  In start-row form that
    is start[c] = c + 1 (the column stays visible to its own — padding — row only, which keeps that row's softmax
    non-empty; its output carries label -100 / is discarded by the caller).  A trailing run of padding columns (right
    padding) is already invisible to every real row under the causal mask and is left at S.  This covers left- and
    right-padded batches (the Llama tokenizer pads on the left, llama/tokenizer.py:52); zeros in the middle of a row give
    non-monotonic start rows and are rejected by the engine's form check.  No host sync."""
    m = attention_mask != 0
    B, S = m.shape
    dev = m.device
    later_real = torch.flip(torch.cumsum(torch.flip(m.to(torch.int32), dims=[1]), dim=1), dims=[1]) > 0   # any real col >= c
    own = torch.arange(1, S + 1, dtype=torch.int32, device=dev)[None, :].expand(B, S)
    full = torch.full((B, S), S, dtype=torch.int32, device=dev)
    return torch.where(m | ~later_real, full, own).contiguous()


def _resolve_mask(attention_mask, attn_mask_startend_row_indices):
    """attn_mask_startend_row_indices wins when both are given (llama/modeling.py:1683-1688)."""
    if attn_mask_startend_row_indices is not None:
        return attn_mask_startend_row_indices
    if attention_mask is not None:
        if attention_mask.dim() != 2:
            raise NotImplementedError("attention_mask must be 2-D [batch, seq]")
        return _mask_rows_from_padding_mask(attention_mask)
    return None


class LlamaPretrainedModel(PretrainedModel):
    config_class = LlamaConfig
    base_model_prefix = "llama"


class LlamaModel(LlamaPretrainedModel):
    """Decoder stack without the head: returns final-norm hidden states [b, s, h]."""

    def __init__(self, config: LlamaConfig, device=None):
        super().__init__(config)
        self._build_engine(config, device)

    @torch.no_grad()
    def forward(self, input_ids=None, position_ids=None, attention_mask=None, inputs_embeds=None, use_cache=False,
                past_key_values=None, output_attentions=False, output_hidden_states=None, return_dict=False,
                attn_mask_startend_row_indices=None, **kw):
        _check_unsupported(attention_mask, inputs_embeds, use_cache, past_key_values, output_attentions)
        ms = _resolve_mask(attention_mask, attn_mask_startend_row_indices)
        B, S, _, _, _, hf, _ = self.engine.hidden_states(input_ids, position_ids, attn_mask_startend_row_indices=ms)
        hs = hf.view(B, S, -1)
        if return_dict:
            return BaseModelOutputWithPastAndCrossAttentions(last_hidden_state=hs)
        return (hs,)


class LlamaForCausalLM(LlamaPretrainedModel):
    def __init__(self, config: LlamaConfig, device=None):
        super().__init__(config)
        self._build_engine(config, device)
        self.criterion = LlamaPretrainingCriterion(config)

    def forward(self, input_ids=None, position_ids=None, attention_mask=None, inputs_embeds=None, labels=None,
                use_cache=False, past_key_values=None, output_attentions=None, output_hidden_states=None,
                return_dict=None, attn_mask_startend_row_indices=None, **kw):
        _check_unsupported(attention_mask, inputs_embeds, use_cache, past_key_values, output_attentions)
        # FlashMask start rows of packed samples ([B, S] or [B, 1, S(, 1)]), or derived from a 2-D padding mask
        ms = _resolve_mask(attention_mask, attn_mask_startend_row_indices)
        loss = None
        if labels is not None and torch.is_grad_enabled():
            loss, logits = _CausalLMLossFn.apply(self._anchor, self.engine, input_ids, labels, position_ids,
                                                 self.criterion.ignore_index, ms)
        elif labels is not None:
            loss_out, logits = self.engine.forward_loss(input_ids, labels, position_ids, self.criterion.ignore_index,
                                                        keep_for_backward=False, attn_mask_startend_row_indices=ms)
            loss = loss_out[0]
        elif torch.is_grad_enabled() and self.training:
            # no labels, gradient mode, train(): logits stay differentiable (the caller applies its own criterion and calls
            # loss.backward(), trainer.py:2157-2197); use torch.no_grad() / .eval() for inference
            logits = _CausalLMLogitsFn.apply(self._anchor, self.engine, input_ids, position_ids, ms)
        else:
            logits = self.engine.forward_logits(input_ids, position_ids, attn_mask_startend_row_indices=ms)
        if return_dict:
            return CausalLMOutputWithCrossAttentions(loss=loss, logits=logits)
        return (loss, logits) if loss is not None else (logits,)

    @torch.no_grad()
    def greedy_next_tokens(self, input_ids, position_ids=None):
        """argmax over the last position's logits (paddlenlp/generation/utils.py greedy branch)."""
        logits = self.engine.forward_logits(input_ids, position_ids)
        return ops.argmax(logits[:, -1, :].contiguous())
