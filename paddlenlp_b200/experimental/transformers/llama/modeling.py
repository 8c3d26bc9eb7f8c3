"""LlamaInferenceModel / LlamaForCausalLMInferenceModel — paddlenlp/experimental/transformers/llama/modeling.py
(:388 LlamaInferenceModel, :731 forward, :901-1060 set_state_dict weight fusion, :1751-1913 ForCausalLM wrapper).
Qwen2 (q/k/v bias) uses the same stack."""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional, Union

import torch

from .... import ops
from ..fused_transformer_layers import (FusedBlockMultiTransformer, FusedBlockMultiTransformerWeightOnly, FusedMultiTransformerBase,
                                        FusedMultiTransformerConfig, FusedMultiTransformerWeightOnly)
from ..generation_utils import GenerationInferenceModel

BF16 = torch.bfloat16


class LlamaForCausalLMInferenceModel(GenerationInferenceModel):
    def __init__(self, config, device=None, block_attn: bool = False, block_size: int = 64, append_attn: bool = False,
                 quant_type=None, cachekv_int8_type=None):
        """block_attn=True selects the paged KV cache (`--block_attn` of llm/predict/predictor.py:1507-1520:
        LlamaBlockInferenceModel on FusedBlockMultiTransformer); append_attn=True (`--append_attn`) additionally routes prefill
        and decode attention through the unified append_attention op.  quant_type (`--quant_type`, predictor.py:86,1250; None
        reads config.quant_type, where the predictor puts it): "weight_only_int8" holds the layer matrices as int8 with
        per-channel scales (FusedMultiTransformerWeightOnly); embeddings, norms and the head stay bf16.
        cachekv_int8_type (`--cachekv_int8_type`, predictor.py:117-122; None reads config.cachekv_int8_type): "static" holds
        the paged KV cache as uint8 with one static scale per layer and kv head, loaded with set_cache_scales() or measured
        with calibrate_cache_scales(); it needs block_attn=True and composes with either quant_type."""
        if append_attn and not block_attn:
            raise ValueError("append_attn needs block_attn=True (the op works on the paged cache)")
        ct = getattr(config, "cachekv_int8_type", None) if cachekv_int8_type is None else cachekv_int8_type
        if ct is not None and not block_attn:
            if ct == "dynamic":
                raise NotImplementedError('cachekv_int8_type "dynamic" is not implemented; "static" is')
            raise NotImplementedError(f"cachekv_int8_type {ct!r} is implemented for the paged cache only: build the model with "
                                      f"block_attn=True")
        self.config = config
        self.block_attn = bool(block_attn)
        self.block_size = int(block_size)
        self.block_tables = None
        c = config
        self.prefix = c.model_type
        fcfg = FusedMultiTransformerConfig(
            embed_dim=c.hidden_size, num_heads=c.num_attention_heads, dim_feedforward=c.intermediate_size,
            kv_num_heads=c.num_key_value_heads, num_layers=c.num_hidden_layers, epsilon=c.rms_norm_eps,
            rope_theta=c.rope_theta, max_position_embeddings=max(int(getattr(c, "max_position_embeddings", 4096)), 128),
            qkv_bias=(c.model_type == "qwen2"), append_attn=bool(append_attn),
            quant_type=(getattr(c, "quant_type", "") if quant_type is None else quant_type) or "", cachekv_int8_type=ct)
        if fcfg.quant_type:
            block = FusedBlockMultiTransformerWeightOnly if self.block_attn else FusedMultiTransformerWeightOnly
        else:
            block = FusedBlockMultiTransformer if self.block_attn else FusedMultiTransformerBase
        self.transformer_block = block(fcfg, device)
        self.device = self.transformer_block.device
        self.cache_dtype = ops.CACHE_INT8 if ct is not None else BF16
        self.embed_tokens = torch.zeros(c.vocab_size, c.hidden_size, dtype=BF16, device=self.device)
        self.norm_weight = torch.ones(c.hidden_size, dtype=BF16, device=self.device)
        # tied embeddings (llama/modeling.py:1924-1938): the head reads embed_tokens [V, h] as the GEMM's K-major operand
        self.tied = bool(getattr(c, "tie_word_embeddings", False))
        self.lm_head_weight = (None if self.tied else
                               torch.zeros(c.hidden_size, c.vocab_size, dtype=BF16, device=self.device))

    # ---- weights (experimental/transformers/llama/modeling.py:901-1060) ----
    @torch.no_grad()
    def set_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Accepts the training-format names (`llama.layers.N.self_attn.q_proj.weight` [in,out], ...) and fuses them into
        the FusedMultiTransformer layouts: qkv_weight = concat([Wq,Wk,Wv],-1).T, ffn1_weight = concat([Wg,Wu],-1).
        A tied model reads no `lm_head.weight` (one in `sd` is ignored).  A weight-only block quantises each fused matrix on
        the device as it is built: one bf16 fused matrix is staged at a time."""
        t = self.transformer_block
        pre = self.prefix
        dev = self.device

        def g(name):
            return sd[name].to(device=dev, dtype=BF16)

        def cat_cols(names):
            """concat(..., -1) built in one device buffer: no device copy of the parts is staged beside it."""
            parts = [sd[n] for n in names]
            out = torch.empty(parts[0].shape[0], sum(p.shape[1] for p in parts), dtype=BF16, device=dev)
            c0 = 0
            for p in parts:
                out[:, c0:c0 + p.shape[1]].copy_(p)
                c0 += p.shape[1]
            return out

        self.embed_tokens.copy_(g(f"{pre}.embed_tokens.weight"))
        self.norm_weight.copy_(g(f"{pre}.norm.weight"))
        if not self.tied:
            self.lm_head_weight.copy_(g("lm_head.weight"))
        for i in range(t.L):
            lp = f"{pre}.layers.{i}."
            qkv = cat_cols([lp + "self_attn.q_proj.weight", lp + "self_attn.k_proj.weight", lp + "self_attn.v_proj.weight"])
            t.set_layer_matrix("qkv", i, qkv.t())
            del qkv
            if t.qkv_biases[i] is not None:
                t.qkv_biases[i].copy_(torch.cat([g(lp + "self_attn.q_proj.bias"), g(lp + "self_attn.k_proj.bias"),
                                                 g(lp + "self_attn.v_proj.bias")]))
                t._bias_f32[i] = None
            t.set_layer_matrix("linear", i, g(lp + "self_attn.o_proj.weight"))
            t.set_layer_matrix("ffn1", i, cat_cols([lp + "mlp.gate_proj.weight", lp + "mlp.up_proj.weight"]))
            t.set_layer_matrix("ffn2", i, g(lp + "mlp.down_proj.weight"))
            t.ln_scales[i].copy_(g(lp + "input_layernorm.weight"))
            t.ffn_ln_scales[i].copy_(g(lp + "post_attention_layernorm.weight"))
        t.weights_changed()

    @torch.no_grad()
    def init_random(self, seed: int = 42, std: float = 0.02):
        """Normal(0, std) weights.  A weight-only block draws each layer matrix in the bf16 block's shape from the same generator
        sequence and quantises it: bf16 and int8 models of one seed hold the same underlying weights."""
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        t = self.transformer_block
        head = [] if self.tied else [self.lm_head_weight]
        for w in [self.embed_tokens] + head:
            w.normal_(0.0, std, generator=gen)
        for name in t.MATRICES:
            for i in range(t.L):
                if t.config.quant_type:
                    w = torch.empty(t.layer_matrix_shape(name), dtype=BF16, device=self.device).normal_(0.0, std, generator=gen)
                    t.set_layer_matrix(name, i, w)
                    del w
                else:
                    getattr(t, name + "_weights")[i].normal_(0.0, std, generator=gen)
        t.weights_changed()

    def allocate_caches(self, batch: int, max_len: int) -> List[torch.Tensor]:
        """cache_kvs = [zeros([2, bsz, kvh, max_len, d])] * L (llm/predict/predictor.py:697-706)."""
        t = self.transformer_block
        if self.block_attn:
            return self.allocate_block_caches(batch, max_len)
        return [torch.zeros(2, batch, t.kvh, max_len, t.d, dtype=BF16, device=self.device) for _ in range(t.L)]

    def allocate_block_caches(self, batch: int, max_len: int, max_block_nums: int = 0) -> List[torch.Tensor]:
        """cache_kvs = [key_cache_0, value_cache_0, ...], each zeros([max_block_nums, kvh, block_size, d])
        (get_cache_kvs_shape, experimental/transformers/llama/modeling.py; predictor.py:960-964), plus the block tables the
        predictor builds (predictor.py:923-930): -1 everywhere, then every sequence takes ceil(max_len / block_size) blocks
        popped from the end of the free list."""
        t = self.transformer_block
        bs = self.block_size
        per_seq = (max_len + bs - 1) // bs
        n = max(max_block_nums, batch * per_seq)
        free_list = list(range(n))
        tables = torch.full((batch, per_seq), -1, dtype=torch.int32)
        for i in range(batch):
            for j in range(per_seq):
                tables[i, j] = free_list.pop()
        self.block_tables = tables.to(self.device)
        # zero pages: a uint8 cache byte of 128 reads back as 0 too, but every position a kernel reads has been written first
        return [torch.zeros(n, t.kvh, bs, t.d, dtype=self.cache_dtype, device=self.device) for _ in range(2 * t.L)]

    # ---- static int8 KV-cache scales (cachekv_int8_type="static") ----
    def set_cache_scales(self, scales: Union[Dict[str, list], str]):
        """Load the reference's cachekv_scales.json (a path or its parsed content): keys
        `<model_type>.layers.<i>.self_attn.cachek_matmul.activation_quanter` and `...cachev_matmul...`, each holding
        num_attention_heads absmax values.  Under GQA every group-th value is kept (one per kv head), then s = 127 / absmax and
        o = 1 / s, both cast to bf16, as CacheScaleLoader does (experimental/model_utils.py:433-468).  A missing key or a
        missing, non-finite or non-positive absmax raises ValueError (the reference fills in -1)."""
        if isinstance(scales, (str, os.PathLike)):
            with open(scales) as f:
                scales = json.load(f)
        t = self.transformer_block
        nh = self.config.num_attention_heads
        group = nh // t.kvh
        out = {}
        for kind in ("k", "v"):
            rows = []
            for i in range(t.L):
                key = f"{self.prefix}.layers.{i}.self_attn.cache{kind}_matmul.activation_quanter"
                if key not in scales:
                    raise ValueError(f"set_cache_scales: no {key!r}")
                vals = list(scales[key])
                if len(vals) != nh:
                    raise ValueError(f"set_cache_scales: {key!r} holds {len(vals)} values, expected num_attention_heads {nh}")
                rows.append([float(vals[j]) for j in range(0, nh, group)])
            out[kind] = torch.tensor(rows, dtype=torch.float64)
        t.set_cache_scales(out["k"], out["v"])

    @torch.no_grad()
    def calibrate_cache_scales(self, input_ids: torch.Tensor, seq_len_encoder: Optional[torch.Tensor] = None):
        """Measure static cache scales on sample prompts: one prefill of input_ids [B, S] (right padded to seq_len_encoder)
        into a bf16 paged cache, then the absmax of the cached K and V per (layer, kv head).  Positions no prompt reaches stay
        zero and do not move an absmax.  Returns the (k, v) absmax tensors [L, kvh] after setting the scales from them."""
        t = self.transformer_block
        if t.config.cachekv_int8_type is None:
            raise ValueError("calibrate_cache_scales: the model was built without cachekv_int8_type")
        B, S = input_ids.shape
        ids = input_ids.to(self.device, torch.int64).contiguous()
        enc = (torch.full((B,), S, dtype=torch.int32, device=self.device) if seq_len_encoder is None
               else seq_len_encoder.to(self.device, torch.int32).reshape(B).contiguous())
        t.ensure_rope(S)
        saved_tables, saved_dtype = self.block_tables, self.cache_dtype
        try:
            self.cache_dtype = BF16
            caches = self.allocate_block_caches(B, S)
            self._prefill(ids, enc, caches)
        finally:
            self.block_tables, self.cache_dtype = saved_tables, saved_dtype
        absmax = [torch.stack([caches[2 * i + w].abs().amax(dim=(0, 2, 3)).double() for i in range(t.L)]).cpu() for w in (0, 1)]
        del caches
        t.set_cache_scales(absmax[0], absmax[1])
        return absmax[0], absmax[1]

    def _cache_kw(self):
        return {"block_tables": self.block_tables} if self.block_attn else {}

    # ---- forward ----
    def _head(self, hidden, decode=True):
        """Logits of the given rows.  decode=False (prefill, once per prompt): the training path's GEMM, whose per-row sums run
        in the same order as the training forward's, so prefill logits carry its bits; the decode step's split-K kernel
        (few rows, weight streaming) adds K-range partials in L2 and can round a logit one bf16 ulp differently."""
        hn, _ = ops.add_rmsnorm(hidden, None, self.norm_weight, self.config.rms_norm_eps, want_residual=False)
        w, trans_b = (self.embed_tokens, True) if self.tied else (self.lm_head_weight, False)
        if not decode:
            return ops.gemm(hn, w, trans_b=trans_b)
        return self.transformer_block._mm(hn, w, trans_b=trans_b)

    def _prefill(self, input_ids, seq_lens_encoder, caches):
        B, S = input_ids.shape
        emb = ops.embedding_fwd(input_ids.reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=S, seq_lens_encoder=seq_lens_encoder, **self._cache_kw())
        # rebuild_padding: keep the last valid position of every sequence
        last = (torch.arange(B, device=self.device) * S + seq_lens_encoder.to(torch.int64) - 1)
        return self._head(hidden.index_select(0, last).contiguous(), decode=False)

    def _decode(self, tgt_ids, seq_lens_decoder, caches):
        B = tgt_ids.numel()
        emb = ops.embedding_fwd(tgt_ids.reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=1, seq_lens_decoder=seq_lens_decoder, time_step=0,
                                        **self._cache_kw())
        return self._head(hidden)

    def _forward_packed(self, ids, caches, block_tables, enc, dec, this_time, cu_seqlens_q, cum_offsets, max_q_len, max_len):
        """One continuous-batching step over the packed rows `ids` [token_num] of every slot (append_attention), then each
        slot's last row (rebuild_padding; an idle slot gives a zero row) through the head: logits [slots, V]."""
        emb = ops.embedding_fwd(ids, self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=this_time.numel(), S=0, block_tables=block_tables,
                                        packed=(enc, dec, this_time, cu_seqlens_q, max_q_len))
        last = ops.rebuild_padding(hidden, cum_offsets, dec, enc, max_len)
        return self._head(last, decode=max_q_len == 1)

    @torch.no_grad()
    def forward_logits_prefill(self, input_ids):
        """All-position logits of the prefill pass (parity checks against the training-path forward)."""
        B, S = input_ids.shape
        caches = self.allocate_caches(B, S)
        emb = ops.embedding_fwd(input_ids.to(self.device).reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=S, seq_lens_encoder=None, **self._cache_kw())
        return self._head(hidden, decode=False).view(B, S, -1)
