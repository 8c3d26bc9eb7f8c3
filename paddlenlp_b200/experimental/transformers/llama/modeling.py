"""LlamaInferenceModel / LlamaForCausalLMInferenceModel — paddlenlp/experimental/transformers/llama/modeling.py
(:388 LlamaInferenceModel, :731 forward, :901-1060 set_state_dict weight fusion, :1751-1913 ForCausalLM wrapper).
Qwen2 (q/k/v bias) uses the same stack."""
from __future__ import annotations

from typing import Dict, List

import torch

from .... import ops
from ..fused_transformer_layers import FusedBlockMultiTransformer, FusedMultiTransformerBase, FusedMultiTransformerConfig
from ..generation_utils import GenerationInferenceModel

BF16 = torch.bfloat16


class LlamaForCausalLMInferenceModel(GenerationInferenceModel):
    def __init__(self, config, device=None, block_attn: bool = False, block_size: int = 64, append_attn: bool = False):
        """block_attn=True selects the paged KV cache (`--block_attn` of llm/predict/predictor.py:1507-1520:
        LlamaBlockInferenceModel on FusedBlockMultiTransformer); append_attn=True (`--append_attn`) additionally routes prefill
        and decode attention through the unified append_attention op."""
        if append_attn and not block_attn:
            raise ValueError("append_attn needs block_attn=True (the op works on the paged cache)")
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
            qkv_bias=(c.model_type == "qwen2"), append_attn=bool(append_attn))
        self.transformer_block = (FusedBlockMultiTransformer if self.block_attn else FusedMultiTransformerBase)(fcfg, device)
        self.device = self.transformer_block.device
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
        A tied model reads no `lm_head.weight` (one in `sd` is ignored)."""
        t = self.transformer_block
        pre = self.prefix
        dev = self.device

        def g(name):
            return sd[name].to(device=dev, dtype=BF16)

        self.embed_tokens.copy_(g(f"{pre}.embed_tokens.weight"))
        self.norm_weight.copy_(g(f"{pre}.norm.weight"))
        if not self.tied:
            self.lm_head_weight.copy_(g("lm_head.weight"))
        for i in range(t.L):
            lp = f"{pre}.layers.{i}."
            qkv = torch.cat([g(lp + "self_attn.q_proj.weight"), g(lp + "self_attn.k_proj.weight"),
                             g(lp + "self_attn.v_proj.weight")], dim=-1)
            t.qkv_weights[i].copy_(qkv.t())
            if t.qkv_biases[i] is not None:
                t.qkv_biases[i].copy_(torch.cat([g(lp + "self_attn.q_proj.bias"), g(lp + "self_attn.k_proj.bias"),
                                                 g(lp + "self_attn.v_proj.bias")]))
                t._bias_f32[i] = None
            t.linear_weights[i].copy_(g(lp + "self_attn.o_proj.weight"))
            t.ffn1_weights[i].copy_(torch.cat([g(lp + "mlp.gate_proj.weight"), g(lp + "mlp.up_proj.weight")], dim=-1))
            t.ffn2_weights[i].copy_(g(lp + "mlp.down_proj.weight"))
            t.ln_scales[i].copy_(g(lp + "input_layernorm.weight"))
            t.ffn_ln_scales[i].copy_(g(lp + "post_attention_layernorm.weight"))
        t.weights_changed()

    @torch.no_grad()
    def init_random(self, seed: int = 42, std: float = 0.02):
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        t = self.transformer_block
        head = [] if self.tied else [self.lm_head_weight]
        for w in [self.embed_tokens] + head + t.qkv_weights + t.linear_weights + t.ffn1_weights + t.ffn2_weights:
            w.normal_(0.0, std, generator=gen)
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
        return [torch.zeros(n, t.kvh, bs, t.d, dtype=BF16, device=self.device) for _ in range(2 * t.L)]

    def _cache_kw(self):
        return {"block_tables": self.block_tables} if self.block_attn else {}

    # ---- forward ----
    def _head(self, hidden):
        hn, _ = ops.add_rmsnorm(hidden, None, self.norm_weight, self.config.rms_norm_eps, want_residual=False)
        if self.tied:
            return self.transformer_block._mm(hn, self.embed_tokens, trans_b=True)
        return self.transformer_block._mm(hn, self.lm_head_weight)

    def _prefill(self, input_ids, seq_lens_encoder, caches):
        B, S = input_ids.shape
        emb = ops.embedding_fwd(input_ids.reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=S, seq_lens_encoder=seq_lens_encoder, **self._cache_kw())
        # rebuild_padding: keep the last valid position of every sequence
        last = (torch.arange(B, device=self.device) * S + seq_lens_encoder.to(torch.int64) - 1)
        return self._head(hidden.index_select(0, last).contiguous())

    def _decode(self, tgt_ids, seq_lens_decoder, caches):
        B = tgt_ids.numel()
        emb = ops.embedding_fwd(tgt_ids.reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=1, seq_lens_decoder=seq_lens_decoder, time_step=0,
                                        **self._cache_kw())
        return self._head(hidden)

    @torch.no_grad()
    def forward_logits_prefill(self, input_ids):
        """All-position logits of the prefill pass (parity checks against the training-path forward)."""
        B, S = input_ids.shape
        caches = self.allocate_caches(B, S)
        emb = ops.embedding_fwd(input_ids.to(self.device).reshape(-1), self.embed_tokens)
        hidden = self.transformer_block(emb, caches, B=B, S=S, seq_lens_encoder=None, **self._cache_kw())
        return self._head(hidden).view(B, S, -1)
