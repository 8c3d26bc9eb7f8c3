"""FusedMultiTransformer — the stacked-layer inference block of
paddlenlp/experimental/transformers/fused_transformer_layers.py (:205-345 config, :348-792 weights, :1027-1182 forward)
for the rmsnorm + swiglu + rotate-half-RoPE case, on the native sm_90a kernels: bf16 layer weights, or weight-only int8
(quant_type="weight_only_int8": FusedMultiTransformerWeightOnly / FusedBlockMultiTransformerWeightOnly, :1221-1440).

Weight layouts are the reference's (SURVEY.md Appendix B):
    qkv_weight    [(nh + 2*kvh) * d, h]   (transposed, trans_qkvw=True)      -> GEMM with B stored [N, K]
    linear_weight [nh * d, h]             ffn1_weight [h, 2*I] (gate | up)    ffn2_weight [I, h]
    ln_scale / ffn_ln_scale [h]
KV cache per layer: bf16 [2, B, kvh, max_len, d]; paged (FusedBlockMultiTransformer): bf16 pages, or uint8 pages with static
per-kv-head scales (cachekv_int8_type="static", fused_transformer_layers.py:2389-2395).
Layer loop (:1126-1174): the output norm of layer i is fused with the residual add and is layer i+1's input norm.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional

import torch

from ... import ops

BF16 = torch.bfloat16


@dataclass
class FusedMultiTransformerConfig:
    embed_dim: int
    num_heads: int
    dim_feedforward: int
    kv_num_heads: int = -1
    num_layers: int = -1
    epsilon: float = 1e-5
    norm_type: str = "rmsnorm"
    activation: str = "swiglu"
    use_neox_rotary_style: bool = True       # csrc naming: neox == rotate-half (encode_rotary_qk.cu:18-56)
    rope_theta: float = 10000.0
    max_position_embeddings: int = 4096
    qkv_bias: bool = False
    nranks: int = 1
    trans_qkvw: bool = True
    append_attn: bool = False                # FusedBlockMultiTransformer: route attention through the unified append_attention op
    quant_type: str = ""                     # "" (bf16 layer weights) or "weight_only_int8" (FusedMultiTransformerWeightOnly)
    cachekv_int8_type: Optional[str] = None  # None (bf16 cache) or "static": uint8 paged cache, per-kv-head scales

    def __post_init__(self):
        if self.kv_num_heads <= 0:
            self.kv_num_heads = self.num_heads
        if self.norm_type != "rmsnorm" or self.activation != "swiglu":
            raise NotImplementedError("only the rmsnorm + swiglu (Llama / Qwen2) block is implemented")
        if not self.use_neox_rotary_style:
            raise NotImplementedError("interleaved-pair RoPE is not used by Llama/Qwen2 (SURVEY.md §8 naming trap)")
        if self.nranks != 1:
            raise NotImplementedError("tensor-parallel generation is out of scope (config 5 is single-GPU)")
        if not self.trans_qkvw:
            raise NotImplementedError("trans_qkvw=False")
        ops.check_head_dim(self.embed_dim // self.num_heads, "FusedMultiTransformerConfig")
        qt = self.quant_type
        if qt not in ("", "weight_only_int8"):
            if qt == "weight_only_int4" or qt.startswith("a8w8") or "fp8" in qt:
                raise NotImplementedError(f"quant_type {qt!r} is not implemented (weight_only_int8 is)")
            raise ValueError(f"unknown quant_type {qt!r}")
        ct = self.cachekv_int8_type
        if ct == "dynamic":
            raise NotImplementedError('cachekv_int8_type "dynamic" (per-step scales) is not implemented; "static" is')
        if ct not in (None, "static"):
            raise ValueError(f"unknown cachekv_int8_type {ct!r} (None or 'static')")


class FusedMultiTransformerBase:
    def __init__(self, config: FusedMultiTransformerConfig, device=None):
        if config.cachekv_int8_type is not None and not isinstance(self, FusedBlockMultiTransformer):
            raise NotImplementedError(f"cachekv_int8_type {config.cachekv_int8_type!r} needs the paged cache (block_attn=True); "
                                      f"the dense cache is bf16 only")
        # every cache path ends in the decode-attention kernels: refuse a head layout they do not cover now, not at the
        # first decode step after a prefill
        nh, kvh = config.num_heads, config.kv_num_heads
        if nh % kvh:
            raise ValueError(f"num_heads {nh} is not a multiple of kv_num_heads {kvh}")
        if nh // kvh not in ops.DECODE_GQA_GROUPS:
            raise ValueError(f"GQA group size {nh // kvh} (num_heads {nh} / kv_num_heads {kvh}) is not supported by the decode "
                             f"attention kernels ({ops.DECODE_GQA_GROUPS.start} to {ops.DECODE_GQA_GROUPS.stop - 1})")
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("FusedMultiTransformer needs a CUDA device: there is no CPU implementation")
            device = torch.device("cuda", torch.cuda.current_device())
        self.config = config
        self.device = torch.device(device)
        c = config
        self.h, self.nh, self.kvh, self.I, self.L = c.embed_dim, c.num_heads, c.kv_num_heads, c.dim_feedforward, c.num_layers
        self.d = self.h // self.nh
        self.qkv_n = (self.nh + 2 * self.kvh) * self.d

        self.ln_scales = [torch.ones(self.h, dtype=BF16, device=self.device) for _ in range(self.L)]
        self.qkv_biases: List[Optional[torch.Tensor]] = [torch.zeros(self.qkv_n, dtype=BF16, device=self.device) if c.qkv_bias
                                                         else None for _ in range(self.L)]
        self.ffn_ln_scales = [torch.ones(self.h, dtype=BF16, device=self.device) for _ in range(self.L)]
        self._alloc_layer_matrices()
        self._bias_f32 = [None] * self.L
        self.rope = ops.rope_tables(self.d, c.max_position_embeddings, float(c.rope_theta), self.device)

    MATRICES = ("qkv", "linear", "ffn1", "ffn2")

    def layer_matrix_shape(self, name):
        """Shape of layer matrix `name` in the bf16 block (the reference's layouts above: qkv is stored transposed)."""
        return {"qkv": (self.qkv_n, self.h), "linear": (self.nh * self.d, self.h), "ffn1": (self.h, 2 * self.I),
                "ffn2": (self.I, self.h)}[name]

    def _alloc_layer_matrices(self):
        for name in self.MATRICES:
            setattr(self, name + "_weights", [torch.zeros(*self.layer_matrix_shape(name), dtype=BF16, device=self.device)
                                              for _ in range(self.L)])

    def set_layer_matrix(self, name, i, w):
        """Load layer i's matrix `name` from a bf16 tensor of layer_matrix_shape(name)."""
        getattr(self, name + "_weights")[i].copy_(w)

    def ensure_rope(self, positions: int):
        """Grow the fp32 cos/sin tables to cover `positions` rows.  The decode kernels index them with the running sequence
        length (decode_rope_append reads row seq_len of the tables): a cache longer than config.max_position_embeddings
        must not read past the tables.  Call outside CUDA-graph capture (generate() does, before the first step)."""
        if self.rope[0].shape[0] < positions:
            self.rope = ops.rope_tables(self.d, int(positions), float(self.config.rope_theta), self.device)

    def _bias(self, i):
        if self.qkv_biases[i] is None:
            return None
        if self._bias_f32[i] is None:
            self._bias_f32[i] = self.qkv_biases[i].float()
        return self._bias_f32[i]

    def weights_changed(self):
        """Call after editing the weight tensors in place (set_state_dict does): derived copies are rebuilt lazily."""
        self._bias_f32 = [None] * self.L

    SKINNY_M = 128     # at or below this many token rows the GEMMs are weight-streaming bound: split-K kernel

    def _mm(self, a, w, trans_b=False, bias=None):
        n = w.shape[0] if trans_b else w.shape[1]
        if a.shape[0] <= self.SKINNY_M:
            if n >= 100 * 256:        # enough 256-wide column tiles to keep most SMs streaming: no split-K needed
                return ops.gemm(a, w, trans_b=trans_b, bias=bias)
            return ops.gemm_skinny(a, w, trans_b=trans_b, bias=bias)
        return ops.gemm(a, w, trans_b=trans_b, bias=bias)

    # ---- per-matrix hooks (overridden by the weight-only blocks); `name` is one of MATRICES ----
    def linear(self, x, name, i, bias=None):
        """bf16 output of layer i's matrix `name` applied to x (+ fp32 bias)."""
        return self._mm(x, getattr(self, name + "_weights")[i], trans_b=name == "qkv", bias=bias)

    def linear_f32(self, x, name, i, tag):
        """The decode step's form: fp32 sums left in the workspace `tag` for the consumer kernel to round and re-zero."""
        return ops.gemm_skinny_f32(x, getattr(self, name + "_weights")[i], trans_b=name == "qkv", tag=tag)

    def ffn1_act(self, x, i):
        """The decode step's ffn1 + SwiGLU."""
        if self.I % 64 == 0:
            # SwiGLU in the ffn1 epilogue of the persistent kernel: the 256-column tile pairs 128 gate columns with the
            # 128 up columns of the same channels straight from the reference-layout weight; only the activation is stored
            _, act = ops.gemm_swiglu(x, self.ffn1_weights[i], store_gate_up=False)
            return act
        return ops.swiglu_fwd(self.linear(x, "ffn1", i))

    # compute_qkv (:817-820): linear(ln_out, qkv_weight, transpose_weight=True)
    def compute_qkv(self, ln_out, i):
        return self.linear(ln_out, "qkv", i, bias=self._bias(i))

    # ---- the three places that touch the KV cache (overridden by FusedBlockMultiTransformer) ----
    def _write_cache(self, qkv, caches, i, B, S, seq_lens_encoder, kw):
        ops.write_cache_kv(qkv, caches[i], seq_lens_encoder, B, S, self.nh, self.kvh, self.d)

    def _rope_append(self, qkv, acc, caches, i, seq_lens_decoder, kw):
        cos, sin = self.rope
        if acc is not None:
            return ops.decode_rope_append_f32(acc, self._bias(i), caches[i], cos, sin, seq_lens_decoder, self.nh, self.kvh, self.d)
        ops.decode_rope_append(qkv, caches[i], cos, sin, seq_lens_decoder, self.nh, self.kvh, self.d)
        return qkv

    def _attend(self, qkv, caches, i, seq_lens_decoder, kw):
        return ops.decode_attention(qkv, caches[i], seq_lens_decoder, self.nh, self.kvh, self.d)

    # compute_fmha (:829-882): qkv_transpose_split -> encode_rotary_qk -> write_cache_kv -> var-len attention
    def compute_fmha(self, qkv, caches, i, B, S, seq_lens_encoder, kw):
        cos, sin = self.rope
        ops.rope_inplace(qkv, cos, sin, S, self.nh + self.kvh, self.d)
        self._write_cache(qkv, caches, i, B, S, seq_lens_encoder, kw)
        q4 = qkv.view(B, S, self.qkv_n)
        qn, kn = self.nh * self.d, self.kvh * self.d
        q = q4[:, :, :qn].unflatten(2, (self.nh, self.d))
        k = q4[:, :, qn:qn + kn].unflatten(2, (self.kvh, self.d))
        v = q4[:, :, qn + kn:].unflatten(2, (self.kvh, self.d))
        attn, _ = ops.flash_attn_fwd(q, k, v)           # right-padded prompts are exact under the causal mask
        return attn.view(B * S, qn)

    # compute_mmha (:884-893): masked_multihead_attention over the cache
    def compute_mmha(self, qkv, caches, i, seq_lens_decoder, kw):
        qkv = self._rope_append(qkv, None, caches, i, seq_lens_decoder, kw)
        return self._attend(qkv, caches, i, seq_lens_decoder, kw)

    def forward(self, src: torch.Tensor, caches: List[torch.Tensor], *, B: int, S: int, seq_lens_encoder=None,
                seq_lens_decoder=None, time_step=None, **kw) -> torch.Tensor:
        """src [B*S, h] embeddings.  time_step None = prefill (S prompt positions per sequence, right padded);
        otherwise decode (S == 1, seq_lens_decoder[b] = number of cached tokens).  Returns hidden states [B*S, h]."""
        eps = self.config.epsilon
        decode = time_step is not None
        residual = src
        ln_out, _ = ops.add_rmsnorm(src, None, self.ln_scales[0], eps, want_residual=False)   # compute_layernorm_before_qkv
        fused = decode and src.shape[0] <= self.SKINNY_M and not getattr(self.config, "append_attn", False)
        for i in range(self.L):
            if fused:
                # decode step: the split-K GEMMs leave fp32 sums that the next kernel rounds once (same rounding points,
                # three launches fewer per layer)
                acc = self.linear_f32(ln_out, "qkv", i, "splitk_qkv")
                qkv = self._rope_append(None, acc, caches, i, seq_lens_decoder, kw)
                attn = self._attend(qkv, caches, i, seq_lens_decoder, kw)
                acc = self.linear_f32(attn, "linear", i, "splitk_h")
                ln_out, residual = ops.add_rmsnorm_f32(acc, residual, self.ffn_ln_scales[i], eps)
                act = self.ffn1_act(ln_out, i)
                acc = self.linear_f32(act, "ffn2", i, "splitk_h")
                if i != self.L - 1:
                    ln_out, residual = ops.add_rmsnorm_f32(acc, residual, self.ln_scales[i + 1], eps)
                else:
                    _, residual = ops.add_rmsnorm_f32(acc, residual, None, eps, want_normed=False)
                continue
            qkv = self.compute_qkv(ln_out, i)
            if decode:
                attn = self.compute_mmha(qkv, caches, i, seq_lens_decoder, kw)
            else:
                attn = self.compute_fmha(qkv, caches, i, B, S, seq_lens_encoder, kw)
            out = self.linear(attn, "linear", i)                                              # compute_out_linear (:895-896)
            ln_out, residual = ops.add_rmsnorm(out, residual, self.ffn_ln_scales[i], eps)     # compute_ffn_layernorm (:937-949)
            ffn1 = self.linear(ln_out, "ffn1", i)
            act = ops.swiglu_fwd(ffn1)                                                        # fused_bias_act("swiglu") (:100-168)
            ffn2 = self.linear(act, "ffn2", i)
            if i != self.L - 1:                                                               # compute_bias_residual_layernorm (:976-999)
                ln_out, residual = ops.add_rmsnorm(ffn2, residual, self.ln_scales[i + 1], eps)
            else:
                _, residual = ops.add_rmsnorm(ffn2, residual, None, eps, want_normed=False)
        return residual

    __call__ = forward


class FusedBlockMultiTransformer(FusedMultiTransformerBase):
    """Paged ("block") KV cache variant (fused_transformer_layers.py:2192-2354, `compute_attn` -> append_attention /
    block_multihead_attention).  `caches` is the reference's list of 2*L tensors [key_cache_0, value_cache_0, key_cache_1, ...],
    each [max_block_nums, kv_num_heads, block_size, head_dim]; `block_tables` [B, max_blocks_per_seq] int32 (-1 = unused)
    arrives as a keyword argument, as in the reference.  The math is the dense path's: only cache addressing changes."""

    def __init__(self, config: FusedMultiTransformerConfig, device=None):
        super().__init__(config, device)
        self.cache_scales_set = False
        if config.cachekv_int8_type is not None:
            # the reference's names (fused_transformer_layers.py:2389-2395): quantise scales s and dequantise scales o = 1 / s,
            # bf16 [kvh] per layer; zero until set_cache_scales()
            for name in ("cache_k_scales", "cache_v_scales", "cache_k_out_scales", "cache_v_out_scales"):
                setattr(self, name, [torch.zeros(self.kvh, dtype=BF16, device=self.device) for _ in range(self.L)])

    @torch.no_grad()
    def set_cache_scales(self, k_absmax, v_absmax):
        """Static int8-cache scales from the absolute maxima of the cached K and V values, [L, kvh] each: s = 127 / absmax and
        o = 1 / s in fp64, each cast to bf16 (CacheScaleLoader, experimental/model_utils.py:433-468).  A missing, non-finite or
        non-positive absmax raises ValueError."""
        if self.config.cachekv_int8_type is None:
            raise ValueError("set_cache_scales: the block was built without cachekv_int8_type")
        for name, a in (("k", k_absmax), ("v", v_absmax)):
            a = torch.as_tensor(a, dtype=torch.float64).cpu()
            if tuple(a.shape) != (self.L, self.kvh):
                raise ValueError(f"set_cache_scales: {name} absmax must be [{self.L}, {self.kvh}], got {tuple(a.shape)}")
            if not bool(torch.isfinite(a).all()) or not bool((a > 0).all()):
                bad = [(int(i), int(j)) for i, j in zip(*torch.nonzero(~(torch.isfinite(a) & (a > 0)), as_tuple=True))]
                raise ValueError(f"set_cache_scales: cache {name} absmax must be finite and positive; (layer, kv head) {bad[:8]}")
            s = 127.0 / a
            o = 1.0 / s
            for i in range(self.L):
                getattr(self, f"cache_{name}_scales")[i].copy_(s[i].to(BF16))
                getattr(self, f"cache_{name}_out_scales")[i].copy_(o[i].to(BF16))
        self.cache_scales_set = True

    def check_cache_scales(self, caches):
        """Raise unless a uint8 cache has its scales (the reference runs with -1 scales when the file lacks them)."""
        if caches and caches[0].dtype == ops.CACHE_INT8 and not self.cache_scales_set:
            raise ValueError("the int8 KV cache has no scales: call set_cache_scales() (the reference's cachekv_scales.json) or "
                             "calibrate_cache_scales() first")

    # the scale arguments of the paged ops for layer i: none for a bf16 cache (an int8 block calibrates through one)
    def _write_scales(self, caches, i):
        if caches[2 * i].dtype != ops.CACHE_INT8:
            return {}
        return dict(cache_k_scale=self.cache_k_scales[i], cache_v_scale=self.cache_v_scales[i])

    def _read_scales(self, caches, i):
        if caches[2 * i].dtype != ops.CACHE_INT8:
            return {}
        return dict(cache_k_out_scale=self.cache_k_out_scales[i], cache_v_out_scale=self.cache_v_out_scales[i])

    @staticmethod
    def _tables(kw):
        bt = kw.get("block_tables")
        if bt is None:
            raise ValueError("FusedBlockMultiTransformer needs block_tables=[B, max_blocks_per_seq] int32")
        return bt

    def _write_cache(self, qkv, caches, i, B, S, seq_lens_encoder, kw):
        ops.write_cache_kv_paged(qkv, caches[2 * i], caches[2 * i + 1], self._tables(kw), seq_lens_encoder, B, S, self.nh,
                                 **self._write_scales(caches, i))

    def _rope_append(self, qkv, acc, caches, i, seq_lens_decoder, kw):
        cos, sin = self.rope
        return ops.decode_rope_append_paged(qkv, caches[2 * i], caches[2 * i + 1], self._tables(kw), cos, sin, seq_lens_decoder,
                                            self.nh, acc_f32=acc, bias=self._bias(i) if acc is not None else None,
                                            **self._write_scales(caches, i))

    def _attend(self, qkv, caches, i, seq_lens_decoder, kw):
        return ops.decode_attention_paged(qkv, caches[2 * i], caches[2 * i + 1], self._tables(kw), seq_lens_decoder, self.nh,
                                          **self._read_scales(caches, i))

    # ---- config.append_attn (fused_transformer_layers.py:2215-2262): ONE op does RoPE + cache append + attention for the prompt
    # rows and the decode rows alike; the padded [B, S] prefill layout is the packed layout with cu_seqlens_q[b] = b * S ----
    def _append(self, qkv, caches, i, B, S, enc, dec, this_time, kw):
        cos, sin = self.rope
        cu = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device=qkv.device)
        return ops.append_attention(qkv, caches[2 * i], caches[2 * i + 1], enc, dec, this_time, cu, self._tables(kw), cos, sin,
                                    self.nh, max_q_len=S, **self._write_scales(caches, i), **self._read_scales(caches, i))

    def compute_fmha(self, qkv, caches, i, B, S, seq_lens_encoder, kw):
        packed = kw.get("packed")
        if packed is not None:
            # continuous batching: rows are already packed (get_padding_offset) — prompts, recovered sequences and decode rows
            # of one step in one call; packed = (seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, max_q_len)
            enc, dec, this_time, cu, max_q_len = packed
            cos, sin = self.rope
            return ops.append_attention(qkv, caches[2 * i], caches[2 * i + 1], enc, dec, this_time, cu, self._tables(kw), cos, sin,
                                        self.nh, max_q_len=max_q_len, **self._write_scales(caches, i),
                                        **self._read_scales(caches, i))
        if not self.config.append_attn:
            return super().compute_fmha(qkv, caches, i, B, S, seq_lens_encoder, kw)
        enc = (seq_lens_encoder if seq_lens_encoder is not None
               else torch.full((B,), S, dtype=torch.int32, device=qkv.device)).to(torch.int32)
        return self._append(qkv, caches, i, B, S, enc, torch.zeros_like(enc), enc, kw)

    def compute_mmha(self, qkv, caches, i, seq_lens_decoder, kw):
        if not self.config.append_attn:
            return super().compute_mmha(qkv, caches, i, seq_lens_decoder, kw)
        B = qkv.shape[0]
        one = torch.ones(B, dtype=torch.int32, device=qkv.device)
        return self._append(qkv, caches, i, B, 1, torch.zeros_like(one), seq_lens_decoder, one, kw)


class WeightOnlyInt8Mixin:
    """Layer matrices as int8 weights with one bf16 scale per output channel (quant_type="weight_only_int8";
    FusedMultiTransformerWeightOnly, fused_transformer_layers.py:1221-1440: weight_quantize at load, weight_only_linear in the
    forward).  `<name>_weights[i]` holds the packed int8 weights of the [in, out] matrix W (ops.weight_quantize: [out, in],
    exactly out * in bytes) and `<name>_weights_scale[i]` the bf16 [out] scales; no bf16 copy of a layer matrix is kept.
    Only the per-matrix hooks differ from the bf16 block: the forward, the cache paths and the bf16 head are shared."""

    def _alloc_layer_matrices(self):
        for name in self.MATRICES:
            k, n = self._in_out(name)
            setattr(self, name + "_weights", [torch.zeros(n, k, dtype=torch.int8, device=self.device) for _ in range(self.L)])
            setattr(self, name + "_weights_scale", [torch.zeros(n, dtype=BF16, device=self.device) for _ in range(self.L)])

    def _in_out(self, name):
        rows, cols = self.layer_matrix_shape(name)
        return (cols, rows) if name == "qkv" else (rows, cols)

    def set_layer_matrix(self, name, i, w):
        """Quantise a bf16 matrix of layer_matrix_shape(name) into layer i's int8 weights and scales (on its device)."""
        w_in_out = (w.t() if name == "qkv" else w).to(device=self.device, dtype=BF16).contiguous()
        q, scale = ops.weight_quantize(w_in_out, algo=self.config.quant_type)
        getattr(self, name + "_weights")[i].copy_(q)
        getattr(self, name + "_weights_scale")[i].copy_(scale)

    def linear(self, x, name, i, bias=None):
        return ops.weight_only_linear(x, getattr(self, name + "_weights")[i], bias=bias,
                                      weight_scale=getattr(self, name + "_weights_scale")[i], weight_dtype="int8")

    def linear_f32(self, x, name, i, tag):
        return ops.weight_only_linear_f32(x, getattr(self, name + "_weights")[i], getattr(self, name + "_weights_scale")[i],
                                          tag=tag)

    def ffn1_act(self, x, i):
        # no int8 twin of the fused gate|up + SwiGLU epilogue: fp32 sums, then SwiGLU rounds them and re-zeroes the workspace
        return ops.swiglu_fwd_f32(self.linear_f32(x, "ffn1", i, "splitk_ffn1"))


class FusedMultiTransformerWeightOnly(WeightOnlyInt8Mixin, FusedMultiTransformerBase):
    """Dense-cache block with weight-only int8 layer matrices."""


class FusedBlockMultiTransformerWeightOnly(WeightOnlyInt8Mixin, FusedBlockMultiTransformer):
    """Paged-cache block with weight-only int8 layer matrices."""
