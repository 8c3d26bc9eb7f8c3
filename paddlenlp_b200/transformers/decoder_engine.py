"""DecoderEngine: the Llama/Qwen2 decoder hot path (forward, backward, flat parameter/gradient buffers).

This is the host-side orchestration of the sm_90a kernels behind the C-ABI.  It replaces the per-op eager execution
of the reference's
    LlamaModel.forward            paddlenlp/transformers/llama/modeling.py:1588-1774
    LlamaDecoderLayer.forward     paddlenlp/transformers/llama/modeling.py:1138-1232
    LlamaAttention.forward        paddlenlp/transformers/llama/modeling.py:866-1119
    LlamaMLP.forward              paddlenlp/transformers/llama/modeling.py:632-652
    LlamaLMHead / Criterion       paddlenlp/transformers/llama/modeling.py:1894-1921, 1799-1825
and their autograd backward with an explicit saved-tensor plan.  Per layer, forward is
    rmsnorm -> QKV GEMM(+bias) -> RoPE (in place) -> flash attention -> O GEMM(+residual epilogue)
            -> rmsnorm -> gate|up GEMM -> SwiGLU -> down GEMM(+residual epilogue)
i.e. 4 wgmma GEMMs, 1 mma.sync attention and 4 HBM-bound fusions; the residual adds live in GEMM epilogues.

Data layout in HBM
  * ONE flat bf16 parameter buffer and ONE flat bf16 gradient buffer (the buffer the data-parallel all-reduce and
    the AdamW kernel operate on).  Matrices first (weight-decayed), then norm weights and biases (not decayed).
  * config.tie_word_embeddings: the layout has no `head` entry; the logits are hf @ E^T with E = embed [V, h]
    (llama/modeling.py:1924-1938, LlamaLMHead(transpose_y=True)) and both gradient terms land in the one embed gradient.
  * q/k/v weights are stored fused as [hidden, (nh + 2*kvh) * d] (= concat of the reference's three [in,out]
    matrices along out) and gate/up as [hidden, 2*I]; the reference names are exposed as column-slice views.
  * activations are token-major [T, features] bf16; q/k/v are strided views of the packed QKV projection.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import ops

BF16 = torch.bfloat16


def _align8(n: int) -> int:
    return (n + 7) // 8 * 8


class DecoderEngine:
    def __init__(self, config, device=None, prefix: Optional[str] = None):
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("DecoderEngine needs a CUDA device: the hot path has no CPU implementation")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self.cfg = config
        self.prefix = prefix or config.model_type          # "llama" / "qwen2": top-level name in state dicts
        self.h = config.hidden_size
        self.nh = config.num_attention_heads
        self.kvh = config.num_key_value_heads
        self.d = self.h // self.nh
        self.I = config.intermediate_size
        self.V = config.vocab_size
        self.L = config.num_hidden_layers
        self.eps = config.rms_norm_eps
        self.qkv_bias = config.model_type == "qwen2"
        self.tied = bool(getattr(config, "tie_word_embeddings", False))
        if self.d != 128:
            raise NotImplementedError(f"head_dim {self.d}: the attention kernels are written for head_dim 128")
        if self.h % 8 or self.I % 8 or self.V % 8:
            raise ValueError("hidden_size, intermediate_size and vocab_size must be multiples of 8")
        self.qkv_n = (self.nh + 2 * self.kvh) * self.d
        # SwiGLU fused into the gate|up GEMM epilogue (needs 128-channel tiles); B200_FUSE_SWIGLU=0 selects GEMM + swiglu kernel
        import os as _os
        self.fuse_swiglu = (self.I % 128 == 0) and _os.environ.get("B200_FUSE_SWIGLU", "1") != "0"
        # the backward twin: SwiGLU backward in the down-proj dX epilogue (bit-identical to GEMM + swiglu_bwd kernel; the epilogue reads
        # the saved gate|up values of its accumulator's rows and columns).  B200_FUSE_SWIGLU_BWD=0 unfuses
        self.fuse_swiglu_bwd = (self.I % 64 == 0) and _os.environ.get("B200_FUSE_SWIGLU_BWD", "1") != "0"
        # recompute (llama/modeling.py:1706-1733 `recompute_training_full`): keep only each layer's input and re-run the
        # layer forward inside backward.  Only the "full" granularity exists here (the "full_attn" / "core_attn" splits
        # exist to trade memory against the reference's unfused attention; the fused attention keeps no S x S tensor).
        self.recompute = bool(getattr(config, "recompute", False))
        gran = getattr(config, "recompute_granularity", "full") or "full"
        if self.recompute and gran != "full":
            raise NotImplementedError(f"recompute_granularity={gran!r}: only 'full' (whole decoder layer) is implemented")

        # ---- flat layout: [matrices | vectors] ----
        mats: List[Tuple[str, Tuple[int, ...]]] = [("embed", (self.V, self.h))]
        vecs: List[Tuple[str, Tuple[int, ...]]] = []
        for i in range(self.L):
            mats += [(f"l{i}.qkv_w", (self.h, self.qkv_n)), (f"l{i}.o_w", (self.nh * self.d, self.h)),
                     (f"l{i}.gu_w", (self.h, 2 * self.I)), (f"l{i}.down_w", (self.I, self.h))]
            vecs += [(f"l{i}.ln1", (self.h,)), (f"l{i}.ln2", (self.h,))]
            if self.qkv_bias:
                vecs += [(f"l{i}.qkv_b", (self.qkv_n,))]
        if not self.tied:
            mats += [("head", (self.h, self.V))]
        vecs += [("norm", (self.h,))]
        self._offsets: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        off = 0
        for name, shape in mats:
            self._offsets[name] = (off, shape)
            off += _align8(math.prod(shape))
        self.decay_end = off
        for name, shape in vecs:
            self._offsets[name] = (off, shape)
            off += _align8(math.prod(shape))
        self.numel = off
        self.flat_params = torch.zeros(self.numel, dtype=BF16, device=self.device)
        self.flat_grads = torch.zeros(self.numel, dtype=BF16, device=self.device)
        self.p = {n: self.flat_params[o:o + math.prod(s)].view(s) for n, (o, s) in self._offsets.items()}
        self.g = {n: self.flat_grads[o:o + math.prod(s)].view(s) for n, (o, s) in self._offsets.items()}
        self.grads_fresh = True          # True: the next backward overwrites instead of accumulating
        self.grad_ready_hook = None      # callable(lo, hi): flat_grads[lo:hi] is final (set by distributed.DataParallel)
        self._rope = None
        self._saved = None
        self._bias_f32: Dict[int, torch.Tensor] = {}

    # ------------------------------------------------------------------------------------------------
    # parameters
    # ------------------------------------------------------------------------------------------------
    def num_parameters(self) -> int:
        return sum(math.prod(s) for _, s in self._offsets.values())

    def init_weights(self, seed: int = 42, on_host: Optional[bool] = None):
        """Reference init (llama/modeling.py:1386-1436): N(0, initializer_range) for every Linear / Embedding /
        lm_head weight, o_proj and down_proj scaled by 1/sqrt(2L), RMSNorm weights 1, biases 0.

        on_host=True draws every tensor in fp32 from ONE seeded CPU generator in the reference's parameter order
        (embed_tokens, then per layer q, k, v, o[, q/k/v bias = 0], gate, up, down, then lm_head unless the embeddings are
        tied: a tied model's parameter list has no lm_head), applies the 1/sqrt(2L)
        factor in fp32 and rounds to bf16 once — so a CPU restatement that draws the same way holds the same bits
        (SURVEY.md §8a row a10).  Default: host for models below 2^28 parameters, device draws (bf16 normals straight
        into the flat buffer, same distribution, no 30 GB fp32 host round trip) above."""
        if on_host is None:
            on_host = bool(getattr(self.cfg, "init_on_host", self.num_parameters() < (1 << 28)))
        if on_host:
            return self._init_weights_host(seed)
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        std = self.cfg.initializer_range
        chunk = 1 << 28
        flat = self.flat_params
        for s in range(0, self.decay_end, chunk):
            e = min(self.decay_end, s + chunk)
            flat[s:e].normal_(0.0, std, generator=gen)
        factor = 1.0 / math.sqrt(2 * self.L)
        for i in range(self.L):
            self.p[f"l{i}.o_w"].mul_(factor)
            self.p[f"l{i}.down_w"].mul_(factor)
            self.p[f"l{i}.ln1"].fill_(1.0)
            self.p[f"l{i}.ln2"].fill_(1.0)
            if self.qkv_bias:
                self.p[f"l{i}.qkv_b"].zero_()
        self.p["norm"].fill_(1.0)
        self._bias_f32.clear()

    def _init_weights_host(self, seed: int):
        g = torch.Generator().manual_seed(seed)
        std = float(self.cfg.initializer_range)
        factor = 1.0 / math.sqrt(2 * self.L)
        qn, kn = self.nh * self.d, self.kvh * self.d

        def draw(*shape, scale=1.0):
            t = torch.randn(*shape, generator=g, dtype=torch.float32) * std
            if scale != 1.0:
                t = t * scale
            return t.to(BF16)

        with torch.no_grad():
            self.p["embed"].copy_(draw(self.V, self.h))
            for i in range(self.L):
                w = self.p[f"l{i}.qkv_w"]
                w[:, :qn].copy_(draw(self.h, qn))
                w[:, qn:qn + kn].copy_(draw(self.h, kn))
                w[:, qn + kn:].copy_(draw(self.h, kn))
                self.p[f"l{i}.o_w"].copy_(draw(qn, self.h, scale=factor))
                gu = self.p[f"l{i}.gu_w"]
                gu[:, :self.I].copy_(draw(self.h, self.I))
                gu[:, self.I:].copy_(draw(self.h, self.I))
                self.p[f"l{i}.down_w"].copy_(draw(self.I, self.h, scale=factor))
                self.p[f"l{i}.ln1"].fill_(1.0)
                self.p[f"l{i}.ln2"].fill_(1.0)
                if self.qkv_bias:
                    self.p[f"l{i}.qkv_b"].zero_()
            self.p["norm"].fill_(1.0)
            if not self.tied:
                self.p["head"].copy_(draw(self.h, self.V))
        self._bias_f32.clear()

    def named_views(self, grads: bool = False, flat: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Reference-named views (llama/modeling.py:1243-1274 name map) onto the flat parameter buffer, the flat gradient
        buffer, or any other flat buffer with the same layout (e.g. the optimizer's fp32 master weights)."""
        if flat is not None:
            src = {n: flat[o:o + math.prod(s)].view(s) for n, (o, s) in self._offsets.items()}
        else:
            src = self.g if grads else self.p
        pre = self.prefix
        out = {f"{pre}.embed_tokens.weight": src["embed"]}
        qn, kn = self.nh * self.d, self.kvh * self.d
        for i in range(self.L):
            lp = f"{pre}.layers.{i}."
            w = src[f"l{i}.qkv_w"]
            out[lp + "self_attn.q_proj.weight"] = w[:, :qn]
            out[lp + "self_attn.k_proj.weight"] = w[:, qn:qn + kn]
            out[lp + "self_attn.v_proj.weight"] = w[:, qn + kn:]
            if self.qkv_bias:
                b = src[f"l{i}.qkv_b"]
                out[lp + "self_attn.q_proj.bias"] = b[:qn]
                out[lp + "self_attn.k_proj.bias"] = b[qn:qn + kn]
                out[lp + "self_attn.v_proj.bias"] = b[qn + kn:]
            out[lp + "self_attn.o_proj.weight"] = src[f"l{i}.o_w"]
            gu = src[f"l{i}.gu_w"]
            out[lp + "mlp.gate_proj.weight"] = gu[:, :self.I]
            out[lp + "mlp.up_proj.weight"] = gu[:, self.I:]
            out[lp + "mlp.down_proj.weight"] = src[f"l{i}.down_w"]
            out[lp + "input_layernorm.weight"] = src[f"l{i}.ln1"]
            out[lp + "post_attention_layernorm.weight"] = src[f"l{i}.ln2"]
        out[f"{pre}.norm.weight"] = src["norm"]
        if not self.tied:
            out["lm_head.weight"] = src["head"]
        return out

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Copies every named view from `sd`.  Entries without a view are ignored: a tied model takes a state dict that
        still carries `lm_head.weight` and keeps its embedding (the reference's tie_weights() after load)."""
        views = self.named_views()
        missing = [k for k in views if k not in sd]
        if missing:
            raise KeyError(f"state dict is missing {len(missing)} tensors, e.g. {missing[:3]}")
        with torch.no_grad():
            for k, dst in views.items():
                src = sd[k]
                if tuple(src.shape) != tuple(dst.shape):
                    raise ValueError(f"{k}: shape {tuple(src.shape)} != {tuple(dst.shape)}")
                dst.copy_(src.to(device=self.device, dtype=BF16))
        self._bias_f32.clear()

    def _bias(self, i: int) -> Optional[torch.Tensor]:
        if not self.qkv_bias:
            return None
        b = self._bias_f32.get(i)
        if b is None:
            b = self.p[f"l{i}.qkv_b"].float()
            self._bias_f32[i] = b
        return b

    def params_changed(self):
        """Call after the optimizer updated the flat buffer (fp32 bias copies are stale)."""
        self._bias_f32.clear()

    def _rope_tables(self, need_pos: int):
        if self._rope is None or self._rope[0].shape[0] < need_pos:
            mpe = int(getattr(self.cfg, "max_position_embeddings", 0) or 0)
            n = max(need_pos, mpe)
            spec = self.cfg.rope_scaling_spec() if hasattr(self.cfg, "rope_scaling_spec") else None
            if spec and spec.get("type") == "linear":
                n = max(n, int(mpe * float(spec["factor"])))             # llama/modeling.py:443: table covers mpe * factor
            self._rope = ops.rope_tables(self.d, n, float(self.cfg.rope_theta), self.device, scaling=spec,
                                         max_position_embeddings=mpe)
        return self._rope

    # ------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------
    def _layer_fwd(self, i: int, x: torch.Tensor, B: int, S: int, pos, save: Optional[list], mask=None):
        T = B * S
        p = self.p
        n1, rstd1 = ops.rmsnorm_fwd(x, p[f"l{i}.ln1"], self.eps)
        qkv = ops.gemm(n1, p[f"l{i}.qkv_w"], bias=self._bias(i))
        cos, sin = self._rope
        ops.rope_inplace(qkv, cos, sin, S, self.nh + self.kvh, self.d, position_ids=pos)
        q4 = qkv.view(B, S, self.qkv_n)
        qn, kn = self.nh * self.d, self.kvh * self.d
        q = q4[:, :, :qn].unflatten(2, (self.nh, self.d))
        k = q4[:, :, qn:qn + kn].unflatten(2, (self.kvh, self.d))
        v = q4[:, :, qn + kn:].unflatten(2, (self.kvh, self.d))
        attn, lse = ops.flash_attn_fwd(q, k, v, mask_start=mask)
        attn2 = attn.view(T, qn)
        x1 = ops.gemm(attn2, p[f"l{i}.o_w"], residual=x)
        n2, rstd2 = ops.rmsnorm_fwd(x1, p[f"l{i}.ln2"], self.eps)
        if self.fuse_swiglu:
            gu, m = ops.gemm_swiglu(n2, p[f"l{i}.gu_w"])          # SwiGLU in the gate|up GEMM's epilogue
        else:
            gu = ops.gemm(n2, p[f"l{i}.gu_w"])
            m = ops.swiglu_fwd(gu)
        x2 = ops.gemm(m, p[f"l{i}.down_w"], residual=x1)
        if save is not None:
            save.append((x, rstd1, n1, qkv, attn2, lse, x1, rstd2, n2, gu, m))
        return x2

    def _layer_fwd_ckpt(self, i: int, x: torch.Tensor, B: int, S: int, pos, save: Optional[list], mask=None):
        """Recompute mode: run the layer without keeping its activations; remember only the layer input."""
        x2 = self._layer_fwd(i, x, B, S, pos, None, mask)
        if save is not None:
            save.append((x,))
        return x2

    def _prep_inputs(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor]):
        if input_ids.dim() != 2:
            raise ValueError("input_ids must be [batch, seq]")
        B, S = input_ids.shape
        ids = input_ids.to(device=self.device, dtype=torch.int64, non_blocking=True).contiguous().view(-1)
        pos = None
        need = S
        if position_ids is not None:
            pos = position_ids.to(device=self.device, dtype=torch.int32, non_blocking=True).contiguous().view(-1)
            need = max(S, int(getattr(self.cfg, "max_position_embeddings", S)))
        self._rope_tables(need)
        return B, S, ids, pos

    def _prep_mask(self, attn_mask_startend_row_indices, B: int, S: int):
        """FlashMask start rows -> int32 [B, S] on the device, in the kernels' canonical form: every column is visible at least
        to its own row.  The reference right-pads the indices with 0 (tokenizer_utils_base.py:3256-3264: padding columns hidden
        from every row, which leaves the padding rows with an empty softmax); here a padding column becomes a one-token
        document — same result for every real token, finite values on the (label -100) padding rows."""
        if attn_mask_startend_row_indices is None:
            return None
        ms = attn_mask_startend_row_indices.to(device=self.device, dtype=torch.int32, non_blocking=True).reshape(B, S)
        own = torch.arange(1, S + 1, dtype=torch.int32, device=self.device)
        ms = torch.maximum(ms, own[None, :]).contiguous()
        if not getattr(self, "_mask_form_checked", False):
            # one-time (first batch) check of the form the kernels rely on for tile skipping: non-decreasing start rows, i.e.
            # contiguous packed documents.  Costs one host sync, once per engine.
            self._mask_form_checked = True
            if S > 1 and bool((ms[:, 1:] < ms[:, :-1]).any()):
                raise ValueError("attn_mask_startend_row_indices must be non-decreasing along the sequence (packed contiguous "
                                 "samples, each column -> end of its sample); general FlashMask patterns are not implemented")
        return ms

    def hidden_states(self, input_ids, position_ids=None, save: Optional[list] = None, attn_mask_startend_row_indices=None):
        """Embedding + decoder stack + final norm -> ([T, h] normed states, pre-norm states, rstd)."""
        B, S, ids, pos = self._prep_inputs(input_ids, position_ids)
        mask = self._prep_mask(attn_mask_startend_row_indices, B, S)
        self._mask = mask
        x = ops.embedding_fwd(ids, self.p["embed"])
        layer = self._layer_fwd_ckpt if (self.recompute and save is not None) else self._layer_fwd
        for i in range(self.L):
            x = layer(i, x, B, S, pos, save, mask)
        hf, rstd_f = ops.rmsnorm_fwd(x, self.p["norm"], self.eps)
        return B, S, ids, pos, x, hf, rstd_f

    def _logits(self, hf: torch.Tensor) -> torch.Tensor:
        """[T, V] = hf @ head, or hf @ E^T when tied (E [V, h] is the GEMM's K-major B operand)."""
        if self.tied:
            return ops.gemm(hf, self.p["embed"], trans_b=True)
        return ops.gemm(hf, self.p["head"])

    @torch.no_grad()
    def forward_logits(self, input_ids, position_ids=None, attn_mask_startend_row_indices=None) -> torch.Tensor:
        """Inference forward: logits [B, S, V] (bf16).  Nothing is saved for backward."""
        B, S, ids, pos, x, hf, _ = self.hidden_states(input_ids, position_ids, save=None,
                                                      attn_mask_startend_row_indices=attn_mask_startend_row_indices)
        logits = self._logits(hf)
        return logits.view(B, S, self.V)

    @torch.no_grad()
    def forward_loss(self, input_ids, labels, position_ids=None, ignore_index: int = -100, keep_for_backward=True,
                     attn_mask_startend_row_indices=None):
        """Training forward: returns loss_out (device [2] = masked-mean loss, token count).
        Activations are kept for backward().  attn_mask_startend_row_indices [B, S]: FlashMask start rows of packed
        samples (llama/modeling.py:1588-1774 forwards it to every layer's attention)."""
        save: Optional[list] = [] if keep_for_backward else None
        B, S, ids, pos, x, hf, rstd_f = self.hidden_states(input_ids, position_ids, save=save,
                                                           attn_mask_startend_row_indices=attn_mask_startend_row_indices)
        logits = self._logits(hf)
        lab = labels.to(device=self.device, dtype=torch.int64, non_blocking=True).contiguous().view(-1)
        loss_out, loss_tok, lse = ops.ce_fwd(logits, lab, ignore_index)
        if keep_for_backward:
            self._saved = dict(B=B, S=S, ids=ids, pos=pos, mask=self._mask, layers=save, x_last=x, hf=hf, rstd_f=rstd_f, logits=logits,
                               labels=lab, loss_tok=loss_tok, lse=lse, loss_out=loss_out)
        return loss_out, logits.view(B, S, self.V)

    @torch.no_grad()
    def forward_logits_train(self, input_ids, position_ids=None, attn_mask_startend_row_indices=None) -> torch.Tensor:
        """Training forward WITHOUT the fused criterion: logits [B, S, V] (bf16) with the activations kept, for a caller-side
        loss (Trainer(criterion=<any callable>), trainer.py:2157-2197).  backward(dlogits=...) completes the step."""
        save: list = []
        B, S, ids, pos, x, hf, rstd_f = self.hidden_states(input_ids, position_ids, save=save,
                                                           attn_mask_startend_row_indices=attn_mask_startend_row_indices)
        logits = self._logits(hf)
        self._saved = dict(B=B, S=S, ids=ids, pos=pos, mask=self._mask, layers=save, x_last=x, hf=hf, rstd_f=rstd_f,
                           logits=None, labels=None)
        return logits.view(B, S, self.V)

    # ------------------------------------------------------------------------------------------------
    # backward
    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def backward(self, grad_scale: float = 1.0, grad_scale_dev: Optional[torch.Tensor] = None,
                 dlogits: Optional[torch.Tensor] = None):
        """Backward of the last forward_loss() (or forward_logits_train() + caller-supplied `dlogits` [T, V] bf16): gradients
        are accumulated into flat_grads (or overwrite it if grads_fresh).  The logits buffer is consumed (overwritten by
        dlogits)."""
        st = self._saved
        if st is None:
            raise RuntimeError("backward() without a preceding forward_loss()")
        self._saved = None
        acc = not self.grads_fresh
        p, g = self.p, self.g
        B, S = st["B"], st["S"]
        if st["labels"] is None:
            if dlogits is None:
                raise RuntimeError("backward() after forward_logits_train() needs dlogits")
            dlogits = dlogits.reshape(B * S, self.V)
            if dlogits.dtype != BF16 or not dlogits.is_contiguous():
                dlogits = dlogits.to(BF16).contiguous()
            if grad_scale != 1.0:
                dlogits = dlogits * grad_scale
        else:
            dlogits = ops.ce_bwd_(st["logits"], st["labels"], st["loss_tok"], st["lse"], st["loss_out"], grad_scale,
                                  grad_scale_dev)
        hook, self.grad_ready_hook = self.grad_ready_hook, None      # one backward per arming
        if self.tied:
            # dhf = dlogits @ E; the head's term dlogits^T @ hf starts (or adds to) the embedding gradient, and the token
            # scatter of embedding_bwd adds on top after the layers
            dhf = ops.gemm(dlogits, p["embed"])
            ops.gemm(dlogits, st["hf"], out=g["embed"], trans_a=True, accumulate=acc)
        else:
            dhf = ops.gemm(dlogits, p["head"], trans_b=True)
            ops.gemm(st["hf"], dlogits, out=g["head"], trans_a=True, accumulate=acc)
            if hook is not None:
                hook(*self._range("head", "head"))
        del dlogits
        st["logits"] = None
        dx = ops.rmsnorm_bwd(dhf, st["x_last"], p["norm"], st["rstd_f"], g["norm"], accumulate_dw=acc)
        del dhf
        layers = st["layers"]
        for i in range(self.L - 1, -1, -1):
            dx = self._layer_bwd(i, dx, layers[i], B, S, st["pos"], acc, st.get("mask"))
            layers[i] = None
            if hook is not None:
                hook(*self._range(f"l{i}.qkv_w", f"l{i}.down_w"))       # this layer's four matrices are contiguous
        if not acc and not self.tied:
            g["embed"].zero_()
        ops.embedding_bwd(st["ids"], dx, g["embed"])
        if hook is not None:
            hook(*self._range("embed", "embed"))
            hook(self.decay_end, self.numel)                            # norm weights / biases of every layer
        self.grads_fresh = False

    def _range(self, first: str, last: str):
        """[lo, hi) of the flat buffers covering the parameters `first` .. `last` (contiguous in the layout)."""
        lo = self._offsets[first][0]
        o, shp = self._offsets[last]
        return lo, o + _align8(math.prod(shp))

    def _layer_bwd(self, i, dx2, saved, B, S, pos, acc, mask=None):
        if len(saved) == 1:                      # recompute: rebuild this layer's activations from its input
            tmp: list = []
            self._layer_fwd(i, saved[0], B, S, pos, tmp, mask)
            saved = tmp[0]
        (x, rstd1, n1, qkv, attn2, lse, x1, rstd2, n2, gu, m) = saved
        p, g = self.p, self.g
        T = B * S
        qn, kn = self.nh * self.d, self.kvh * self.d
        # ---- MLP ----
        if self.fuse_swiglu_bwd:
            dgu = ops.gemm_swiglu_bwd(dx2, p[f"l{i}.down_w"], gu)      # SwiGLU backward in the dX GEMM's epilogue
            ops.gemm(m, dx2, out=g[f"l{i}.down_w"], trans_a=True, accumulate=acc)
            del m
        else:
            dm = ops.gemm(dx2, p[f"l{i}.down_w"], trans_b=True)
            ops.gemm(m, dx2, out=g[f"l{i}.down_w"], trans_a=True, accumulate=acc)
            del m
            dgu = ops.swiglu_bwd(gu, dm)
            del dm
        dn2 = ops.gemm(dgu, p[f"l{i}.gu_w"], trans_b=True)
        ops.gemm(n2, dgu, out=g[f"l{i}.gu_w"], trans_a=True, accumulate=acc)
        del dgu, gu, n2
        dx1 = ops.rmsnorm_bwd(dn2, x1, p[f"l{i}.ln2"], rstd2, g[f"l{i}.ln2"], dres=dx2, accumulate_dw=acc)
        del dn2, dx2, x1
        # ---- attention ----
        dattn = ops.gemm(dx1, p[f"l{i}.o_w"], trans_b=True)
        ops.gemm(attn2, dx1, out=g[f"l{i}.o_w"], trans_a=True, accumulate=acc)
        q4 = qkv.view(B, S, self.qkv_n)
        q = q4[:, :, :qn].unflatten(2, (self.nh, self.d))
        k = q4[:, :, qn:qn + kn].unflatten(2, (self.kvh, self.d))
        v = q4[:, :, qn + kn:].unflatten(2, (self.kvh, self.d))
        dqkv = torch.empty_like(qkv)
        d4 = dqkv.view(B, S, self.qkv_n)
        dq = d4[:, :, :qn].unflatten(2, (self.nh, self.d))
        dk = d4[:, :, qn:qn + kn].unflatten(2, (self.kvh, self.d))
        dv = d4[:, :, qn + kn:].unflatten(2, (self.kvh, self.d))
        ops.flash_attn_bwd(q, k, v, attn2.view(B, S, self.nh, self.d), dattn.view(B, S, self.nh, self.d), lse, dq, dk, dv,
                           mask_start=mask)
        del dattn, attn2, qkv, q, k, v, q4
        cos, sin = self._rope
        ops.rope_inplace(dqkv, cos, sin, S, self.nh + self.kvh, self.d, position_ids=pos, backward=True)
        if self.qkv_bias:
            ops.colsum(dqkv, g[f"l{i}.qkv_b"], accumulate=acc)
        dn1 = ops.gemm(dqkv, p[f"l{i}.qkv_w"], trans_b=True)
        ops.gemm(n1, dqkv, out=g[f"l{i}.qkv_w"], trans_a=True, accumulate=acc)
        del dqkv, n1
        dx0 = ops.rmsnorm_bwd(dn1, x, p[f"l{i}.ln1"], rstd1, g[f"l{i}.ln1"], dres=dx1, accumulate_dw=acc)
        return dx0

    def clear_grad(self):
        """Lazy clear: the next backward overwrites the gradient buffer instead of accumulating into it."""
        self.grads_fresh = True
