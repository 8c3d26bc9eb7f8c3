"""CPU oracle: straight-line torch restatement of the reference's Llama / Qwen2 decoder math.

TEST INFRASTRUCTURE ONLY.  Nothing under paddlenlp_b200/ may import this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, and only as the checker
or the timed CPU baseline, never as the product path.

What it follows (paths relative to the PaddleNLP tree, /root/reference):
  RMSNorm            paddlenlp/transformers/llama/modeling.py:367-386   (unfused branch)
  rotary tables      paddlenlp/transformers/llama/modeling.py:402-439
  rotate_half/apply  paddlenlp/transformers/llama/modeling.py:557-577
  attention (eager)  paddlenlp/transformers/llama/modeling.py:240-301   (pre-scaled q, triu(-min) mask, fp32 softmax)
  repeat_kv (GQA)    paddlenlp/transformers/llama/modeling.py:389-399
  MLP + swiglu       paddlenlp/transformers/llama/modeling.py:38-45, 632-652
  decoder layer      paddlenlp/transformers/llama/modeling.py:1138-1232
  model loop         paddlenlp/transformers/llama/modeling.py:1634, 1706-1758
  lm_head            paddlenlp/transformers/llama/modeling.py:1894-1921  (weight [hidden, vocab])
  criterion          paddlenlp/transformers/llama/modeling.py:1799-1825  (fp32 CE, ignore_index -100, mask loss>0)
  init               paddlenlp/transformers/llama/modeling.py:1386-1436
  Qwen2 deltas       paddlenlp/transformers/qwen2/modeling.py:266-295 (norm), :478-480 (q/k/v bias), :1166-1181 (loss)

Parity pinning: PaddlePaddle itself is not installable in this environment (no network; it is not under
/root/reference), so this restatement cannot be checked against the reference executing.  It is pinned instead
against HuggingFace `transformers` Llama/Qwen2 with transposed weights — the numerical twin the reference itself
declares in tests/transformers/llama/test_modeling.py:398-506 (LlamaCompatibilityTest, rtol 1e-2 / atol 1e-3) —
see oracle/make_golden.py and tests/test_oracle.py, and against the committed golden vectors in tests/golden/.

Two arithmetic modes:
  mode="fp32" : everything in fp32 (the mathematical reference)
  mode="bf16" : fp32 arithmetic with a round-to-bf16 at every point where the reference's bf16 (AMP O2) path rounds
                (SURVEY.md §8a "rounding points"); this is what the CUDA path is compared against.
Weight layout is Paddle's: every Linear weight is [in_features, out_features].
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch


@dataclass
class RefConfig:
    vocab_size: int = 128256
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    rms_norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    initializer_range: float = 0.02
    max_position_embeddings: int = 8192
    qkv_bias: bool = False          # Qwen2
    model_type: str = "llama"
    rope_scaling: Optional[dict] = None   # {"rope_type": "llama3", ...} or {"type": "linear"|"ntk"|"dynamic_ntk", "factor": f}

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


def llama3_8b() -> RefConfig:
    return RefConfig()


def llama3_2_3b() -> RefConfig:
    """Llama-3.2-3B shapes with untied embeddings (the pre-training benchmark's model)."""
    return RefConfig(hidden_size=3072, intermediate_size=8192, num_hidden_layers=28, num_attention_heads=24, num_key_value_heads=8)


def qwen2_7b() -> RefConfig:
    return RefConfig(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                     num_attention_heads=28, num_key_value_heads=4, rms_norm_eps=1e-6, rope_theta=1e6,
                     qkv_bias=True, model_type="qwen2", max_position_embeddings=32768)


def rnd(x: torch.Tensor, mode: str) -> torch.Tensor:
    """Rounding point: bf16 round-trip in mode 'bf16', identity in 'fp32'."""
    if mode == "bf16":
        return x.to(torch.bfloat16).to(torch.float32)
    return x


# --------------------------------------------------------------------------------------------------
# init  (llama/modeling.py:1386-1436; RMSNorm weight = 1, :356-360; Paddle nn.Linear bias init = 0)
# --------------------------------------------------------------------------------------------------
def init_weights(cfg: RefConfig, seed: int = 42, round_bf16: bool = True) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    h, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    kvd = cfg.num_key_value_heads * cfg.head_dim
    std = cfg.initializer_range
    factor = 1.0 / math.sqrt(2 * cfg.num_hidden_layers)
    pre = cfg.model_type  # "llama" / "qwen2" top-level attribute name in the reference

    def normal(*shape):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    w: Dict[str, torch.Tensor] = {}
    w[f"{pre}.embed_tokens.weight"] = normal(V, h)
    for i in range(cfg.num_hidden_layers):
        p = f"{pre}.layers.{i}."
        w[p + "self_attn.q_proj.weight"] = normal(h, h)
        w[p + "self_attn.k_proj.weight"] = normal(h, kvd)
        w[p + "self_attn.v_proj.weight"] = normal(h, kvd)
        w[p + "self_attn.o_proj.weight"] = normal(h, h) * factor
        if cfg.qkv_bias:
            # Paddle default bias init is zeros; use small non-zero values so the bias path is actually tested.
            w[p + "self_attn.q_proj.bias"] = normal(h)
            w[p + "self_attn.k_proj.bias"] = normal(kvd)
            w[p + "self_attn.v_proj.bias"] = normal(kvd)
        w[p + "mlp.gate_proj.weight"] = normal(h, I)
        w[p + "mlp.up_proj.weight"] = normal(h, I)
        w[p + "mlp.down_proj.weight"] = normal(I, h) * factor
        w[p + "input_layernorm.weight"] = torch.ones(h)
        w[p + "post_attention_layernorm.weight"] = torch.ones(h)
    w[f"{pre}.norm.weight"] = torch.ones(h)
    w["lm_head.weight"] = normal(h, V)
    if round_bf16:
        w = {k: v.to(torch.bfloat16).to(torch.float32) for k, v in w.items()}
    return w


# --------------------------------------------------------------------------------------------------
# ops
# --------------------------------------------------------------------------------------------------
def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float, mode: str) -> torch.Tensor:
    # modeling.py:377-386: variance in fp32; rsqrt(var+eps)*x in fp32; cast to weight dtype; * weight (bf16 mult).
    var = x.pow(2).mean(-1, keepdim=True)
    y = torch.rsqrt(var + eps) * x
    y = rnd(y, mode)
    return rnd(y * weight, mode)


def rope_inv_freq(head_dim: int, theta: float, scaling: Optional[dict] = None, seq_len: int = 0,
                  max_position_embeddings: int = 0) -> torch.Tensor:
    """Inverse frequencies of the reference's rotary variants (llama/modeling.py):
    plain :409-411; Llama3RotaryEmbedding :535-553 (wavelength bands, smooth interpolation between them);
    LlamaNTKScalingRotaryEmbedding :467-470 (base * f**(d/(d-2))); LlamaDynamicNTKScalingRotaryEmbedding :482-487 (the same
    with alpha = f*seq/max_pos - (f-1), only when seq_len > max_position_embeddings)."""
    kind = None if not scaling else (scaling.get("rope_type") or scaling.get("type"))
    base = float(theta)
    if kind == "ntk":
        base = base * float(scaling["factor"]) ** (head_dim / (head_dim - 2))
    elif kind == "dynamic_ntk" and max_position_embeddings and seq_len > max_position_embeddings:
        f = float(scaling["factor"])
        base = base * ((f * seq_len / max_position_embeddings) - (f - 1)) ** (head_dim / (head_dim - 2))
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim))
    if kind == "llama3":
        factor, lo, hi = float(scaling["factor"]), float(scaling["low_freq_factor"]), float(scaling["high_freq_factor"])
        orig = float(scaling["original_max_position_embeddings"])
        wavelen = 2 * math.pi / inv_freq
        smooth = (orig / wavelen - lo) / (hi - lo)
        mid = (1 - smooth) * inv_freq / factor + smooth * inv_freq
        inv_freq = torch.where(wavelen < orig / hi, inv_freq, torch.where(wavelen > orig / lo, inv_freq / factor, mid))
    return inv_freq


def rope_tables(head_dim: int, seq_len: int, theta: float, device="cpu", scaling: Optional[dict] = None,
                max_position_embeddings: int = 0):
    # modeling.py:409-423: inv_freq = 1 / base**(arange(0,dim,2)/dim); emb = concat([freqs, freqs]); cos/sin fp32.
    inv_freq = rope_inv_freq(head_dim, theta, scaling, seq_len, max_position_embeddings)
    t = torch.arange(seq_len, dtype=torch.float32)
    if scaling and (scaling.get("rope_type") or scaling.get("type")) == "linear":
        t = t / float(scaling["factor"])              # LlamaLinearScalingRotaryEmbedding :446-450
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat([freqs, freqs], dim=-1)
    return emb.cos().to(device), emb.sin().to(device)  # [S, d]; always computed on the CPU first


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    d = x.shape[-1] // 2
    return torch.cat([-x[..., d:], x[..., :d]], dim=-1)


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, mode: str,
               position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: [b, s, heads, d].  Rounding follows the FUSED op (fp32 math, one rounding), the choice documented in
    SURVEY.md §8a row a4 (in-tree twin: csrc/gpu/encode_rotary_qk.cu:42-53)."""
    if position_ids is None:
        c = cos[None, : x.shape[1], None, :]
        s = sin[None, : x.shape[1], None, :]
    else:
        c = cos[position_ids][:, :, None, :]
        s = sin[position_ids][:, :, None, :]
    return rnd(x * c + rotate_half(x) * s, mode)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mode: str,
              mask_start: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Causal GQA attention; q [b,s,nh,d], k/v [b,s,kvh,d] -> [b,s,nh*d].
    mask_start [b, s] (optional): FlashMask causal-LT start rows (fusion_ops.py:218-231): key column c is hidden from query
    rows i >= mask_start[b, c]  (packed-document masking, llm/utils/data.py:200-204).
    Rounding points of the flash path (SURVEY.md §8a a5): S, softmax in fp32 with the scale applied to S;
    P rounded to bf16 before P@V; output rounded to bf16."""
    b, s, nh, d = q.shape
    kvh = k.shape[2]
    rep = nh // kvh
    k = k[:, :, :, None, :].expand(b, s, kvh, rep, d).reshape(b, s, nh, d)   # repeat_kv, modeling.py:389-399
    v = v[:, :, :, None, :].expand(b, s, kvh, rep, d).reshape(b, s, nh, d)
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    scores = torch.matmul(qt, kt.transpose(-1, -2)) / math.sqrt(d)
    mask = torch.full((s, s), float("-inf"), device=q.device).triu(1)
    if mask_start is not None:
        rows = torch.arange(s, device=q.device)[None, :, None]                       # [1, s(row), 1]
        hidden = rows >= mask_start.to(q.device)[:, None, :]                         # [b, row, col]
        mask = mask[None].expand(b, s, s).masked_fill(hidden, float("-inf"))[:, None]
    p = torch.softmax(scores + mask, dim=-1)
    p = rnd(p, mode)
    out = torch.matmul(p, vt).transpose(1, 2).reshape(b, s, nh * d)
    return rnd(out, mode)


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], mode: str) -> torch.Tensor:
    y = x @ w                       # Paddle weight layout [in, out]; fp32 accumulate
    if bias is not None:
        y = y + bias                # bias added in fp32 before the single rounding (SURVEY.md §8a a3)
    return rnd(y, mode)


def swiglu(g: torch.Tensor, u: torch.Tensor, mode: str) -> torch.Tensor:
    return rnd(torch.nn.functional.silu(g) * u, mode)   # fused swiglu op: fp32 math, one rounding (a6)


@dataclass
class KvQuant:
    """A static int8 KV cache for the reference forward (oracle/cachekv_int8_ref.py).

    scales      per layer (s_k, o_k, s_v, o_v), bf16 [kvh] each: quantise and dequantise scales
    quant_from  [b] positions: query rows at positions >= quant_from[b] attend over fake-quantised post-RoPE K and V (what
                the cache holds), earlier rows over the unquantised values.  0 restates append_attention, which attends over
                the cache for every row; the prompt length restates the fused path, whose prefill attends over the
                projection's bf16 K / V and whose decode rows read the cache."""
    scales: list
    quant_from: torch.Tensor


def fake_quant_rows(x: torch.Tensor, s, o) -> torch.Tensor:
    """x [b, s, kvh, d], s / o bf16 [kvh] -> the values the int8 cache holds for x, dequantised."""
    from oracle import cachekv_int8_ref as C

    return C.fake_quant(x, s.to(x.device).view(-1, 1), o.to(x.device).view(-1, 1))


def decoder_layer(x: torch.Tensor, w: Dict[str, torch.Tensor], p: str, cfg: RefConfig, cos, sin, mode: str,
                  position_ids=None, capture: Optional[dict] = None, mask_start=None, kv_quant: Optional[KvQuant] = None,
                  layer: int = 0) -> torch.Tensor:
    b, s, h = x.shape
    nh, kvh, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    n1 = rms_norm(x, w[p + "input_layernorm.weight"], cfg.rms_norm_eps, mode)
    q = linear(n1, w[p + "self_attn.q_proj.weight"], w.get(p + "self_attn.q_proj.bias"), mode).reshape(b, s, nh, d)
    k = linear(n1, w[p + "self_attn.k_proj.weight"], w.get(p + "self_attn.k_proj.bias"), mode).reshape(b, s, kvh, d)
    v = linear(n1, w[p + "self_attn.v_proj.weight"], w.get(p + "self_attn.v_proj.bias"), mode).reshape(b, s, kvh, d)
    q = apply_rope(q, cos, sin, mode, position_ids)
    k = apply_rope(k, cos, sin, mode, position_ids)
    if kv_quant is None:
        a = attention(q, k, v, mode, mask_start=mask_start)
    else:
        s_k, o_k, s_v, o_v = kv_quant.scales[layer]
        pos = (torch.arange(s, device=x.device).expand(b, s) if position_ids is None else position_ids.to(x.device))
        quant = pos >= kv_quant.quant_from.to(x.device).view(-1, 1)
        a = attention(q, fake_quant_rows(k, s_k, o_k), fake_quant_rows(v, s_v, o_v), mode, mask_start=mask_start)
        if not bool(quant.all()):
            a = torch.where(quant[:, :, None], a, attention(q, k, v, mode, mask_start=mask_start))
    o = linear(a, w[p + "self_attn.o_proj.weight"], None, mode)
    x1 = rnd(x + o, mode)
    n2 = rms_norm(x1, w[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps, mode)
    g = linear(n2, w[p + "mlp.gate_proj.weight"], None, mode)
    u = linear(n2, w[p + "mlp.up_proj.weight"], None, mode)
    m = swiglu(g, u, mode)
    y = linear(m, w[p + "mlp.down_proj.weight"], None, mode)
    x2 = rnd(x1 + y, mode)
    if capture is not None:
        capture.update(n1=n1, q=q, k=k, v=v, attn=a, x1=x1, n2=n2, act=m, out=x2)
    return x2


def model_forward(input_ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg: RefConfig, mode: str = "bf16",
                  position_ids=None, return_hidden: bool = False, kv_quant: Optional[KvQuant] = None):
    """input_ids [b, s] int64 -> logits [b, s, V] (fp32 tensor holding bf16-rounded values in mode 'bf16').  kv_quant: attend
    over a static int8 KV cache (KvQuant); None is the plain forward."""
    pre = cfg.model_type
    x = w[f"{pre}.embed_tokens.weight"][input_ids]
    cos, sin = rope_tables(cfg.head_dim, max(input_ids.shape[1], int(position_ids.max()) + 1 if position_ids is not None else 0),
                           cfg.rope_theta, x.device, scaling=cfg.rope_scaling, max_position_embeddings=cfg.max_position_embeddings)
    for i in range(cfg.num_hidden_layers):
        x = decoder_layer(x, w, f"{pre}.layers.{i}.", cfg, cos, sin, mode, position_ids, kv_quant=kv_quant, layer=i)
    hf = rms_norm(x, w[f"{pre}.norm.weight"], cfg.rms_norm_eps, mode)
    logits = linear(hf, w["lm_head.weight"], None, mode)
    if return_hidden:
        return logits, hf
    return logits


def criterion(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """LlamaPretrainingCriterion (modeling.py:1799-1825): fp32 CE with reduction none, then mean over loss>0."""
    lg = logits.reshape(-1, logits.shape[-1]).float()
    lb = labels.reshape(-1)
    per_tok = torch.nn.functional.cross_entropy(lg, lb, reduction="none", ignore_index=ignore_index)
    keep = (per_tok > 0).float()
    cnt = keep.sum()
    total = (per_tok * keep).sum()
    return total if cnt.item() == 0 else total / cnt


def loss_and_grads(input_ids, labels, w, cfg: RefConfig, mode: str = "bf16"):
    """Forward + autograd backward of the oracle (casts are straight-through), for gradient parity checks."""
    wl = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    logits = model_forward(input_ids, wl, cfg, mode)
    loss = criterion(logits, labels)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in wl.items()}


# --------------------------------------------------------------------------------------------------
# HF bridge (name map / transposes: llama/modeling.py:1243-1274)
# --------------------------------------------------------------------------------------------------
def to_hf_state_dict(w: Dict[str, torch.Tensor], cfg: RefConfig) -> Dict[str, torch.Tensor]:
    pre = cfg.model_type
    out = {}
    for k, v in w.items():
        if k.startswith(pre + "."):
            hk = "model." + k[len(pre) + 1:]
        else:
            hk = k
        is_linear = k.endswith("_proj.weight") or k == "lm_head.weight"
        out[hk] = v.t().contiguous() if is_linear else v.clone()
    return out


def hf_config(cfg: RefConfig):
    import transformers

    common = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                  num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                  num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps,
                  max_position_embeddings=cfg.max_position_embeddings, tie_word_embeddings=False,
                  attn_implementation="eager")
    if cfg.model_type == "qwen2":
        c = transformers.Qwen2Config(**common)
    else:
        c = transformers.LlamaConfig(attention_bias=False, mlp_bias=False, **common)
    # transformers >= 5 keeps rope settings in rope_parameters; older versions use rope_theta
    try:
        c.rope_theta = cfg.rope_theta
        if getattr(c, "rope_parameters", None) is not None:
            c.rope_parameters["rope_theta"] = cfg.rope_theta
    except Exception:
        pass
    return c
