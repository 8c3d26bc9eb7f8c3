"""Thin torch-tensor wrappers over the C-ABI (include/b200nlp.h).

PyTorch is only the device-memory carrier here: every function validates shapes/dtypes, allocates outputs with
torch.empty and forwards raw pointers + the current CUDA stream to libb200nlp.so.  No op has a fallback.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib
from ._lib import call, ptr, stream_ptr

BF16 = torch.bfloat16
# The decode-attention kernels (dense, paged and the decode rows of append_attention) are compiled for these GQA group sizes
# (query heads per kv head) and accept at most this many split-KV partials per (sequence, head).
DECODE_GQA_GROUPS = range(1, 9)
DECODE_MAX_SPLITS = 64
# Every attention kernel (training forward / backward, decode, append_attention) is compiled for these head dims.
ATTENTION_HEAD_DIMS = (64, 128)


def check_head_dim(head_dim: int, what: str) -> None:
    """Raise NotImplementedError unless the attention kernels are compiled for `head_dim`."""
    if head_dim not in ATTENTION_HEAD_DIMS:
        raise NotImplementedError(f"{what}: head_dim {head_dim} is not supported; the attention kernels are written for head_dim "
                                  f"{' and '.join(map(str, ATTENTION_HEAD_DIMS))}")


def _chk(t: torch.Tensor, name: str, dtype=BF16):
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (the hot path has no CPU fallback)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")


def _is_f32_grad(t: torch.Tensor, name: str) -> bool:
    """A gradient operand is bf16, or fp32 (fp32 master gradients, amp_master_grad): True for fp32."""
    _chk(t, name, torch.float32 if t.dtype == torch.float32 else BF16)
    return t.dtype == torch.float32


_workspaces = {}


def _workspace(nbytes: int, device, tag: str = "") -> torch.Tensor:
    """Grow-only scratch buffer per (device, tag); kernels never allocate, the caller (this module) does."""
    key = (device, tag)
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)
        _workspaces[key] = buf
    return buf


def _zero_workspace(nbytes: int, device, tag: str) -> torch.Tensor:
    """Scratch buffer that is zero-filled when (re)allocated; its users must hand it back zeroed."""
    key = (device, tag)
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.zeros(max(int(nbytes), 1), dtype=torch.uint8, device=device)
        _workspaces[key] = buf
    return buf


# ----------------------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *, trans_a: bool = False,
         trans_b: bool = False, accumulate: bool = False, bias: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, max_ctas: int = 0) -> torch.Tensor:
    """out (+)= op(a) @ op(b) (+ bias)   or   out = bf16(bf16(op(a) @ op(b) + bias) + residual).
    a, b 2-D bf16 with unit inner stride.
    trans_a: a is stored [K, M];  trans_b: b is stored [N, K].  Default b layout [K, N] is Paddle's nn.Linear weight.
    An fp32 `out` (fp32 weight gradients) takes the fp32-output form: out = op(a) @ op(b), or out += op(a) @ op(b) with one
    fp32 add per element and no bf16 rounding; it has no bias, residual or max_ctas."""
    _chk(a, "a"); _chk(b, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if trans_a:
        K, M = a.shape
    else:
        M, K = a.shape
    if trans_b:
        N, Kb = b.shape
    else:
        Kb, N = b.shape
    if K != Kb:
        raise ValueError(f"gemm: inner dimensions differ ({K} vs {Kb})")
    if out is None:
        if accumulate:
            raise ValueError("gemm: accumulate=True needs an output tensor")
        out = torch.empty(M, N, dtype=BF16, device=a.device)
    if _is_f32_grad(out, "out"):
        if bias is not None or residual is not None or max_ctas:
            raise ValueError("gemm: an fp32 output takes no bias, residual or max_ctas")
        assert out.shape == (M, N) and out.stride(1) == 1
        call("b200_gemm_bf16_f32", ptr(a), ptr(b), ptr(out), M, N, K, a.stride(0), b.stride(0), out.stride(0),
             1 if trans_a else 0, 0 if trans_b else 1, 1 if accumulate else 0, stream_ptr())
        return out
    assert out.shape == (M, N) and out.stride(1) == 1
    if bias is not None:
        _chk(bias, "bias", torch.float32)
        assert bias.numel() == N
    ldr = 0
    if residual is not None:
        _chk(residual, "residual")
        assert residual.shape == (M, N) and residual.stride(1) == 1 and not accumulate
        ldr = residual.stride(0)
    call("b200_gemm_bf16_ex", ptr(a), ptr(b), ptr(out), ptr(bias), ptr(residual), M, N, K, a.stride(0), b.stride(0),
         out.stride(0), ldr, 1 if trans_a else 0, 0 if trans_b else 1, 1 if accumulate else 0, max_ctas, stream_ptr())
    return out


def gemm_swiglu(x: torch.Tensor, w_gate_up: torch.Tensor, gate_up: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, store_gate_up: bool = True):
    """(gate_up [M, 2I], m [M, I]) = fused gate|up projection + SwiGLU (one wgmma GEMM; the epilogue holds gate and up of the
    same channels).  w_gate_up is the reference-layout fused weight [K, 2I] (gate | up).  Requires I % 64 == 0.
    store_gate_up=False (inference): only m is written and (None, m) is returned."""
    _chk(x, "x"); _chk(w_gate_up, "w_gate_up")
    assert x.dim() == 2 and w_gate_up.dim() == 2 and x.stride(1) == 1 and w_gate_up.stride(1) == 1
    M, K = x.shape
    Kw, two_i = w_gate_up.shape
    if K != Kw or two_i % 2:
        raise ValueError(f"gemm_swiglu: shapes {tuple(x.shape)} x {tuple(w_gate_up.shape)}")
    inter = two_i // 2
    if gate_up is None and store_gate_up:
        gate_up = torch.empty(M, two_i, dtype=BF16, device=x.device)
    if out is None:
        out = torch.empty(M, inter, dtype=BF16, device=x.device)
    call("b200_gemm_swiglu_bf16", ptr(x), ptr(w_gate_up), ptr(gate_up) if store_gate_up else 0, ptr(out), M, inter, K, x.stride(0),
         w_gate_up.stride(0), gate_up.stride(0) if store_gate_up else two_i, out.stride(0), stream_ptr())
    return (gate_up if store_gate_up else None), out


def gemm_swiglu_bwd(dy: torch.Tensor, w_down: torch.Tensor, gate_up: torch.Tensor,
                    dgate_up: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dgate_up [M, 2I] = SwiGLU backward of d(m) = dy @ w_down^T, computed in the GEMM epilogue (d(m) is never written).
    w_down is the reference-layout down_proj weight [I, h]; gate_up the saved projection [M, 2I].  Requires I % 64 == 0."""
    _chk(dy, "dy"); _chk(w_down, "w_down"); _chk(gate_up, "gate_up")
    M, K = dy.shape
    inter, Kw = w_down.shape
    assert K == Kw and gate_up.shape == (M, 2 * inter) and dy.stride(1) == 1 and w_down.stride(1) == 1 and gate_up.stride(1) == 1
    if dgate_up is None:
        dgate_up = torch.empty_like(gate_up)
    call("b200_gemm_swiglu_bwd_bf16", ptr(dy), ptr(w_down), ptr(gate_up), ptr(dgate_up), M, inter, K, dy.stride(0), w_down.stride(0),
         gate_up.stride(0), dgate_up.stride(0), stream_ptr())
    return dgate_up


def gemm_skinny(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, *, trans_b: bool = False,
                bias: Optional[torch.Tensor] = None, split_k: int = 0) -> torch.Tensor:
    """Decode-step GEMM (few token rows, weight-streaming bound): split-K over all SMs, fp32 TMA reduce, one rounding."""
    _chk(a, "a"); _chk(b, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = a.shape
    N, Kb = (b.shape if trans_b else (b.shape[1], b.shape[0]))
    if K != Kb:
        raise ValueError(f"gemm_skinny: inner dimensions differ ({K} vs {Kb})")
    if out is None:
        out = torch.empty(M, N, dtype=BF16, device=a.device)
    if bias is not None:
        _chk(bias, "bias", torch.float32)
    ws = _zero_workspace(M * N * 4, a.device, "splitk")
    call("b200_gemm_bf16_splitk", ptr(a), ptr(b), ptr(out), ptr(bias), ptr(ws), M, N, K, a.stride(0), b.stride(0),
         out.stride(0), 0, 0 if trans_b else 1, split_k, stream_ptr())
    return out


def reserve_gemm_skinny_workspace(max_rows: int, max_cols: int, device) -> None:
    """Size gemm_skinny's split-K workspace for every call up to max_rows x max_cols now.  The buffer grows with the row
    count, and a CUDA graph captured later bakes in its address: it must not be reallocated while such a graph lives."""
    device = torch.empty(0, device=device).device        # the key gemm_skinny uses: a tensor's device, index included
    _zero_workspace(int(max_rows) * int(max_cols) * 4, device, "splitk")


def gemm_skinny_f32(a: torch.Tensor, b: torch.Tensor, *, trans_b: bool = False, split_k: int = 0, tag: str = "splitk_f32"):
    """Split-K GEMM that leaves its result as fp32 sums in a (zero-on-entry) workspace [M, N]; the consumer kernel
    (add_rmsnorm_f32 / decode_rope_append_f32) rounds once and re-zeroes it.  Returns the fp32 workspace view."""
    _chk(a, "a"); _chk(b, "b")
    M, K = a.shape
    N = b.shape[0] if trans_b else b.shape[1]
    ws = _zero_workspace(M * N * 4, a.device, tag)
    call("b200_gemm_bf16_splitk", ptr(a), ptr(b), None, None, ptr(ws), M, N, K, a.stride(0), b.stride(0), N, 0,
         0 if trans_b else 1, split_k, stream_ptr())
    return ws[: M * N * 4].view(torch.float32).view(M, N)


# ----------------------------------------------------------------------------------------------------------
# Weight-only int8 (weight_quantize / weight_only_linear, --quant_type weight_only_int8)
# ----------------------------------------------------------------------------------------------------------
SKINNY_M = 128     # at or below this many token rows the weight-only GEMM may split K (the decode-step workspace covers it)


def weight_quantize(x: torch.Tensor, algo: str = "weight_only_int8"):
    """(weight, weight_scale) of a bf16 [K, N] matrix (Paddle's [in, out] layout): per-output-channel scales bf16 [N] and the
    int8 weights in the GEMM's packed layout (include/b200nlp.h), int8 [N, K] holding exactly N * K bytes."""
    if algo == "weight_only_int4":
        raise NotImplementedError("weight_quantize: weight_only_int4 is not implemented")
    if algo != "weight_only_int8":
        raise ValueError(f"weight_quantize: unknown algo {algo!r}")
    _chk(x, "x")
    assert x.dim() == 2 and x.stride(1) == 1
    K, N = x.shape
    weight = torch.empty(N, K, dtype=torch.int8, device=x.device)
    scale = torch.empty(N, dtype=BF16, device=x.device)
    call("b200_weight_quantize_int8", ptr(x), ptr(weight), ptr(scale), K, N, x.stride(0), stream_ptr())
    return weight, scale


def _weight_only_args(x, weight, weight_scale, weight_dtype):
    if weight_dtype != "int8":
        raise NotImplementedError(f"weight_only_linear: weight_dtype {weight_dtype!r} is not implemented (int8 only)")
    if weight_scale is None:
        raise ValueError("weight_only_linear: weight_scale is required")
    _chk(x, "x"); _chk(weight, "weight", torch.int8); _chk(weight_scale, "weight_scale")
    if x.dim() != 2 or x.stride(1) != 1 or weight.dim() != 2 or not weight.is_contiguous():
        raise ValueError("weight_only_linear: x [M, K] with unit inner stride and a packed weight [N, K] are required")
    M, K = x.shape
    N = weight.shape[0]
    if weight.shape[1] != K or weight_scale.shape != (N,):
        raise ValueError(f"weight_only_linear: shapes x {tuple(x.shape)}, weight {tuple(weight.shape)}, "
                         f"weight_scale {tuple(weight_scale.shape)}")
    return M, N, K


def weight_only_linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None,
                       weight_scale: Optional[torch.Tensor] = None, weight_dtype: str = "int8",
                       out: Optional[torch.Tensor] = None, split_k: int = 0) -> torch.Tensor:
    """y = bf16(scale * (x @ q) + bias): x bf16 [M, K], (weight, weight_scale) from weight_quantize, bias fp32 [N].
    At M <= SKINNY_M the kernel may split K (split_k 0 = choose) through the "splitk" workspace that gemm_skinny uses; a wider
    call never splits, so it never grows that buffer (a captured CUDA graph may hold its address)."""
    M, N, K = _weight_only_args(x, weight, weight_scale, weight_dtype)
    if out is None:
        out = torch.empty(M, N, dtype=BF16, device=x.device)
    assert out.shape == (M, N) and out.stride(1) == 1
    if bias is not None:
        _chk(bias, "bias", torch.float32)
        assert bias.numel() == N
    ws = None
    if M <= SKINNY_M:
        ws = _zero_workspace(M * N * 4, x.device, "splitk")
    elif split_k > 1:
        raise ValueError(f"weight_only_linear: split_k={split_k} at {M} rows (K is split at most {SKINNY_M} rows)")
    call("b200_weight_only_gemm_bf16", ptr(x), ptr(weight), ptr(weight_scale), ptr(bias), ptr(out), ptr(ws), M, N, K,
         x.stride(0), out.stride(0), split_k, stream_ptr())
    return out


def weight_only_linear_f32(x: torch.Tensor, weight: torch.Tensor, weight_scale: torch.Tensor, *, tag: str = "splitk_f32",
                           split_k: int = 0) -> torch.Tensor:
    """weight_only_linear whose result stays as fp32 sums in a (zero-on-entry) workspace [M, N]; the consumer kernel
    (add_rmsnorm_f32 / decode_rope_append_f32 / swiglu_fwd_f32) rounds once and re-zeroes it, as after gemm_skinny_f32.
    Returns the fp32 workspace view."""
    M, N, K = _weight_only_args(x, weight, weight_scale, "int8")
    ws = _zero_workspace(M * N * 4, x.device, tag)
    call("b200_weight_only_gemm_f32", ptr(x), ptr(weight), ptr(weight_scale), ptr(ws), M, N, K, x.stride(0), split_k,
         stream_ptr())
    return ws[: M * N * 4].view(torch.float32).view(M, N)


# ----------------------------------------------------------------------------------------------------------
# RMSNorm
# ----------------------------------------------------------------------------------------------------------
def rmsnorm_fwd(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None,
                rstd: Optional[torch.Tensor] = None):
    _chk(x, "x"); _chk(w, "w")
    h = x.shape[-1]
    rows = x.numel() // h
    assert x.is_contiguous() and w.numel() == h
    if out is None:
        out = torch.empty_like(x)
    if rstd is None:
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    call("b200_rmsnorm_fwd", ptr(x), ptr(w), ptr(out), ptr(rstd), rows, h, float(eps), stream_ptr())
    return out, rstd


def rmsnorm_bwd(dy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, rstd: torch.Tensor, dw: torch.Tensor,
                dres: Optional[torch.Tensor] = None, accumulate_dw: bool = True, dx: Optional[torch.Tensor] = None):
    """dx = RMSNorm backward (+ dres); dw (+)= its weight gradient, bf16 or fp32 (dw's dtype)."""
    _chk(dy, "dy"); _chk(x, "x"); _chk(w, "w"); _chk(rstd, "rstd", torch.float32)
    name = "b200_rmsnorm_bwd_f32" if _is_f32_grad(dw, "dw") else "b200_rmsnorm_bwd"
    h = x.shape[-1]
    rows = x.numel() // h
    assert dy.is_contiguous() and x.is_contiguous() and dw.numel() == h
    if dx is None:
        dx = torch.empty_like(x)
    ws = _workspace(_lib.load().b200_rmsnorm_bwd_workspace_bytes(rows, h), x.device, "rmsnorm_bwd")
    call(name, ptr(dy), ptr(x), ptr(w), ptr(rstd), ptr(dres), ptr(dx), ptr(dw), 1 if accumulate_dw else 0,
         ptr(ws), rows, h, stream_ptr())
    return dx


def colsum(a: torch.Tensor, out: torch.Tensor, accumulate: bool = True):
    """out[n] (+)= sum over rows of a[rows, n] (a may be a column slice: unit inner stride, any row stride); out bf16 or fp32."""
    _chk(a, "a")
    name = "b200_colsum_f32" if _is_f32_grad(out, "out") else "b200_colsum_bf16"
    rows, n = a.shape
    assert a.stride(1) == 1 and out.numel() == n
    ws = _workspace(_lib.load().b200_colsum_workspace_bytes(rows, n), a.device, "colsum")
    call(name, ptr(a), ptr(out), 1 if accumulate else 0, ptr(ws), rows, n, a.stride(0), stream_ptr())
    return out


# ----------------------------------------------------------------------------------------------------------
# RoPE
# ----------------------------------------------------------------------------------------------------------
def rope_inv_freq(head_dim: int, theta: float, scaling: Optional[dict] = None, seq_len: int = 0,
                  max_position_embeddings: int = 0) -> torch.Tensor:
    """fp32 inverse frequencies [head_dim/2] on the CPU for the reference's rotary variants (llama/modeling.py):
      None / {}                          LlamaRotaryEmbedding                    :402-439
      {"rope_type": "llama3", factor, low_freq_factor, high_freq_factor, original_max_position_embeddings}
                                         Llama3RotaryEmbedding                   :520-554  (Llama-3.1 wavelength bands)
      {"type": "ntk", "factor": f}       LlamaNTKScalingRotaryEmbedding          :464-470  (base * f^(d/(d-2)))
      {"type": "dynamic_ntk", "factor"}  LlamaDynamicNTKScalingRotaryEmbedding   :473-517  (base rescaled only when
                                         seq_len > max_position_embeddings)
      {"type": "linear", "factor": f}    handled in rope_tables (positions / f)  :440-461"""
    kind = None if not scaling else (scaling.get("rope_type") or scaling.get("type"))
    base = float(theta)
    d = head_dim
    if kind == "ntk":
        base = base * float(scaling["factor"]) ** (d / (d - 2))
    elif kind == "dynamic_ntk" and max_position_embeddings and seq_len > max_position_embeddings:
        f = float(scaling["factor"])
        alpha = (f * seq_len / max_position_embeddings) - (f - 1)
        base = base * alpha ** (d / (d - 2))
    inv_freq = 1.0 / (base ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    if kind == "llama3":
        factor = float(scaling["factor"])
        lo, hi = float(scaling["low_freq_factor"]), float(scaling["high_freq_factor"])
        orig = float(scaling["original_max_position_embeddings"])
        low_wavelen, high_wavelen = orig / lo, orig / hi
        out = []
        for freq in inv_freq:                          # per-frequency loop in fp32 tensor arithmetic, as the reference (:540-552)
            wavelen = 2 * math.pi / freq
            if wavelen < high_wavelen:
                out.append(freq)
            elif wavelen > low_wavelen:
                out.append(freq / factor)
            else:
                smooth = (orig / wavelen - lo) / (hi - lo)
                out.append((1 - smooth) * freq / factor + smooth * freq)
        inv_freq = torch.stack(out).to(torch.float32)
    elif kind not in (None, "ntk", "dynamic_ntk", "linear", "default"):
        raise ValueError(f"Unknown RoPE scaling type {kind}")       # llama/modeling.py:864
    return inv_freq


def rope_tables(head_dim: int, max_pos: int, theta: float, device, scaling: Optional[dict] = None,
                max_position_embeddings: int = 0):
    """fp32 cos/sin tables [max_pos, head_dim/2], computed on the CPU exactly as the reference does
    (llama/modeling.py:409-423) so that host and device share bits, then uploaded once."""
    inv_freq = rope_inv_freq(head_dim, theta, scaling, seq_len=max_pos, max_position_embeddings=max_position_embeddings)
    t = torch.arange(max_pos, dtype=torch.float32)
    if scaling and (scaling.get("rope_type") or scaling.get("type")) == "linear":
        t = t / float(scaling["factor"])
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    return freqs.cos().contiguous().to(device), freqs.sin().contiguous().to(device)


def rope_inplace(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, seq_len: int, num_heads: int, head_dim: int,
                 position_ids: Optional[torch.Tensor] = None, backward: bool = False):
    """x: [tokens, ld] view whose first num_heads*head_dim columns are the heads to rotate (row stride = ld)."""
    _chk(x, "x"); _chk(cos, "cos", torch.float32); _chk(sin, "sin", torch.float32)
    assert x.dim() == 2 and x.stride(1) == 1
    tokens = x.shape[0]
    if position_ids is not None:
        _chk(position_ids, "position_ids", torch.int32)
        assert position_ids.numel() == tokens
    else:
        assert cos.shape[0] >= seq_len
    call("b200_rope_inplace", ptr(x), ptr(cos), ptr(sin), ptr(position_ids), tokens, seq_len, x.stride(0), num_heads,
         head_dim, 1 if backward else 0, stream_ptr())
    return x


# ----------------------------------------------------------------------------------------------------------
# SwiGLU / embedding
# ----------------------------------------------------------------------------------------------------------
def swiglu_fwd(gate_up: torch.Tensor, out: Optional[torch.Tensor] = None):
    _chk(gate_up, "gate_up")
    rows, two_i = gate_up.shape
    assert gate_up.is_contiguous() and two_i % 2 == 0
    inter = two_i // 2
    if out is None:
        out = torch.empty(rows, inter, dtype=BF16, device=gate_up.device)
    call("b200_swiglu_fwd", ptr(gate_up), ptr(out), rows, inter, stream_ptr())
    return out


def swiglu_fwd_f32(acc_f32: torch.Tensor, out: Optional[torch.Tensor] = None):
    """SwiGLU fed by the fp32 split-K workspace [rows, 2I] of the ffn1 GEMM (rounded here, workspace re-zeroed)."""
    _chk(acc_f32, "acc_f32", torch.float32)
    rows, two_i = acc_f32.shape
    assert acc_f32.is_contiguous() and two_i % 2 == 0
    inter = two_i // 2
    if out is None:
        out = torch.empty(rows, inter, dtype=BF16, device=acc_f32.device)
    call("b200_swiglu_fwd_f32", ptr(acc_f32), ptr(out), rows, inter, stream_ptr())
    return out


def swiglu_bwd(gate_up: torch.Tensor, dout: torch.Tensor, dgate_up: Optional[torch.Tensor] = None):
    _chk(gate_up, "gate_up"); _chk(dout, "dout")
    rows, two_i = gate_up.shape
    inter = two_i // 2
    assert gate_up.is_contiguous() and dout.is_contiguous() and dout.shape == (rows, inter)
    if dgate_up is None:
        dgate_up = torch.empty_like(gate_up)
    call("b200_swiglu_bwd", ptr(gate_up), ptr(dout), ptr(dgate_up), rows, inter, stream_ptr())
    return dgate_up


def embedding_fwd(ids: torch.Tensor, table: torch.Tensor, out: Optional[torch.Tensor] = None):
    _chk(ids, "ids", torch.int64); _chk(table, "table")
    tokens = ids.numel()
    vocab, h = table.shape
    assert ids.is_contiguous() and table.is_contiguous()
    if out is None:
        out = torch.empty(tokens, h, dtype=BF16, device=table.device)
    call("b200_embedding_fwd", ptr(ids), ptr(table), ptr(out), tokens, h, vocab, stream_ptr())
    return out


def embedding_bwd(ids: torch.Tensor, dout: torch.Tensor, dtable: torch.Tensor):
    """dtable[ids[t]] += dout[t]; dtable bf16 or fp32."""
    _chk(ids, "ids", torch.int64); _chk(dout, "dout")
    name = "b200_embedding_bwd_f32" if _is_f32_grad(dtable, "dtable") else "b200_embedding_bwd"
    vocab, h = dtable.shape
    assert dout.is_contiguous() and dtable.is_contiguous()
    call(name, ptr(ids), ptr(dout), ptr(dtable), ids.numel(), h, vocab, stream_ptr())
    return dtable


# ----------------------------------------------------------------------------------------------------------
# Flash attention
# ----------------------------------------------------------------------------------------------------------
def _tok_stride(t: torch.Tensor, heads: int, d: int) -> int:
    """t: [B, S, heads, d] view with unit stride in d, d-stride between heads and a uniform token stride."""
    B, S, H, D = t.shape
    assert (H, D) == (heads, d) and t.stride(3) == 1 and (H == 1 or t.stride(2) == d)
    ld = t.stride(1)
    assert B == 1 or t.stride(0) == S * ld, "batch stride must be S * token stride"
    return ld


def check_mask_form(mask_start: torch.Tensor) -> None:
    """Raise ValueError unless FlashMask start rows [B, S] (or [B, 1, S]) have the form the attention kernels assume.

    The kernels skip kv tiles (forward: the leading tiles; backward: the q tiles past a kv tile's last column) and decide
    whether a tile needs the mask from one column of it, which is exact only if the canonical start rows (every column
    visible at least to its own row: max(start, c + 1)) are non-decreasing along the sequence, i.e. contiguous packed
    documents.  Any other layout would give wrong values silently.  Raw collator rows (right padding 0) are accepted.
    Check host tensors before they are copied: on a device tensor this synchronises."""
    ms = mask_start.reshape(-1, mask_start.shape[-1])
    S = ms.shape[-1]
    own = torch.arange(1, S + 1, dtype=ms.dtype, device=ms.device)
    canon = torch.maximum(ms, own)
    if S > 1 and bool((canon[:, 1:] < canon[:, :-1]).any()):
        raise ValueError("attn_mask_startend_row_indices must be non-decreasing along the sequence (packed contiguous "
                         "samples, each column -> end of its sample); general FlashMask patterns are not implemented")


def _mask_rows(mask_start, B, S):
    if mask_start is None:
        return None
    _chk(mask_start, "mask_start", torch.int32)
    assert mask_start.is_contiguous() and mask_start.numel() == B * S, "mask_start must be int32 [B, S]"
    return mask_start


def flash_attn_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: Optional[float] = None,
                   out: Optional[torch.Tensor] = None, mask_start: Optional[torch.Tensor] = None):
    """Causal GQA attention.  q [B,S,nh,d], k/v [B,S,kvh,d], d = 64 or 128 (may be strided views of a packed QKV buffer).
    mask_start [B,S] int32 (optional): FlashMask start rows — row i sees column c iff c <= i < mask_start[b, c].
    Returns (o [B,S,nh,d] contiguous, lse [B,nh,S] fp32)."""
    _chk(q, "q"); _chk(k, "k"); _chk(v, "v")
    B, S, nh, d = q.shape
    kvh = k.shape[2]
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    if out is None:
        out = torch.empty(B, S, nh, d, dtype=BF16, device=q.device)
    lse = torch.empty(B, nh, S, dtype=torch.float32, device=q.device)
    call("b200_fa_fwd_flashmask", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(_mask_rows(mask_start, B, S)), B, S, nh, kvh,
         d, _tok_stride(q, nh, d), _tok_stride(k, kvh, d), _tok_stride(v, kvh, d), _tok_stride(out, nh, d),
         float(softmax_scale), stream_ptr())
    return out, lse


def flash_attn_bwd(q, k, v, o, dout, lse, dq, dk, dv, softmax_scale: Optional[float] = None, mask_start=None):
    """Gradients written into dq/dk/dv (views allowed, e.g. slices of a packed dQKV buffer); head_dim 64 or 128."""
    for name, t in (("q", q), ("k", k), ("v", v), ("o", o), ("dout", dout), ("dq", dq), ("dk", dk), ("dv", dv)):
        _chk(t, name)
    _chk(lse, "lse", torch.float32)
    B, S, nh, d = q.shape
    kvh = k.shape[2]
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    ws = _workspace(_lib.load().b200_fa_bwd_workspace_bytes(B, S, nh, d), q.device, "fa_bwd")
    call("b200_fa_bwd_flashmask", ptr(q), ptr(k), ptr(v), ptr(o), ptr(dout), ptr(lse), ptr(_mask_rows(mask_start, B, S)),
         ptr(dq), ptr(dk), ptr(dv), ptr(ws), B, S, nh, kvh, d, _tok_stride(q, nh, d), _tok_stride(k, kvh, d), _tok_stride(v, kvh, d), _tok_stride(o, nh, d),
         _tok_stride(dout, nh, d), _tok_stride(dq, nh, d), _tok_stride(dk, kvh, d), _tok_stride(dv, kvh, d),
         float(softmax_scale), stream_ptr())
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------------------
# Criterion / sampling
# ----------------------------------------------------------------------------------------------------------
def ce_fwd(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100):
    """Returns (loss_out [2] = (masked mean loss, count), loss_tok [T], lse [T])."""
    _chk(logits, "logits"); _chk(labels, "labels", torch.int64)
    T, V = logits.shape
    assert logits.stride(1) == 1 and labels.numel() == T and labels.is_contiguous()
    loss_tok = torch.empty(T, dtype=torch.float32, device=logits.device)
    lse = torch.empty(T, dtype=torch.float32, device=logits.device)
    loss_out = torch.empty(2, dtype=torch.float32, device=logits.device)
    call("b200_ce_fwd", ptr(logits), ptr(labels), ptr(loss_tok), ptr(lse), ptr(loss_out), T, V, logits.stride(0),
         ignore_index, stream_ptr())
    return loss_out, loss_tok, lse


def ce_rows_fwd(logits: torch.Tensor, labels: torch.Tensor, loss_tok: torch.Tensor, pred: Optional[torch.Tensor] = None,
                row0: int = 0, ignore_index: int = -100):
    """Evaluation row pass: `logits` [rows, V] holds rows [row0, row0 + rows) of a [T, V] logits matrix; fills
    loss_tok[row0:row0 + rows] (fp32 [T], as ce_fwd's loss_tok) and, if given, pred[row0:row0 + rows] (int64 [T], as
    argmax) from one read of those rows."""
    _chk(logits, "logits"); _chk(labels, "labels", torch.int64); _chk(loss_tok, "loss_tok", torch.float32)
    rows, V = logits.shape
    T = labels.numel()
    assert logits.stride(1) == 1 and labels.is_contiguous() and loss_tok.is_contiguous() and loss_tok.numel() == T
    assert 0 <= row0 and row0 + rows <= T
    if pred is not None:
        _chk(pred, "pred", torch.int64)
        assert pred.is_contiguous() and pred.numel() == T
    call("b200_ce_rows_fwd", ptr(logits), ptr(labels), ptr(loss_tok), ptr(pred), row0, rows, V, logits.stride(0),
         ignore_index, stream_ptr())


def ce_reduce(loss_tok: torch.Tensor) -> torch.Tensor:
    """loss_out [2] = (masked mean of loss_tok over l > 0, count): ce_fwd's reduction."""
    _chk(loss_tok, "loss_tok", torch.float32)
    assert loss_tok.dim() == 1 and loss_tok.is_contiguous()
    loss_out = torch.empty(2, dtype=torch.float32, device=loss_tok.device)
    call("b200_ce_reduce", ptr(loss_tok), ptr(loss_out), loss_tok.numel(), stream_ptr())
    return loss_out


def ce_bwd_(logits: torch.Tensor, labels: torch.Tensor, loss_tok, lse, loss_out, grad_scale: float = 1.0,
            grad_scale_dev: Optional[torch.Tensor] = None):
    """Overwrites logits with dlogits.  grad_scale_dev: optional fp32 device scalar multiplied into grad_scale."""
    T, V = logits.shape
    if grad_scale_dev is not None:
        _chk(grad_scale_dev, "grad_scale_dev", torch.float32)
    call("b200_ce_bwd", ptr(logits), ptr(labels), ptr(loss_tok), ptr(lse), ptr(loss_out), float(grad_scale),
         ptr(grad_scale_dev), T, V, logits.stride(0), stream_ptr())
    return logits


def argmax(logits: torch.Tensor) -> torch.Tensor:
    _chk(logits, "logits")
    rows, V = logits.shape
    out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    call("b200_argmax_bf16", ptr(logits), ptr(out), rows, V, logits.stride(0), stream_ptr())
    return out


# ----------------------------------------------------------------------------------------------------------
# Optimizer
# ----------------------------------------------------------------------------------------------------------
def grad_sqnorm(grads: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None):
    """out[0] = ||scale * grads||^2 of a bf16 or fp32 gradient buffer."""
    name = "b200_grad_sqnorm_f32" if _is_f32_grad(grads, "grads") else "b200_grad_sqnorm"
    assert grads.is_contiguous()
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=grads.device)
    ws = _workspace(_lib.load().b200_grad_sqnorm_workspace_bytes(), grads.device, "sqnorm")
    call(name, ptr(grads), ptr(out), ptr(ws), grads.numel(), float(scale), stream_ptr())
    return out


def adamw_step(params, grads, master, exp_avg, exp_avg_sq, sqnorm, *, decay_end: int, lr: float, beta1: float,
               beta2: float, eps: float, weight_decay: float, step: int, grad_scale: float = 1.0,
               max_grad_norm: float = 1.0):
    """Clip + AdamW over the flat buffers; grads bf16 or fp32."""
    _chk(params, "params")
    name = "b200_adamw_step_f32" if _is_f32_grad(grads, "grads") else "b200_adamw_step"
    for n_, t in (("master", master), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _chk(t, n_, torch.float32)
    n = params.numel()
    call(name, ptr(params), ptr(grads), ptr(master), ptr(exp_avg), ptr(exp_avg_sq), ptr(sqnorm), n,
         decay_end, float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step), float(grad_scale),
         float(max_grad_norm), stream_ptr())


def bf16_to_f32(src: torch.Tensor, dst: torch.Tensor):
    _chk(src, "src"); _chk(dst, "dst", torch.float32)
    call("b200_bf16_to_f32", ptr(src), ptr(dst), src.numel(), stream_ptr())
    return dst


# ----------------------------------------------------------------------------------------------------------
# Generation path
# ----------------------------------------------------------------------------------------------------------
def add_rmsnorm(x, residual, w, eps, want_normed=True, want_residual=True):
    """(normed, residual_out) = fused_rms_norm(x, w, residual=residual); either output may be skipped."""
    _chk(x, "x")
    h = x.shape[-1]
    rows = x.numel() // h
    normed = torch.empty_like(x) if want_normed else None
    res_out = torch.empty_like(x) if want_residual else None
    call("b200_add_rmsnorm", ptr(x), ptr(residual), ptr(w), ptr(normed), ptr(res_out), rows, h, float(eps), stream_ptr())
    return normed, res_out


def add_rmsnorm_f32(x_f32, residual, w, eps, want_normed=True, want_residual=True):
    """add_rmsnorm whose x is the fp32 split-K workspace of the producing GEMM (consumed and re-zeroed)."""
    _chk(x_f32, "x_f32", torch.float32)
    rows, h = x_f32.shape
    normed = torch.empty(rows, h, dtype=BF16, device=x_f32.device) if want_normed else None
    res_out = torch.empty(rows, h, dtype=BF16, device=x_f32.device) if want_residual else None
    call("b200_add_rmsnorm_f32", ptr(x_f32), ptr(residual), ptr(w), ptr(normed), ptr(res_out), rows, h, float(eps), stream_ptr())
    return normed, res_out


def decode_rope_append_f32(acc_f32, bias, cache, cos, sin, seq_lens, nh, kvh, d):
    """RoPE + cache append on the fp32 split-K QKV accumulation; returns the bf16 packed projection [B, (nh+2kvh)*d]."""
    _chk(acc_f32, "acc_f32", torch.float32); _chk(cache, "cache"); _chk(seq_lens, "seq_lens", torch.int32)
    B, n = acc_f32.shape
    qkv = torch.empty(B, n, dtype=BF16, device=acc_f32.device)
    call("b200_decode_rope_append_f32", ptr(qkv), ptr(acc_f32), ptr(bias), ptr(cache), ptr(cos), ptr(sin), ptr(seq_lens), B,
         nh, kvh, d, cache.shape[3], n, stream_ptr())
    return qkv


def write_cache_kv(qkv, cache, seq_lens, B, S, nh, kvh, d):
    """qkv [B*S, ld] (post-RoPE) -> cache [2, B, kvh, max_len, d] for s < seq_lens[b]."""
    _chk(qkv, "qkv"); _chk(cache, "cache")
    assert cache.is_contiguous() and cache.shape[0] == 2 and cache.shape[1] == B and cache.shape[2] == kvh
    max_len = cache.shape[3]
    call("b200_write_cache_kv", ptr(qkv), ptr(cache), ptr(seq_lens), B, S, nh, kvh, d, max_len, qkv.stride(0), stream_ptr())


def decode_rope_append(qkv, cache, cos, sin, seq_lens, nh, kvh, d):
    _chk(qkv, "qkv"); _chk(cache, "cache"); _chk(seq_lens, "seq_lens", torch.int32)
    B = qkv.shape[0]
    call("b200_decode_rope_append", ptr(qkv), ptr(cache), ptr(cos), ptr(sin), ptr(seq_lens), B, nh, kvh, d, cache.shape[3],
         qkv.stride(0), stream_ptr())


def _decode_splits(B: int, kvh: int, max_len: int) -> int:
    """Split-KV count of the bulk-copy decode-attention kernels (dense, paged and append_attention's decode rows): split only
    when there are too few (b, kv head) pairs to give every SM ~3 CTAs (a split costs partial traffic, a merge launch and a
    CTA boundary), with at most one split per 128 cache rows."""
    return max(1, min((max_len + 127) // 128, (3 * 132 + B * kvh - 1) // (B * kvh), DECODE_MAX_SPLITS))


def decode_attention(qkv, cache, seq_lens, nh, kvh, d, softmax_scale=None, out=None, num_splits: int = 0, impl: str = "tc"):
    """Attention of one query row per sequence over the dense cache [2, B, kvh, max_len, d]: sequence b attends to its first
    min(seq_lens[b] + 1, max_len) rows (the new token was appended at row seq_lens[b]).  GQA group nh / kvh in 1..8,
    d = 64 or 128.  impl "tc": the bulk-copy kernel (decode_attn_tc.cu); "simt": the CUDA-core kernel of generation.cu with plain
    global loads, the cross-check.  num_splits <= 0 lets each pick its split-KV count (at most 64)."""
    _chk(qkv, "qkv"); _chk(cache, "cache"); _chk(seq_lens, "seq_lens", torch.int32)
    B = qkv.shape[0]
    if out is None:
        out = torch.empty(B, nh * d, dtype=BF16, device=qkv.device)
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    max_len = cache.shape[3]
    if impl == "tc":
        if num_splits <= 0:
            num_splits = _decode_splits(B, kvh, max_len)
        fn = "b200_decode_attention_tc"
    elif impl == "simt":
        if num_splits <= 0:
            # enough CTAs for ~8 per SM without making the ranges shorter than ~64 cache rows at full length
            num_splits = max(1, min(max_len // 64, (8 * 132 + B * kvh - 1) // (B * kvh), DECODE_MAX_SPLITS))
        fn = "b200_decode_attention"
    else:
        raise ValueError(f"decode_attention impl {impl!r}")
    ws = None
    if num_splits > 1:
        ws = _workspace(_lib.load().b200_decode_attention_workspace_bytes(B, nh, num_splits), qkv.device, "decode_attn")
    call(fn, ptr(qkv), ptr(cache), ptr(seq_lens), ptr(out), ptr(ws), B, nh, kvh, d, max_len,
         qkv.stride(0), float(softmax_scale), num_splits, stream_ptr())
    return out


# ---- paged ("block") KV cache: FusedBlockMultiTransformer / append_attention ----------------------------------------
# The pages are bf16, or uint8 (cachekv_int8_type="static": include/b200nlp.h gives the formula).  Every paged op dispatches on
# the cache dtype: a uint8 cache needs the per-kv-head bf16 [kvh] scales as keyword arguments (cache_k_scale / cache_v_scale to
# write, cache_k_out_scale / cache_v_out_scale to read), and a bf16 cache refuses them.
CACHE_INT8 = torch.uint8


def _paged_geom(key_cache, value_cache, block_tables):
    dt = CACHE_INT8 if key_cache.dtype == CACHE_INT8 else BF16
    _chk(key_cache, "key_cache", dt); _chk(value_cache, "value_cache", dt); _chk(block_tables, "block_tables", torch.int32)
    assert key_cache.shape == value_cache.shape and key_cache.is_contiguous() and value_cache.is_contiguous()
    assert block_tables.dim() == 2 and block_tables.is_contiguous()
    num_blocks, kvh, block_size, d = key_cache.shape
    return num_blocks, kvh, block_size, d, block_tables.shape[1]


def _cache_scales(key_cache, what, **scales):
    """The scale arguments of a paged op: None for a bf16 cache (which must get none), the checked bf16 [kvh] tensors (in
    argument order) for a uint8 cache (which must get all)."""
    given = {k: v for k, v in scales.items() if v is not None}
    if key_cache.dtype != CACHE_INT8:
        if given:
            raise ValueError(f"{what}: {', '.join(sorted(given))} given for a {key_cache.dtype} cache (scales belong to a uint8 cache)")
        return None
    kvh = key_cache.shape[1]
    out = []
    for name, t in scales.items():
        if t is None:
            raise ValueError(f"{what}: a uint8 cache needs {name}")
        _chk(t, name)
        if tuple(t.shape) != (kvh,) or not t.is_contiguous():
            raise ValueError(f"{what}: {name} must be a contiguous bf16 [{kvh}] tensor, got {tuple(t.shape)}")
        out.append(t)
    return out


def write_cache_kv_paged(qkv, key_cache, value_cache, block_tables, seq_lens, B, S, nh, *, cache_k_scale=None,
                         cache_v_scale=None):
    nb, kvh, bs, d, mb = _paged_geom(key_cache, value_cache, block_tables)
    sc = _cache_scales(key_cache, "write_cache_kv_paged", cache_k_scale=cache_k_scale, cache_v_scale=cache_v_scale)
    if sc is not None:
        call("b200_write_cache_kv_paged_c8", ptr(qkv), ptr(key_cache), ptr(value_cache), ptr(block_tables), ptr(sc[0]), ptr(sc[1]),
             ptr(seq_lens), B, S, nh, kvh, d, bs, mb, qkv.stride(0), stream_ptr())
        return
    call("b200_write_cache_kv_paged", ptr(qkv), ptr(key_cache), ptr(value_cache), ptr(block_tables), ptr(seq_lens), B, S, nh, kvh,
         d, bs, mb, qkv.stride(0), stream_ptr())


def decode_rope_append_paged(qkv, key_cache, value_cache, block_tables, cos, sin, seq_lens, nh, acc_f32=None, bias=None, *,
                             cache_k_scale=None, cache_v_scale=None):
    """RoPE on the new token's q, k + append k, v at position seq_lens[b] of sequence b's block list.  With acc_f32 the packed
    projection arrives as the fp32 split-K workspace (rounded here, workspace re-zeroed) and `qkv` is created."""
    nb, kvh, bs, d, mb = _paged_geom(key_cache, value_cache, block_tables)
    sc = _cache_scales(key_cache, "decode_rope_append_paged", cache_k_scale=cache_k_scale, cache_v_scale=cache_v_scale)
    if acc_f32 is not None:
        B = acc_f32.shape[0]
        qkv = torch.empty(B, (nh + 2 * kvh) * d, dtype=BF16, device=acc_f32.device)
    B = qkv.shape[0]
    if sc is not None:
        call("b200_decode_rope_append_paged_c8", ptr(qkv), ptr(acc_f32), ptr(bias), ptr(key_cache), ptr(value_cache),
             ptr(block_tables), ptr(sc[0]), ptr(sc[1]), ptr(cos), ptr(sin), ptr(seq_lens), B, nh, kvh, d, bs, mb, qkv.stride(0),
             stream_ptr())
        return qkv
    call("b200_decode_rope_append_paged", ptr(qkv), ptr(acc_f32), ptr(bias), ptr(key_cache), ptr(value_cache), ptr(block_tables),
         ptr(cos), ptr(sin), ptr(seq_lens), B, nh, kvh, d, bs, mb, qkv.stride(0), stream_ptr())
    return qkv


def decode_attention_paged(qkv, key_cache, value_cache, block_tables, seq_lens, nh, softmax_scale=None, out=None,
                           num_splits: int = 0, *, cache_k_out_scale=None, cache_v_out_scale=None):
    """decode_attention over the paged cache: sequence b's row t lives in page block_tables[b, t // block_size] (entries
    past a sequence's pages may be -1); it attends to min(seq_lens[b] + 1, max_blocks_per_seq * block_size) rows.
    d = 64 or 128, block_size 32, 64 or 128."""
    _chk(qkv, "qkv"); _chk(seq_lens, "seq_lens", torch.int32)
    nb, kvh, bs, d, mb = _paged_geom(key_cache, value_cache, block_tables)
    sc = _cache_scales(key_cache, "decode_attention_paged", cache_k_out_scale=cache_k_out_scale,
                       cache_v_out_scale=cache_v_out_scale)
    B = qkv.shape[0]
    if out is None:
        out = torch.empty(B, nh * d, dtype=BF16, device=qkv.device)
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    if num_splits <= 0:
        num_splits = _decode_splits(B, kvh, mb * bs)
    ws = None
    if num_splits > 1:
        ws = _workspace(_lib.load().b200_decode_attention_workspace_bytes(B, nh, num_splits), qkv.device, "decode_attn")
    if sc is not None:
        call("b200_decode_attention_paged_c8", ptr(qkv), ptr(key_cache), ptr(value_cache), ptr(block_tables), ptr(sc[0]),
             ptr(sc[1]), ptr(seq_lens), ptr(out), ptr(ws), B, nh, kvh, d, nb, bs, mb, qkv.stride(0), float(softmax_scale), num_splits,
             stream_ptr())
        return out
    call("b200_decode_attention_paged", ptr(qkv), ptr(key_cache), ptr(value_cache), ptr(block_tables), ptr(seq_lens), ptr(out),
         ptr(ws), B, nh, kvh, d, nb, bs, mb, qkv.stride(0), float(softmax_scale), num_splits, stream_ptr())
    return out


def fused_get_rotary_embedding(input_ids, position_ids, head_dim_shape_tensor, prompt_num: int = 0, theta: float = 10000.0,
                               use_neox: bool = True) -> torch.Tensor:
    """fused_get_rotary_embedding op of the reference (csrc/gpu/fused_get_rope.cu:159-223; same positional arguments):
    input_ids [bsz, seq] (only its shape is used), position_ids int64 [bsz, >= seq + prompt_num], head_dim_shape_tensor: any
    tensor whose FIRST dimension is head_dim (the reference's shape-carrier trick) or an int.
    Returns fp32 [2, bsz, 1, seq, head_dim] (cos, sin)."""
    _chk(position_ids, "position_ids", torch.int64)
    bsz, seq = input_ids.shape[0], input_ids.shape[1]
    head_dim = int(head_dim_shape_tensor) if isinstance(head_dim_shape_tensor, int) else int(head_dim_shape_tensor.shape[0])
    assert position_ids.dim() == 2 and position_ids.is_contiguous() and position_ids.shape[0] == bsz
    out = torch.empty(2, bsz, 1, seq, head_dim, dtype=torch.float32, device=position_ids.device)
    call("b200_fused_get_rotary_embedding", ptr(position_ids), ptr(out), bsz, seq, position_ids.shape[1], head_dim,
         int(prompt_num), float(theta), 1 if use_neox else 0, stream_ptr())
    return out


def append_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q,
                     block_tables, cos, sin, nh: int, max_q_len: int, softmax_scale=None, out=None, num_splits: int = 0, *,
                     cache_k_scale=None, cache_v_scale=None, cache_k_out_scale=None, cache_v_out_scale=None):
    """append_attention of the reference (csrc/gpu/append_attention.cu:428-851) for a mixed batch over the paged cache: RoPE +
    cache append for every new token row of the packed projection qkv [token_num, (nh + 2 kvh) d] (modified in place), then
    attention of every row over its sequence's pages — prompts / prompt chunks and decode rows in one call.
    Returns out [token_num, nh * d]."""
    _chk(qkv, "qkv"); _chk(cos, "cos", torch.float32); _chk(sin, "sin", torch.float32)
    for name, t in (("seq_lens_encoder", seq_lens_encoder), ("seq_lens_decoder", seq_lens_decoder),
                    ("seq_lens_this_time", seq_lens_this_time), ("cu_seqlens_q", cu_seqlens_q)):
        _chk(t, name, torch.int32)
        assert t.is_contiguous()
    nb, kvh, bs, d, mb = _paged_geom(key_cache, value_cache, block_tables)
    sc = _cache_scales(key_cache, "append_attention", cache_k_scale=cache_k_scale, cache_v_scale=cache_v_scale,
                       cache_k_out_scale=cache_k_out_scale, cache_v_out_scale=cache_v_out_scale)
    token_num, ld = qkv.shape
    B = seq_lens_this_time.numel()
    assert qkv.stride(1) == 1 and ld == (nh + 2 * kvh) * d and block_tables.shape[0] == B and cu_seqlens_q.numel() >= B
    if out is None:
        out = torch.empty(token_num, nh * d, dtype=BF16, device=qkv.device)
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(d)
    if num_splits <= 0:
        num_splits = _decode_splits(B, kvh, mb * bs)
    ws = _workspace(_lib.load().b200_append_attention_workspace_bytes(B, nh, kvh, d, num_splits), qkv.device, "append_attn")
    if sc is not None:
        call("b200_append_attention_c8", ptr(qkv), ptr(key_cache), ptr(value_cache), *[ptr(t) for t in sc], ptr(seq_lens_encoder),
             ptr(seq_lens_decoder), ptr(seq_lens_this_time), ptr(cu_seqlens_q), ptr(block_tables), ptr(cos), ptr(sin), ptr(out),
             ptr(ws), B, token_num, int(max_q_len), nh, kvh, d, nb, bs, mb, cos.shape[0], qkv.stride(0), out.stride(0),
             float(softmax_scale), num_splits, stream_ptr())
        return out
    call("b200_append_attention", ptr(qkv), ptr(key_cache), ptr(value_cache), ptr(seq_lens_encoder), ptr(seq_lens_decoder),
         ptr(seq_lens_this_time), ptr(cu_seqlens_q), ptr(block_tables), ptr(cos), ptr(sin), ptr(out), ptr(ws), B, token_num,
         int(max_q_len), nh, kvh, d, nb, bs, mb, cos.shape[0], qkv.stride(0), out.stride(0), float(softmax_scale), num_splits,
         stream_ptr())
    return out


def get_padding_offset(input_ids, cum_offsets, token_num, seq_lens):
    """get_padding_offset_v2: returns (x_remove_padding, cum_offsets_out, padding_offset, cu_seqlens_q, cu_seqlens_k)."""
    bsz, max_len = input_ids.shape
    dev = input_ids.device
    xr = torch.zeros(int(token_num), dtype=torch.int64, device=dev)
    po = torch.zeros(int(token_num), dtype=torch.int32, device=dev)
    co = torch.zeros(bsz, dtype=torch.int32, device=dev)
    cq = torch.zeros(bsz + 1, dtype=torch.int32, device=dev)
    ck = torch.zeros(bsz + 1, dtype=torch.int32, device=dev)
    call("b200_get_padding_offset", ptr(input_ids), ptr(cum_offsets), ptr(seq_lens), ptr(xr), ptr(po), ptr(co), ptr(cq), ptr(ck),
         bsz, max_len, stream_ptr())
    return xr, co, po, cq, ck


def rebuild_padding(tmp_out, cum_offsets, seq_lens_decoder, seq_lens_encoder, max_len):
    _chk(tmp_out, "tmp_out")
    bsz, dim = seq_lens_encoder.numel(), tmp_out.shape[1]
    out = torch.zeros(bsz, dim, dtype=BF16, device=tmp_out.device)
    call("b200_rebuild_padding", ptr(tmp_out), ptr(cum_offsets), ptr(seq_lens_decoder), ptr(seq_lens_encoder), ptr(out), bsz,
         max_len, dim, stream_ptr())
    return out


def set_value_by_flags_and_idx(pre_ids_all, pre_ids_now, step_idx, stop_flags):
    bs, length = pre_ids_all.shape
    call("b200_set_value_by_flags_and_idx", ptr(stop_flags), ptr(pre_ids_all), ptr(pre_ids_now), ptr(step_idx), bs, length,
         stream_ptr())


def set_value_by_flags_and_idx_v2(pre_ids_all, input_ids, seq_lens_this_time, seq_lens_encoder, seq_lens_decoder, step_idx,
                                  stop_flags):
    bs, length = pre_ids_all.shape
    call("b200_set_value_by_flags_and_idx_v2", ptr(stop_flags), ptr(pre_ids_all), ptr(input_ids), ptr(seq_lens_encoder),
         ptr(seq_lens_decoder), ptr(step_idx), bs, length, input_ids.shape[1], stream_ptr())


def token_penalty_multi_scores(pre_ids, logits, penalty_scores, frequency_scores, presence_scores, temperatures, bad_tokens,
                               cur_len, min_len, eos_token_id):
    """In place on fp32 logits (get_token_penalty_multi_scores_v2; pass temperatures/bad_tokens=None for the v1 op)."""
    _chk(logits, "logits", torch.float32)
    bs, length = logits.shape
    ws = _workspace(bs * length * 4, logits.device, "penalty")
    call("b200_token_penalty_multi_scores", ptr(pre_ids), ptr(logits), ptr(penalty_scores), ptr(frequency_scores),
         ptr(presence_scores), ptr(temperatures), ptr(bad_tokens), ptr(cur_len), ptr(min_len), ptr(eos_token_id), ptr(ws), bs,
         length, pre_ids.shape[1], 0 if bad_tokens is None else bad_tokens.numel(), eos_token_id.numel(), stream_ptr())
    return logits


def set_stop_value_multi_ends(topk_ids, stop_flags, end_ids, seq_lens=None, next_tokens=None):
    """v2 when seq_lens / next_tokens are given, else the v1 op in mode 2.  In place."""
    v2 = seq_lens is not None
    call("b200_set_stop_value_multi_ends", ptr(stop_flags), ptr(topk_ids), ptr(next_tokens), ptr(end_ids), ptr(seq_lens),
         topk_ids.numel(), end_ids.numel(), 1 if v2 else 0, stream_ptr())


def update_inputs(stop_flags, not_need_stop, seq_lens_this_time, seq_lens_encoder, seq_lens_decoder, input_ids, stop_nums,
                  next_tokens, is_block_step):
    call("b200_update_inputs", ptr(not_need_stop), ptr(seq_lens_this_time), ptr(seq_lens_encoder), ptr(seq_lens_decoder),
         ptr(input_ids), ptr(stop_nums), ptr(stop_flags), ptr(is_block_step), ptr(next_tokens), seq_lens_this_time.numel(),
         stop_flags.numel(), input_ids.shape[1], stream_ptr())


def step_paddle(stop_flags, seq_lens_this_time, ori_seq_lens_encoder, seq_lens_encoder, seq_lens_decoder, block_tables,
                encoder_block_lens, is_block_step, step_block_list, step_lens, recover_block_list, recover_lens, need_block_list,
                need_block_len, used_list_len, free_list, free_list_len, input_ids, pre_ids, step_idx, next_tokens, block_size: int,
                encoder_decoder_block_num: int = 0, first_token_id: int = 0):
    """step_paddle(...) of the reference (csrc/gpu/step.cu:216-283; same argument order and in-place semantics)."""
    for name, t, dt in (("stop_flags", stop_flags, torch.bool), ("is_block_step", is_block_step, torch.bool),
                        ("seq_lens_this_time", seq_lens_this_time, torch.int32), ("block_tables", block_tables, torch.int32),
                        ("free_list", free_list, torch.int32), ("input_ids", input_ids, torch.int64), ("pre_ids", pre_ids, torch.int64),
                        ("step_idx", step_idx, torch.int64), ("next_tokens", next_tokens, torch.int64)):
        _chk(t, name, dt)
        assert t.is_contiguous(), name
    bsz = seq_lens_this_time.shape[0]
    call("b200_step_paddle", ptr(stop_flags), ptr(seq_lens_this_time), ptr(ori_seq_lens_encoder), ptr(seq_lens_encoder),
         ptr(seq_lens_decoder), ptr(block_tables), ptr(encoder_block_lens), ptr(is_block_step), ptr(step_block_list), ptr(step_lens),
         ptr(recover_block_list), ptr(recover_lens), ptr(need_block_list), ptr(need_block_len), ptr(used_list_len), ptr(free_list),
         ptr(free_list_len), ptr(input_ids), ptr(pre_ids), ptr(step_idx), ptr(next_tokens), bsz, int(block_size),
         block_tables.shape[1], input_ids.shape[1], pre_ids.shape[1], int(first_token_id), stream_ptr())


RETIRE_ADMIT_ORDER = ("stop_flags", "is_block_step", "seq_lens_this_time", "seq_lens_encoder", "ori_seq_lens_encoder",
                      "seq_lens_decoder", "step_idx", "pre_ids", "next_tokens", "input_ids", "block_tables", "encoder_block_lens",
                      "used_list_len", "free_list", "free_list_len", "step_lens", "max_dec_len", "min_dec_len", "slot_request",
                      "prompt_ids", "prompt_offsets", "req_max_dec_len", "req_min_dec_len", "cursor", "out_ids", "out_lens")
# int32 words of the step header retire_admit writes (enum B200_RA_* of include/b200nlp.h)
RA_TOKEN_NUM, RA_MAX_Q_LEN, RA_RUNNING, RA_PENDING, RA_PARKED, RA_DONE, RA_FREE_BLOCKS, RA_PREEMPTIONS, RA_RECOVERIES, \
    RA_ADMITTED, RA_RETIRED = range(11)
RA_HEADER_INTS = 16


def retire_admit(st: dict, header: torch.Tensor, block_size: int, max_prompt_len: int, max_seq_len: int):
    """Retire the finished slots and admit queued requests (b200_retire_admit; call right after step_paddle).  `st` maps every
    name of RETIRE_ADMIT_ORDER to its device tensor (updated in place); `header` is a pinned int32 [RA_HEADER_INTS] host tensor.
    max_prompt_len / max_seq_len: the queue's longest prompt and prompt + max_dec_len."""
    dtypes = {"stop_flags": torch.bool, "is_block_step": torch.bool, "step_idx": torch.int64, "pre_ids": torch.int64,
              "next_tokens": torch.int64, "input_ids": torch.int64, "max_dec_len": torch.int64, "min_dec_len": torch.int64,
              "prompt_ids": torch.int64, "req_max_dec_len": torch.int64, "req_min_dec_len": torch.int64, "out_ids": torch.int64}
    for name in RETIRE_ADMIT_ORDER:
        _chk(st[name], name, dtypes.get(name, torch.int32))
        assert st[name].is_contiguous(), name
    assert header.dtype == torch.int32 and header.is_pinned() and header.numel() >= RA_HEADER_INTS
    call("b200_retire_admit", *[ptr(st[k]) for k in RETIRE_ADMIT_ORDER], ptr(header), st["seq_lens_this_time"].numel(),
         int(block_size), st["block_tables"].shape[1], st["input_ids"].shape[1], st["pre_ids"].shape[1],
         st["req_max_dec_len"].numel(), st["out_ids"].shape[1], int(max_prompt_len), int(max_seq_len), stream_ptr())


def generate_step_update(next_tokens, stop_flags, step_idx, max_dec_len, seq_len_decoder, pre_ids, eos_ids, out_tokens,
                         stop_count, out_col=0, out_col_dev=None):
    bs = next_tokens.numel()
    call("b200_generate_step_update", ptr(next_tokens), ptr(stop_flags), ptr(step_idx), ptr(max_dec_len), ptr(seq_len_decoder),
         ptr(pre_ids), pre_ids.shape[1], ptr(eos_ids), eos_ids.numel(), ptr(out_tokens),
         0 if out_tokens is None else out_tokens.shape[1], int(out_col), ptr(out_col_dev), ptr(stop_count), bs, stream_ptr())


def softmax_f32_(logits):
    """In-place fp32 row softmax (generation_utils.py:327)."""
    _chk(logits, "logits", torch.float32)
    rows, V = logits.shape
    assert logits.stride(1) == 1
    call("b200_softmax_f32", ptr(logits), rows, V, logits.stride(0), stream_ptr())
    return logits


def top_p_sampling_reject(probs, top_p, uniform=None, seed: int = 0, max_rounds: int = 32, generator=None):
    """top_p_sampling_reject(probs, top_p, seed) of the reference (csrc/gpu/sample_kernels/top_p_sampling_reject.cu).
    probs [bs, V] fp32, top_p [bs] fp32 -> ids [bs] int64.  `uniform` [max_rounds, bs] may be supplied (tests); otherwise it
    is drawn from `generator` (or a fresh generator seeded with `seed` when seed != 0, else torch's default CUDA generator)."""
    _chk(probs, "probs", torch.float32); _chk(top_p, "top_p", torch.float32)
    bs, V = probs.shape
    assert probs.stride(1) == 1 and top_p.numel() == bs
    if uniform is None:
        if generator is None and seed:
            generator = torch.Generator(device=probs.device)
            generator.manual_seed(int(seed))
        uniform = torch.rand(max_rounds, bs, dtype=torch.float32, device=probs.device, generator=generator)
    _chk(uniform, "uniform", torch.float32)
    assert uniform.is_contiguous() and uniform.shape == (max_rounds, bs)
    out = torch.empty(bs, dtype=torch.int64, device=probs.device)
    call("b200_top_p_sampling_reject", ptr(probs), ptr(top_p), ptr(uniform), ptr(out), bs, V, probs.stride(0), max_rounds,
         stream_ptr())
    return out


def argmax_f32(logits):
    _chk(logits, "logits", torch.float32)
    rows, V = logits.shape
    out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    call("b200_argmax_f32", ptr(logits), ptr(out), rows, V, logits.stride(0), stream_ptr())
    return out


def bf16_rows_to_f32(src, out=None):
    _chk(src, "src")
    rows, cols = src.shape
    if out is None:
        out = torch.empty(rows, cols, dtype=torch.float32, device=src.device)
    call("b200_bf16_rows_to_f32", ptr(src), ptr(out), rows, cols, src.stride(0), stream_ptr())
    return out
