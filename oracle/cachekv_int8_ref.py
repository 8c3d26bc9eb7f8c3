"""Restatement of the static int8 KV cache (cachekv_int8_type="static") in plain torch: quantise, dequantise, the scales of
the reference's cachekv_scales.json (CacheScaleLoader, experimental/model_utils.py:433-468), calibration, and attention over
the dequantised pages in fp64.

    u = clamp(rne(bf16(s * x)), -127, 127) + 128      (uint8; x the post-RoPE bf16 value, s the bf16 quantise scale)
    x_hat = (u - 128) * o                              (o = bf16(1 / s_fp64), the bf16 dequantise scale)

The reference rounds x_hat to bf16 before its attention matmuls; the kernels here do not (the scale is applied once per kv
head), and neither does this restatement.  Its encoder-side write stores + 127 where the decoder side and the dequantise use
128 (encoder_write_cache_with_rope_impl.cuh:839); here every row uses + 128.
"""
from __future__ import annotations

import math

import torch

BF16 = torch.bfloat16


def quantize(x: torch.Tensor, s) -> torch.Tensor:
    """x bf16 [..., kvh, d] (or any shape broadcasting with s), s bf16 scales -> uint8.  The product of two bf16 values is
    exact in fp32, so bf16(s * x) is one rounding of the exact product; torch.round rounds half to even."""
    s = torch.as_tensor(s, dtype=BF16)
    p = (x.to(BF16).float() * s.float()).to(BF16).float()
    return (torch.round(p).clamp(-127, 127) + 128).to(torch.uint8)


def dequantize(u: torch.Tensor, o) -> torch.Tensor:
    """uint8 cache bytes -> fp64 (u - 128) * o."""
    return (u.to(torch.float64) - 128.0) * torch.as_tensor(o, dtype=BF16).double()


def fake_quant(x: torch.Tensor, s, o) -> torch.Tensor:
    """dequantize(quantize(x, s), o) in x's float dtype: the value a kernel reads back for the bf16 value x it cached.  (u - 128) o
    is an integer of at most 8 bits times a bf16 scale, exact in fp32."""
    return dequantize(quantize(x, s), o).to(x.dtype)


def scales_from_absmax(absmax):
    """absmax [..., kvh] -> (s, o) bf16: s = 127 / absmax and o = 1 / s in fp64, each cast to bf16."""
    a = torch.as_tensor(absmax, dtype=torch.float64)
    if not bool(torch.isfinite(a).all()) or not bool((a > 0).all()):
        raise ValueError("absmax must be finite and positive")
    s = 127.0 / a
    return s.to(BF16), (1.0 / s).to(BF16)


def absmax_from_json(scales: dict, prefix: str, num_layers: int, num_heads: int, num_kv_heads: int):
    """cachekv_scales.json content -> (k absmax, v absmax) fp64 [L, kvh]: under GQA every group-th of the num_heads values."""
    group = num_heads // num_kv_heads
    out = []
    for kind in ("k", "v"):
        rows = []
        for i in range(num_layers):
            vals = scales[f"{prefix}.layers.{i}.self_attn.cache{kind}_matmul.activation_quanter"]
            rows.append([float(vals[j]) for j in range(0, num_heads, group)])
        out.append(torch.tensor(rows, dtype=torch.float64))
    return out[0], out[1]


def absmax_of_cache(cache: torch.Tensor) -> torch.Tensor:
    """Calibration: absmax per kv head of a bf16 paged cache [num_blocks, kvh, block_size, d] (zero pages do not move it)."""
    return cache.double().abs().amax(dim=(0, 2, 3))


def gather_pages(cache: torch.Tensor, table_row: torch.Tensor, length: int) -> torch.Tensor:
    """Rows 0 .. length-1 of one sequence from a paged cache [num_blocks, kvh, bs, d] -> [kvh, length, d]."""
    bs = cache.shape[2]
    pages = [int(table_row[j]) for j in range((length + bs - 1) // bs)]
    rows = torch.cat([cache[p] for p in pages], dim=1) if pages else cache[:0, :, :0].reshape(cache.shape[1], 0, cache.shape[3])
    return rows[:, :length]


def attention_fp64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q_pos, scale: float | None = None) -> torch.Tensor:
    """q [n, nh, d], k / v [kvh, L, d] (fp64, dequantised), q_pos [n] absolute positions: row i attends to cache rows
    0 .. q_pos[i] -> [n, nh, d] fp64."""
    n, nh, d = q.shape
    kvh = k.shape[0]
    g = nh // kvh
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    kk = k.repeat_interleave(g, dim=0)                 # [nh, L, d]
    vv = v.repeat_interleave(g, dim=0)
    s = torch.einsum("nhd,hld->nhl", q.double(), kk) * scale
    pos = torch.as_tensor(q_pos, dtype=torch.int64).view(n, 1, 1)
    cols = torch.arange(k.shape[1]).view(1, 1, -1)
    s = s.masked_fill(cols > pos, float("-inf"))
    return torch.einsum("nhl,hld->nhd", torch.softmax(s, dim=-1), vv)
