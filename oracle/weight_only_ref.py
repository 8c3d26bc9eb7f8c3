"""Restatement of weight-only int8 quantisation (weight_quantize(..., algo="weight_only_int8") / weight_only_linear(...,
weight_dtype="int8"), experimental/transformers/llama/modeling.py:971-1052 and fused_transformer_layers.py:1221-1440).

Paddle core implements these ops and their source is not in the reference tree; the arithmetic is stated here instead:
    a[n]     = max_k |W[k, n]|                                   (fp32, exact)
    scale[n] = bf16_rn(a[n] / 127.0f)                            (IEEE fp32 division)
    q[k, n]  = clamp(rint(W[k, n] / float(scale[n])), -127, 127) (IEEE fp32 division, half to even); scale 0 -> q = 0
    y[m, n]  = scale[n] * sum_k x[m, k] q[k, n] (+ bias[n])
Plain torch on the CPU; no project code is imported.
"""
from __future__ import annotations

import torch


def quantize(w: torch.Tensor):
    """w [K, N] (bf16 or fp32 values) -> (q int8 [K, N], scale bf16 [N])."""
    wf = w.float()
    a = wf.abs().amax(dim=0)
    scale = (a / torch.tensor(127.0, dtype=torch.float32)).to(torch.bfloat16)
    s = scale.float()
    safe = torch.where(s == 0, torch.ones_like(s), s)
    q = torch.round(wf / safe)                 # torch.round: half to even
    q = q.clamp(-127, 127)
    q = torch.where(s == 0, torch.zeros_like(q), q)
    return q.to(torch.int8), scale


def pack(q: torch.Tensor) -> torch.Tensor:
    """q int8 [K, N] -> the kernel's packed layout as int8 [N, K] (include/b200nlp.h): 128-byte units (g, s) for channels
    8g .. 8g+7 and k 16s .. 16s+15 at byte (g K/16 + s) 128; lane l's bytes q[16s+c][n], q[16s+c+1][n], q[16s+c+8][n],
    q[16s+c+9][n] with n = 8g + l/4, c = 2 (l % 4)."""
    K, N = q.shape
    assert K % 16 == 0 and N % 8 == 0
    t = q.t().reshape(N // 8, 8, K // 16, 16)                  # [g, row, s, k16]
    t = t.permute(0, 2, 1, 3)                                  # [g, s, row, k16]
    c = torch.arange(4) * 2                                    # lane % 4 -> c
    idx = torch.stack([c, c + 1, c + 8, c + 9], dim=1)         # [4 (lane % 4), 4 bytes]
    u = t[:, :, :, idx]                                        # [g, s, row (= lane / 4), lane % 4, 4 bytes]
    return u.reshape(N, K).contiguous()


def linear_f64(x: torch.Tensor, q: torch.Tensor, scale: torch.Tensor, bias=None) -> torch.Tensor:
    """fp64 y = scale * (x @ q) (+ bias)."""
    y = (x.double() @ q.double()) * scale.double()
    if bias is not None:
        y = y + bias.double()
    return y


def error_allowance(x: torch.Tensor, q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """scale * (|x| @ |q|): the magnitude the fp32 sums' rounding error is measured against."""
    return (x.double().abs() @ q.double().abs()) * scale.double()
