"""The wgmma attention forward (b200_set_fa_fwd_impl(2)) against the mma.sync kernel (impl 1) and an fp32 oracle on the device.

Shapes cover the two benchmarked layouts at head_dim 128 and Llama-3.2-1B at head_dim 64, sequence lengths at the edges of
the 64-row warpgroup halves, the 128-row q and kv tiles and the two-stage ring, GQA groups 1 to 8, batch rows that must not
read into each other (each row against its own oracle), packed documents on and off the 128-row grid, one-token documents,
left-padding start rows and a softmax scale other than 1/sqrt(d).  q / k / v are views of a packed QKV projection and the
output a strided view into a NaN-filled wider buffer whose padding must stay NaN.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BF16 = torch.bfloat16


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def worst_tile_relerr(a, r, tile):
    """Largest relative error over blocks of `tile` sequence rows of one head; a, r [S, heads, d]."""
    a, r = a.float(), r.float()
    S, H = a.shape[0], a.shape[1]
    idx = torch.arange(S, device=a.device) // tile
    nt = (S + tile - 1) // tile
    e2 = torch.zeros(nt, H, device=a.device).index_add_(0, idx, (a - r).pow(2).sum(-1))
    r2 = torch.zeros(nt, H, device=a.device).index_add_(0, idx, r.pow(2).sum(-1))
    return (e2 / r2.clamp_min(1e-30)).sqrt().max().item()


def doc_mask(doc_lens, S):
    ms = torch.empty(S, dtype=torch.int32)
    pos = 0
    for n in doc_lens:
        ms[pos:pos + n] = pos + n
        pos += n
    assert pos == S
    return ms


def pad_mask(pad, S):
    """Left padding in start-row form: a padding column is a one-token document (start = c + 1), real columns keep S."""
    ms = torch.full((S,), S, dtype=torch.int32)
    ms[:pad] = torch.arange(1, pad + 1, dtype=torch.int32)
    return ms


def oracle(q, k, v, scale, ms):
    """fp32 attention of one batch row: q [S, nh, d], k / v [S, kvh, d], ms [S] or None -> (out [S, nh, d], lse [nh, S])."""
    S, nh, d = q.shape
    rep = nh // k.shape[1]
    qf = q.float().transpose(0, 1)
    kf = k.float().repeat_interleave(rep, dim=1).transpose(0, 1)
    vf = v.float().repeat_interleave(rep, dim=1).transpose(0, 1)
    scores = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    rows = torch.arange(S, device=q.device)
    hidden = rows[None, :] > rows[:, None]                       # [row, col]: causal
    if ms is not None:
        hidden = hidden | (rows[:, None] >= ms.to(q.device)[None, :])
    scores.masked_fill_(hidden[None], float("-inf"))
    lse = torch.logsumexp(scores, dim=-1)
    out = torch.matmul(torch.softmax(scores, dim=-1), vf).transpose(0, 1)
    return out, lse


def forward(impl, q, k, v, scale, ms, pad):
    """One forward of kernel `impl`; out is a view into a NaN-filled buffer `pad` columns wider than the output."""
    from paddlenlp_b200 import _lib, ops

    lib = _lib.load()
    B, S, nh, d = q.shape
    buf = torch.full((B, S, nh * d + pad), float("nan"), dtype=BF16, device=DEV)
    out = buf[:, :, pad // 2: pad // 2 + nh * d].view(B, S, nh, d)
    old = lib.b200_set_fa_fwd_impl(impl)
    try:
        _, lse = ops.flash_attn_fwd(q, k, v, scale, out=out, mask_start=ms)
    finally:
        lib.b200_set_fa_fwd_impl(old)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert torch.isnan(buf[:, :, : pad // 2].float()).all() and torch.isnan(buf[:, :, pad // 2 + nh * d:].float()).all()
    return out, lse


CASES = [
    # B, S, nh, kvh, d, mask per batch row: None (plain causal), a list of document lengths, or ("pad", left padding)
    (1, 4096, 24, 8, 128, None),                                          # Llama-3.2-3B pre-training
    (4, 2048, 12, 2, 128, None),                                          # Qwen2-1.5B SFT micro-batch
    (1, 4096, 32, 8, 64, None),                                           # Llama-3.2-1B
    (1, 1, 1, 1, 128, None),                                              # S at the tile and ring edges, GQA groups 1 to 8
    (1, 63, 3, 1, 128, None),
    (1, 64, 4, 2, 64, None),
    (1, 65, 6, 1, 128, None),
    (2, 127, 7, 1, 64, None),
    (1, 128, 4, 4, 128, None),
    (3, 129, 8, 2, 128, None),
    (1, 255, 8, 1, 64, None),
    (2, 256, 5, 1, 128, None),
    (1, 257, 3, 3, 64, None),
    (3, 1000, 8, 1, 128, None),
    (1, 4096, 24, 8, 128, [[1000, 64, 128, 2904]]),                       # documents on and off the 128-row grid
    (4, 2048, 12, 2, 128, [[1, 511, 1024, 512], [2048], [64, 65, 1919], [700, 900, 448]]),
    (3, 129, 6, 2, 64, [[1, 128], [64, 65], [129]]),
    (2, 384, 4, 2, 128, [[1, 1, 1, 125, 128, 1, 127], [256, 1, 127]]),   # one-token documents
    (3, 700, 4, 1, 128, [("pad", 129), ("pad", 0), ("pad", 511)]),        # left padding
    (2, 384, 8, 4, 64, [("pad", 300), ("pad", 1)]),
]


def build_mask(spec, S):
    if spec is None:
        return None
    rows = [pad_mask(m[1], S) if isinstance(m, tuple) else doc_mask(m, S) for m in spec]
    return torch.stack(rows).to(DEV)


def check(B, S, nh, kvh, d, spec, scale):
    g = torch.Generator(device=DEV).manual_seed(S * 131 + nh * 7 + d)
    qkv = torch.randn(B, S, (nh + 2 * kvh) * d, device=DEV, generator=g).to(BF16)
    q = qkv[..., :nh * d].unflatten(-1, (nh, d))
    k = qkv[..., nh * d:(nh + kvh) * d].unflatten(-1, (kvh, d))
    v = qkv[..., (nh + kvh) * d:].unflatten(-1, (kvh, d))
    ms = build_mask(spec, S)
    sc = 1.0 / math.sqrt(d) if scale is None else scale
    out, lse = forward(2, q, k, v, scale, ms, pad=256)
    out1, lse1 = forward(1, q, k, v, scale, ms, pad=0)
    # same rounding points: P's bf16 rounding (the kv tiles, and so the running maxima, differ at d = 128) and summation order
    assert relerr(out, out1) < (1e-3 if d == 64 else 5e-3), relerr(out, out1)
    assert (lse - lse1).abs().max().item() < 1e-4
    again, lse_again = forward(2, q, k, v, scale, ms, pad=0)
    assert torch.equal(again, out) and torch.equal(lse_again, lse)    # deterministic
    worst = 0.0
    for b in range(B):
        ref, lse_ref = oracle(q[b], k[b], v[b], sc, None if ms is None else ms[b])
        assert relerr(out[b], ref) < 2e-2, (b, relerr(out[b], ref))
        e = worst_tile_relerr(out[b], ref, 128)
        worst = max(worst, e)
        assert e < 1e-2, (b, e)
        assert (lse[b] - lse_ref).abs().max().item() < 2e-3, b
        del ref, lse_ref
    return worst


@pytest.mark.parametrize("B,S,nh,kvh,d,spec", CASES)
def test_fa_fwd_wgmma(B, S, nh, kvh, d, spec):
    worst = check(B, S, nh, kvh, d, spec, None)
    print(f"[fa fwd {B}x{S}x{nh}/{kvh} d{d}] worst tile rel err {worst:.2e}")


@pytest.mark.parametrize("B,S,nh,kvh,d,spec,scale", [(2, 1000, 6, 2, 128, None, 0.25), (1, 700, 8, 2, 64, [[300, 400]], 0.05)])
def test_fa_fwd_wgmma_softmax_scale(B, S, nh, kvh, d, spec, scale):
    check(B, S, nh, kvh, d, spec, scale)
