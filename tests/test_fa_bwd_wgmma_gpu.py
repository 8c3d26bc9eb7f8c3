"""The wgmma attention backward (b200_set_fa_bwd_impl(2)) against the mma.sync kernel (impl 1) and the fp32 oracle.

Shapes cover the two benchmarked layouts (plain causal and packed documents whose boundaries fall on and off the 64- and
128-row tile grids), sequence lengths at the edges of the 64-row q tiles, the 128-row kv tiles and the two-stage ring, batch
rows that must not read into each other, GQA ratios 1, 3 and 6, and gradients written into strided views of a larger buffer.
"""
import pytest
import torch

from oracle import llama_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
D = 128


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


def backward(impl, q, k, v, out, dout, lse, ms, pad):
    """Run one backward generation; dq/dk/dv are views into NaN-filled buffers `pad` columns wider than the gradient."""
    from paddlenlp_b200 import _lib, ops

    lib = _lib.load()
    B, S, nh, _ = q.shape
    kvh = k.shape[2]
    bufs = [torch.full((B, S, h * D + pad), float("nan"), dtype=torch.bfloat16, device=DEV) for h in (nh, kvh, kvh)]
    views = [b[:, :, pad // 2: pad // 2 + h * D].view(B, S, h, D) for b, h in zip(bufs, (nh, kvh, kvh))]
    old = lib.b200_set_fa_bwd_impl(impl)
    try:
        ops.flash_attn_bwd(q, k, v, out, dout, lse, *views, mask_start=ms)
    finally:
        lib.b200_set_fa_bwd_impl(old)
    torch.cuda.synchronize()
    for b, vw in zip(bufs, views):
        assert torch.isfinite(vw.float()).all()
        assert torch.isnan(b[:, :, : pad // 2].float()).all() and torch.isnan(b[:, :, pad // 2 + vw.shape[2] * D:].float()).all()
    return views


CASES = [
    # B, S, nh, kvh, documents per batch row (None: plain causal)
    (1, 4096, 24, 8, None),
    (4, 2048, 12, 2, None),
    (1, 4096, 24, 8, [[1000, 64, 128, 2904]]),
    (4, 2048, 12, 2, [[1, 511, 1024, 512], [2048], [64, 65, 1919], [700, 900, 448]]),
    (1, 1, 1, 1, None),
    (1, 63, 3, 1, None),
    (1, 64, 2, 2, None),
    (1, 65, 6, 1, None),
    (3, 127, 3, 1, None),
    (3, 129, 6, 1, [[1, 128], [64, 65], [129]]),
    (1, 4095, 6, 2, None),
]


@pytest.mark.parametrize("B,S,nh,kvh,docs", CASES)
def test_fa_bwd_wgmma(B, S, nh, kvh, docs):
    from paddlenlp_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(S * 131 + nh)
    q = torch.randn(B, S, nh, D, device=DEV, generator=g).bfloat16()
    k = torch.randn(B, S, kvh, D, device=DEV, generator=g).bfloat16()
    v = torch.randn(B, S, kvh, D, device=DEV, generator=g).bfloat16()
    ms = None if docs is None else torch.stack([doc_mask(dl, S) for dl in docs]).to(DEV)
    out, lse = ops.flash_attn_fwd(q, k, v, mask_start=ms)
    dout = torch.randn(B, S, nh, D, device=DEV, generator=g).bfloat16()
    new = backward(2, q, k, v, out, dout, lse, ms, pad=256)
    old = backward(1, q, k, v, out, dout, lse, ms, pad=0)
    for name, a, b in zip(("dq", "dk", "dv"), new, old):
        if name == "dv" or S > 1:   # one row: dS = dP - rowsum(dO o O) = 0 up to rounding, so dq = dk = 0
            assert relerr(a, b) < 1e-3, (name, relerr(a, b))   # same rounding points: summation-order noise (~2e-5)
    for b in range(B):
        qf, kf, vf = (t[b:b + 1].float().detach().requires_grad_(True) for t in (q, k, v))
        ref = R.attention(qf, kf, vf, "fp32", mask_start=None if ms is None else ms[b:b + 1].cpu())
        ref.backward(dout[b:b + 1].float().reshape(1, S, -1))
        for name, a, r, tile in (("dq", new[0], qf.grad, 64), ("dk", new[1], kf.grad, 128), ("dv", new[2], vf.grad, 128)):
            if name != "dv" and S == 1:
                continue
            assert relerr(a[b:b + 1], r) < 2e-2, (name, b, relerr(a[b:b + 1], r))
            e = worst_tile_relerr(a[b], r[0], tile)
            assert e < 1e-2, (name, b, e)
        del ref, qf, kf, vf
