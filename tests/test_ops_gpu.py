"""GPU parity tests of every kernel behind the C-ABI against the oracle (oracle/llama_ref.py, oracle/optim_ref.py).

All calls go through paddlenlp_b200.ops -> ctypes -> libb200nlp.so.  Tolerances are written beside each check:
bf16 outputs are compared with a normalised error  max|a-b| / max|b|  and  ||a-b|| / ||b||.
"""
import math

import pytest
import torch

from oracle import llama_ref as R
from oracle import optim_ref

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BF16 = torch.bfloat16


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def maxerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def rand_bf16(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF16)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [520, 40])    # two-warpgroup (128-row) and one-warpgroup (64-row) tiles
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_layouts(M, ta, tb):
    o = ops()
    N, K = 776, 328           # ragged against every tile dimension
    A = rand_bf16(M, K, seed=1, scale=0.5)
    B = rand_bf16(K, N, seed=2, scale=0.5)
    a_d = (A.t().contiguous() if ta else A).to(DEV)
    b_d = (B.t().contiguous() if tb else B).to(DEV)
    out = o.gemm(a_d, b_d, trans_a=ta, trans_b=tb)
    ref = A.float().to(DEV) @ B.float().to(DEV)
    # one bf16 rounding of an fp32-accumulated result: <= 2^-8 relative to the largest magnitude
    assert maxerr(out, ref) < 2 ** -7
    assert relerr(out, ref) < 4e-3


def test_gemm_accumulate_bias_and_views():
    o = ops()
    M, N, K = 384, 512, 256
    A = rand_bf16(M, K, seed=3).to(DEV)
    Wfull = rand_bf16(K, N + 256, seed=4).to(DEV)
    W = Wfull[:, 128:128 + N]                      # column slice: ldb != N
    C0 = rand_bf16(M, N, seed=5).to(DEV)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(6)).to(DEV)
    C = C0.clone()
    o.gemm(A, W, out=C, accumulate=True, bias=bias)
    ref = A.float() @ W.float() + bias + C0.float()
    assert maxerr(C, ref) < 2 ** -7


def test_gemm_residual_epilogue():
    o = ops()
    M, N, K = 304, 520, 192
    A = rand_bf16(M, K, seed=30).to(DEV)
    W = rand_bf16(K, N, seed=31).to(DEV)
    Rs = rand_bf16(M, N, seed=32, scale=4.0).to(DEV)
    out = o.gemm(A, W, residual=Rs)
    lin = (A.float() @ W.float()).to(BF16).float()            # Linear output rounding ...
    ref = (lin + Rs.float()).to(BF16).float()                  # ... then the residual-add rounding
    mism = (out.float() != ref).float().mean().item()
    assert mism < 0.02 and maxerr(out, ref) < 2 ** -7           # only fp32 accumulation-order ties may differ


# (5 | 33 | 64, ...): decode-step ffn1 shapes (one-warpgroup tiles); I = 192: a last tile of 64 channels, half used
@pytest.mark.parametrize("M,inter,K", [(520, 384, 328), (8192, 14336, 4096), (300, 128, 64), (64, 14336, 4096), (5, 192, 328),
                                       (33, 18944, 3584), (100, 192, 328), (520, 192, 328)])
def test_gemm_swiglu_fused_epilogue(M, inter, K):
    """gate|up projection + SwiGLU in one wgmma GEMM (tile = 128 gate columns | the 128 up columns of the same channels) is
    bit-identical to GEMM followed by the SwiGLU kernel: same accumulation order per element, same rounding points.  The
    inference form (gate|up not stored) is the decode step's ffn1."""
    o = ops()
    x = rand_bf16(M, K, seed=51, scale=0.7).to(DEV)
    w = rand_bf16(K, 2 * inter, seed=52, scale=0.3).to(DEV)
    gu_ref = o.gemm(x, w)
    m_ref = o.swiglu_fwd(gu_ref)
    gu, m = o.gemm_swiglu(x, w)
    assert torch.equal(gu, gu_ref)
    assert torch.equal(m, m_ref)
    ref = R.swiglu((x.float() @ w.float())[:, :inter].to(BF16).float(), (x.float() @ w.float())[:, inter:].to(BF16).float(), "bf16")
    assert maxerr(m, ref) < 2 ** -6
    _, m_only = o.gemm_swiglu(x, w, store_gate_up=False)       # inference form: gate|up are not written
    assert torch.equal(m_only, m_ref)
    with pytest.raises(Exception):
        o.gemm_swiglu(x, w[:, : 2 * 72].contiguous())              # I = 72 is not a multiple of 64


@pytest.mark.parametrize("M,inter,K", [(520, 320, 328), (8192, 14336, 4096), (300, 64, 64), (5, 192, 328), (100, 192, 328),
                                       (520, 192, 328)])
def test_gemm_swiglu_bwd_fused_epilogue(M, inter, K):
    """The down-projection dX GEMM with the SwiGLU backward in its epilogue is bit-identical to GEMM (dX) + swiglu_bwd kernel."""
    o = ops()
    dy = rand_bf16(M, K, seed=53, scale=0.5).to(DEV)
    wd = rand_bf16(inter, K, seed=54, scale=0.3).to(DEV)
    gu = rand_bf16(M, 2 * inter, seed=55, scale=1.5).to(DEV)
    dm = o.gemm(dy, wd, trans_b=True)
    ref = o.swiglu_bwd(gu, dm)
    got = o.gemm_swiglu_bwd(dy, wd, gu)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("tb", [False, True])
@pytest.mark.parametrize("M,N,K,split", [(64, 6144, 4096, 0), (64, 4096, 14336, 0), (8, 520, 328, 3), (100, 1024, 640, 0)])
def test_gemm_skinny_splitk(M, N, K, split, tb):
    o = ops()
    A = rand_bf16(M, K, seed=40, scale=0.5)
    B = rand_bf16(K, N, seed=41, scale=0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(42))
    b_d = (B.t().contiguous() if tb else B).to(DEV)
    out = o.gemm_skinny(A.to(DEV), b_d, trans_b=tb, bias=bias.to(DEV), split_k=split)
    ref = A.float().to(DEV) @ B.float().to(DEV) + bias.to(DEV)
    assert maxerr(out, ref) < 2 ** -7 and relerr(out, ref) < 4e-3


def test_gemm_argument_errors():
    o = ops()
    from paddlenlp_b200._lib import B200Error

    A = rand_bf16(64, 60).to(DEV)   # K = 60 is not a multiple of 8
    B = rand_bf16(60, 64).to(DEV)
    with pytest.raises((B200Error, AssertionError, ValueError)):
        o.gemm(A, B)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,h", [(37, 128), (256, 4096), (64, 3584), (5, 8192)])
def test_rmsnorm_fwd_bwd(rows, h):
    o = ops()
    x = rand_bf16(rows, h, seed=7)
    w = (1.0 + 0.1 * torch.randn(h, generator=torch.Generator().manual_seed(8))).to(BF16)
    dy = rand_bf16(rows, h, seed=9)
    dres = rand_bf16(rows, h, seed=10)
    eps = 1e-5
    y, rstd = o.rmsnorm_fwd(x.to(DEV), w.to(DEV), eps)
    ref = R.rms_norm(x.float(), w.float(), eps, "bf16")
    assert torch.equal(y.float().cpu(), ref) or maxerr(y.cpu(), ref) < 2 ** -7   # same rounding points: ~bit-exact
    assert (y.float().cpu() != ref).float().mean().item() < 0.01                # <1% of elements differ by 1 ulp
    # backward against autograd of the fp32 oracle
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    R.rms_norm(xf, wf, eps, "fp32").backward(dy.float())
    dw0 = rand_bf16(h, seed=11)
    dw = dw0.clone().to(DEV)
    dx = o.rmsnorm_bwd(dy.to(DEV), x.to(DEV), w.to(DEV), rstd, dw, dres=dres.to(DEV), accumulate_dw=True)
    assert relerr(dx.cpu(), xf.grad + dres.float()) < 6e-3        # bf16 output rounding ~ 2^-9 per element
    assert relerr(dw.cpu(), wf.grad + dw0.float()) < 6e-3


def test_colsum():
    o = ops()
    a = rand_bf16(300, 1024, seed=12).to(DEV)
    view = a[:, 256:768]
    out0 = rand_bf16(512, seed=13).to(DEV)
    out = out0.clone()
    o.colsum(view, out, accumulate=True)
    ref = view.float().sum(0) + out0.float()
    assert relerr(out, ref) < 4e-3


@pytest.mark.parametrize("backward", [False, True])
def test_rope(backward):
    o = ops()
    B, S, nh, kvh, d = 2, 96, 4, 2, 128
    ld = (nh + 2 * kvh) * d
    qkv = rand_bf16(B * S, ld, seed=14)
    cos, sin = o.rope_tables(d, 128, 500000.0, DEV)
    x = qkv.clone().to(DEV)
    o.rope_inplace(x, cos, sin, S, nh + kvh, d, backward=backward)
    c, s = R.rope_tables(d, S, 500000.0)
    qk = qkv[:, : (nh + kvh) * d].float().reshape(B, S, nh + kvh, d)
    if backward:
        s = -s
    ref = R.apply_rope(qk, c, s, "bf16").reshape(B * S, -1)
    got = x.cpu().float()
    assert maxerr(got[:, : (nh + kvh) * d], ref) < 2 ** -7
    assert torch.equal(got[:, (nh + kvh) * d:], qkv[:, (nh + kvh) * d:].float())   # v untouched
    # explicit position ids
    pos = torch.randint(0, 128, (B * S,), generator=torch.Generator().manual_seed(15)).int()
    x2 = qkv.clone().to(DEV)
    o.rope_inplace(x2, cos, sin, S, nh + kvh, d, position_ids=pos.to(DEV), backward=backward)
    c2, s2 = R.rope_tables(d, 128, 500000.0)
    if backward:
        s2 = -s2
    ref2 = R.apply_rope(qk, c2, s2, "bf16", position_ids=pos.long().reshape(B, S)).reshape(B * S, -1)
    assert maxerr(x2.cpu().float()[:, : (nh + kvh) * d], ref2) < 2 ** -7


def test_swiglu():
    o = ops()
    rows, inter = 130, 1192
    gu = rand_bf16(rows, 2 * inter, seed=16, scale=2.0)
    dm = rand_bf16(rows, inter, seed=17)
    m = o.swiglu_fwd(gu.to(DEV))
    g, u = gu[:, :inter].float().requires_grad_(True), gu[:, inter:].float().requires_grad_(True)
    ref = R.swiglu(g, u, "fp32")
    assert maxerr(m.cpu(), ref.detach()) < 2 ** -7
    ref.backward(dm.float())
    dgu = o.swiglu_bwd(gu.to(DEV), dm.to(DEV)).cpu()
    assert relerr(dgu[:, :inter], g.grad) < 6e-3
    assert relerr(dgu[:, inter:], u.grad) < 6e-3
    # fp32-workspace variant (decode step): rounds gate/up once, same bits as the bf16 op, hands the workspace back zeroed
    acc = (gu.float() * (1 + 2 ** -12)).to(DEV)                # not representable in bf16: exercises the rounding
    want = o.swiglu_fwd(acc.to(BF16))
    m2 = o.swiglu_fwd_f32(acc)
    assert torch.equal(m2, want) and not acc.any()


def test_embedding():
    o = ops()
    V, h, T = 1000, 256, 300
    table = rand_bf16(V, h, seed=18)
    ids = torch.randint(0, V, (T,), generator=torch.Generator().manual_seed(19))
    out = o.embedding_fwd(ids.to(DEV), table.to(DEV))
    assert torch.equal(out.cpu(), table[ids])
    dout = rand_bf16(T, h, seed=20)
    dtab = torch.zeros(V, h, dtype=BF16, device=DEV)
    o.embedding_bwd(ids.to(DEV), dout.to(DEV), dtab)
    ref = torch.zeros(V, h).index_add_(0, ids, dout.float())
    assert relerr(dtab.cpu(), ref) < 1e-2   # bf16 atomics: each add rounds


# ------------------------------------------------------------------------------------------------
@pytest.fixture
def fa_fwd_impl(request):
    """Select the attention tile height (b200_set_fa_fwd_impl / b200_set_fa_bwd_impl: 2 = 128-row q tiles, 1 = 64-row q tiles)
    for one test, then restore."""
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    old_f = lib.b200_set_fa_fwd_impl(request.param)
    old_b = lib.b200_set_fa_bwd_impl(request.param)
    yield request.param
    lib.b200_set_fa_fwd_impl(old_f)
    lib.b200_set_fa_bwd_impl(old_b)


@pytest.mark.parametrize("fa_fwd_impl", [2, 1], indirect=True)
@pytest.mark.parametrize("B,S,nh,kvh", [(1, 128, 1, 1), (2, 384, 4, 1), (1, 1024, 4, 2), (1, 200, 2, 2), (1, 72, 2, 1),
                                        (2, 640, 2, 2)])
def test_flash_attention_fwd_bwd(B, S, nh, kvh, fa_fwd_impl):
    o = ops()
    d = 128
    ld = (nh + 2 * kvh) * d
    qkv = rand_bf16(B, S, ld, seed=21, scale=1.0).to(DEV)
    q = qkv[:, :, : nh * d].view(B, S, nh, d)
    k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    out, lse = o.flash_attn_fwd(q, k, v)
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    ref = R.attention(qf, kf, vf, "fp32")                     # [B, S, nh*d]
    assert maxerr(out.reshape(B, S, -1), ref.detach()) < 1.5e-2   # P rounded to bf16 before PV + bf16 output
    assert relerr(out.reshape(B, S, -1), ref.detach()) < 1e-2
    # lse check
    scores = torch.einsum("bqhd,bkhd->bhqk", qf, kf.repeat_interleave(nh // kvh, dim=2)) / math.sqrt(d)
    mask = torch.full((S, S), float("-inf"), device=DEV).triu(1)
    lse_ref = torch.logsumexp(scores + mask, dim=-1)
    assert (lse - lse_ref).abs().max().item() < 2e-3
    # backward
    dout = rand_bf16(B, S, nh, d, seed=22).to(DEV)
    ref.backward(dout.float().reshape(B, S, -1))
    dqkv = torch.zeros_like(qkv)
    dq = dqkv[:, :, : nh * d].view(B, S, nh, d)
    dk = dqkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    dv = dqkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    o.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv)
    # tolerance precedent: reference compares bf16 attention grads at 1e-2 (tests/transformers/test_ring_flash_attention.py:94-107)
    assert relerr(dq, qf.grad) < 2e-2
    assert relerr(dk, kf.grad) < 2e-2
    assert relerr(dv, vf.grad) < 2e-2


def _doc_mask(doc_lens, S):
    """FlashMask start rows of packed documents: column c -> end of c's document (zero_padding_dataset.py:84-86)."""
    ms = torch.empty(S, dtype=torch.int32)
    pos = 0
    for n in doc_lens:
        ms[pos:pos + n] = pos + n
        pos += n
    assert pos == S
    return ms


@pytest.mark.parametrize("S,nh,kvh,docs", [(384, 2, 1, [[100, 284], [128, 128, 128]]), (1024, 4, 2, [[1, 700, 323]]),
                                           (200, 2, 2, [[7, 57, 136]]), (640, 1, 1, [[256, 1, 383], [640]]),
                                           (1024, 2, 1, [[300, 724], [130, 126, 256, 512], [257, 255, 129, 383]]),
                                           (1536, 4, 4, [[640, 40, 856], [2, 1300, 234]]),
                                           (900, 2, 2, [[513, 387], [128, 600, 172]]),
                                           (2048, 12, 2, [[1, 511, 1024, 512], [2048]])])
@pytest.mark.parametrize("fa_fwd_impl", [2, 1], indirect=True)
def test_flash_attention_flashmask(S, nh, kvh, docs, fa_fwd_impl):
    """Packed-document (FlashMask causal-LT) attention, forward and backward, vs the oracle's masked softmax; a row of
    [S]*S start rows is plain causal.  Document boundaries on and off the 128-row tile grid (and off the 256-row block grid of
    the two-q-tile forward: its second tile can join the kv stream later than the first), 1-token documents, ragged S.
    The bit-equality properties below compare masked and unmasked runs of the SAME kernel generation."""
    o = ops()
    B, d = len(docs), 128
    ms = torch.stack([_doc_mask(dl, S) for dl in docs])
    ld = (nh + 2 * kvh) * d
    qkv = rand_bf16(B, S, ld, seed=31).to(DEV)
    q = qkv[:, :, : nh * d].view(B, S, nh, d)
    k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    out, lse = o.flash_attn_fwd(q, k, v, mask_start=ms.to(DEV))
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    ref = R.attention(qf, kf, vf, "fp32", mask_start=ms)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert maxerr(out.reshape(B, S, -1), ref.detach()) < 1.5e-2
    dout = rand_bf16(B, S, nh, d, seed=32).to(DEV)
    ref.backward(dout.float().reshape(B, S, -1))
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    o.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, mask_start=ms.to(DEV))
    for name, a, r in (("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
        assert relerr(a, r) < 2e-2, (name, relerr(a, r))
    # packing invariance: the first document alone gives the same bits for its rows (same tiles, same order)
    n0 = docs[0][0]
    if n0 >= 2:
        solo, _ = o.flash_attn_fwd(q[:1, :n0].contiguous(), k[:1, :n0].contiguous(), v[:1, :n0].contiguous())
        assert torch.equal(solo, out[:1, :n0])
    # mask_start = S everywhere == no mask
    full = torch.full((B, S), S, dtype=torch.int32, device=DEV)
    a, la = o.flash_attn_fwd(q, k, v, mask_start=full)
    b, lb = o.flash_attn_fwd(q, k, v)
    assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.parametrize("fa_fwd_impl", [2, 1], indirect=True)
@pytest.mark.parametrize("S,pads", [(512, [200, 0]), (700, [129, 511]), (384, [300, 1])])
def test_flash_attention_left_padding_start_rows(S, pads, fa_fwd_impl):
    """Left-padded batches in start-row form (llama/modeling.py `_mask_rows_from_padding_mask`: a padding column is a one-token
    document, start = c + 1; real columns keep S): the real rows reproduce the un-padded sequence, forward and backward."""
    o = ops()
    B, nh, kvh, d = len(pads), 2, 1, 128
    ms = torch.full((B, S), S, dtype=torch.int32)
    for b, pad in enumerate(pads):
        ms[b, :pad] = torch.arange(1, pad + 1, dtype=torch.int32)
    qkv = rand_bf16(B, S, (nh + 2 * kvh) * d, seed=41).to(DEV)
    q = qkv[:, :, : nh * d].view(B, S, nh, d)
    k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    out, lse = o.flash_attn_fwd(q, k, v, mask_start=ms.to(DEV))
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    dout = rand_bf16(B, S, nh, d, seed=42).to(DEV)
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    o.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, mask_start=ms.to(DEV))
    for b, pad in enumerate(pads):
        qf, kf, vf = (t[b:b + 1, pad:].float().detach().requires_grad_(True) for t in (q, k, v))
        ref = R.attention(qf, kf, vf, "fp32")
        assert maxerr(out[b:b + 1, pad:].reshape(1, S - pad, -1), ref.detach()) < 1.5e-2
        ref.backward(dout[b:b + 1, pad:].float().reshape(1, S - pad, -1))
        for name, a, r in (("dq", dq, qf.grad), ("dk", dk, kf.grad), ("dv", dv, vf.grad)):
            assert relerr(a[b:b + 1, pad:], r) < 2e-2, (name, b, relerr(a[b:b + 1, pad:], r))


def worst_tile_relerr(a, r, tile):
    """Largest relerr over blocks of `tile` consecutive rows of one head: a, r [S, heads, d] (rows = sequence positions)."""
    a, r = a.float(), r.float()
    S, H = a.shape[0], a.shape[1]
    idx = torch.arange(S, device=a.device) // tile
    nt = (S + tile - 1) // tile
    e2 = torch.zeros(nt, H, device=a.device).index_add_(0, idx, (a - r).pow(2).sum(-1))
    r2 = torch.zeros(nt, H, device=a.device).index_add_(0, idx, r.pow(2).sum(-1))
    return (e2 / r2.clamp_min(1e-30)).sqrt().max().item()


@pytest.mark.parametrize("fa_fwd_impl", [2, 1], indirect=True)
@pytest.mark.parametrize("B,S,nh,kvh", [(2, 4096, 32, 8), (1, 2048, 28, 4), (1, 4096, 24, 8), (4, 2048, 12, 2)])
def test_flash_attention_bench_shapes(B, S, nh, kvh, fa_fwd_impl):
    """The attention kernels at large training shapes against the fp32 oracle evaluated on the GPU: the Llama-3-8B (2 x 4096
    x 32/8 heads) and Qwen2-7B (2048 x 28/4) layouts, and the two benchmarked models, Llama-3.2-3B (one 4096-token sequence,
    24/8 heads: GQA ratio 3) and Qwen2-1.5B (4 x 2048, 12/2 heads: GQA ratio 6).  Besides the global errors, every (head,
    128-row q tile) of out and dq and every (kv head, 64-row kv tile) of dk and dv is checked on its own, so that one wrong
    tile among hundreds cannot hide in the tensor's norm."""
    o = ops()
    d = 128
    ld = (nh + 2 * kvh) * d
    qkv = rand_bf16(B, S, ld, seed=61, scale=1.0).to(DEV)
    q = qkv[:, :, : nh * d].view(B, S, nh, d)
    k = qkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    v = qkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    out, lse = o.flash_attn_fwd(q, k, v)
    dout = rand_bf16(B, S, nh, d, seed=62).to(DEV)
    dqkv = torch.zeros_like(qkv)
    dq = dqkv[:, :, : nh * d].view(B, S, nh, d)
    dk = dqkv[:, :, nh * d: (nh + kvh) * d].view(B, S, kvh, d)
    dv = dqkv[:, :, (nh + kvh) * d:].view(B, S, kvh, d)
    o.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv)
    # oracle, one batch row at a time (the fp32 score matrix of one row is nh x S x S x 4 B = 2.1 GB at 32 x 4096)
    worst = {}
    worst_tile = {}
    for b in range(B):
        qf, kf, vf = (t[b:b + 1].float().detach().requires_grad_(True) for t in (q, k, v))
        ref = R.attention(qf, kf, vf, "fp32")
        e_out = (maxerr(out[b:b + 1].reshape(1, S, -1), ref.detach()), relerr(out[b:b + 1].reshape(1, S, -1), ref.detach()))
        assert e_out[0] < 1.5e-2 and e_out[1] < 1e-2, e_out
        # per tile: the worst tile measured on an H100 is 2.4e-3 for out, 3.2e-3 for the gradients; a wrong tile is O(1)
        e = worst_tile_relerr(out[b], ref.detach().view(S, nh, d), 128)
        worst_tile["out"] = max(worst_tile.get("out", 0.0), e)
        assert e < 1e-2, ("out", b, e)
        scores = torch.einsum("bqhd,bkhd->bhqk", qf.detach(), kf.detach().repeat_interleave(nh // kvh, dim=2)) / math.sqrt(d)
        scores += torch.full((S, S), float("-inf"), device=DEV).triu(1)
        lse_ref = torch.logsumexp(scores, dim=-1)
        del scores
        assert (lse[b:b + 1] - lse_ref).abs().max().item() < 2e-3
        ref.backward(dout[b:b + 1].float().reshape(1, S, -1))
        for name, a, r in (("dq", dq[b:b + 1], qf.grad), ("dk", dk[b:b + 1], kf.grad), ("dv", dv[b:b + 1], vf.grad)):
            e = relerr(a, r)
            worst[name] = max(worst.get(name, 0.0), e)
            assert e < 2e-2, (name, b, e)
            e = worst_tile_relerr(a[0], r[0], 128 if name == "dq" else 64)
            worst_tile[name] = max(worst_tile.get(name, 0.0), e)
            assert e < 1e-2, (name, b, e)
        del ref, qf, kf, vf, lse_ref
    print(f"[fa {B}x{S}x{nh}/{kvh} impl {fa_fwd_impl}] grad rel err {worst}, worst tile rel err {worst_tile}")


def test_flash_attention_bwd_impls_agree():
    """Both backward generations from the same forward state: gradients agree to summation-order noise (ragged S, GQA)."""
    from paddlenlp_b200 import _lib
    o = ops()
    lib = _lib.load()
    B, S, nh, kvh, d = 2, 1000, 4, 2, 128
    q, k, v = rand_bf16(B, S, nh, d, seed=81).to(DEV), rand_bf16(B, S, kvh, d, seed=82).to(DEV), rand_bf16(B, S, kvh, d, seed=83).to(DEV)
    out, lse = o.flash_attn_fwd(q, k, v)
    dout = rand_bf16(B, S, nh, d, seed=84).to(DEV)
    res = {}
    old = lib.b200_set_fa_bwd_impl(1)
    try:
        for impl in (1, 2):
            lib.b200_set_fa_bwd_impl(impl)
            dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
            o.flash_attn_bwd(q, k, v, out, dout, lse, dq, dk, dv)
            res[impl] = (dq, dk, dv)
    finally:
        lib.b200_set_fa_bwd_impl(old)
    for name, a, b in zip(("dq", "dk", "dv"), res[2], res[1]):
        assert torch.isfinite(a.float()).all(), name
        assert relerr(a, b) < 5e-3, (name, relerr(a, b))


def test_flash_attention_fwd_impls_agree():
    """The two forward generations implement the same rounding points: outputs agree to P-rounding / summation-order noise and
    the saved log-sum-exp to fp32 noise, on a shape with an odd number of 128-row tiles (the last 256-row block half empty)."""
    from paddlenlp_b200 import _lib
    o = ops()
    lib = _lib.load()
    B, S, nh, kvh, d = 2, 1152 + 40, 4, 2, 128
    q, k, v = rand_bf16(B, S, nh, d, seed=71).to(DEV), rand_bf16(B, S, kvh, d, seed=72).to(DEV), rand_bf16(B, S, kvh, d, seed=73).to(DEV)
    old = lib.b200_set_fa_fwd_impl(1)
    try:
        o1, l1 = o.flash_attn_fwd(q, k, v)
        lib.b200_set_fa_fwd_impl(2)
        o2, l2 = o.flash_attn_fwd(q, k, v)
    finally:
        lib.b200_set_fa_fwd_impl(old)
    assert torch.isfinite(o2.float()).all() and torch.isfinite(l2).all()
    assert maxerr(o2, o1) < 1.5e-2 and relerr(o2, o1) < 5e-3
    assert (l1 - l2).abs().max().item() < 1e-4


# ------------------------------------------------------------------------------------------------
def test_cross_entropy():
    o = ops()
    T, V = 100, 5000
    logits = rand_bf16(T, V, seed=23, scale=2.0)
    labels = torch.randint(0, V, (T,), generator=torch.Generator().manual_seed(24))
    labels[::7] = -100
    lg = logits.clone().to(DEV)
    loss_out, loss_tok, lse = o.ce_fwd(lg, labels.to(DEV))
    lf = logits.float().requires_grad_(True)
    ref = R.criterion(lf, labels)
    assert abs(loss_out[0].item() - ref.item()) < 1e-4 * abs(ref.item())
    assert loss_out[1].item() == float((labels != -100).sum())
    ref.backward()
    o.ce_bwd_(lg, labels.to(DEV), loss_tok, lse, loss_out, grad_scale=1.0)
    assert relerr(lg.cpu(), lf.grad) < 6e-3
    am = o.argmax(logits.to(DEV))
    assert torch.equal(am.cpu(), logits.float().argmax(-1))


def test_adamw_and_clip():
    o = ops()
    n, decay_end = 8 * 5000, 8 * 3000
    g = torch.Generator().manual_seed(25)
    p16 = (torch.randn(n, generator=g) * 0.02).to(BF16)
    grad = (torch.randn(n, generator=g) * 0.01).to(BF16)
    master = p16.float()
    m = torch.randn(n, generator=g) * 1e-3
    v = torch.rand(n, generator=g) * 1e-5
    hp = dict(lr=3e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=7)
    mask = torch.arange(n) < decay_end
    pr, mr, vr, p16r = optim_ref.adamw_step(master, m, v, grad.float(), decay_mask=mask, grad_scale=0.5,
                                            max_grad_norm=1.0, **hp)
    P, G, M_, V_, MA = p16.to(DEV), grad.to(DEV), m.to(DEV), v.to(DEV), master.to(DEV)
    sq = o.grad_sqnorm(G, scale=0.5)
    assert abs(sq.item() - (grad.float() * 0.5).pow(2).sum().item()) < 1e-4 * sq.item()
    o.adamw_step(P, G, MA, M_, V_, sq, decay_end=decay_end, grad_scale=0.5, max_grad_norm=1.0, **hp)
    assert relerr(MA.cpu(), pr) < 1e-6
    assert relerr(M_.cpu(), mr) < 1e-5
    assert relerr(V_.cpu(), vr) < 1e-5
    assert (P.cpu().float() != p16r.float()).float().mean().item() < 1e-3


# ----------------------------------------------------------------------------------------------------------
# The reference's per-op plug-in seam (llama/fusion_ops.py) with autograd: forward and gradients vs the oracle
# ----------------------------------------------------------------------------------------------------------
def test_fusion_ops_seam_autograd():
    from paddlenlp_b200.transformers.llama import fusion_ops as F
    from paddlenlp_b200.transformers.llama.configuration import LlamaConfig

    b, s, nh, kvh, d, h, inter = 2, 256, 4, 2, 128, 512, 384
    g = torch.Generator().manual_seed(5)
    leaf = lambda *shape, sc=1.0: (torch.randn(*shape, generator=g) * sc).to(BF16)

    # --- rms norm
    x, w, dy = leaf(b, s, h), (1 + 0.1 * torch.randn(h, generator=g)).to(BF16), leaf(b, s, h)
    xd, wd = x.to(DEV).requires_grad_(), w.to(DEV).requires_grad_()
    y = F.fusion_rms_norm(xd, wd, 1e-5)
    y.backward(dy.to(DEV))
    xo, wo = x.float().requires_grad_(), w.float().requires_grad_()
    yo = R.rms_norm(xo, wo, 1e-5, "fp32")
    yo.backward(dy.float())
    assert maxerr(y.cpu(), yo) < 1e-2 and relerr(xd.grad.cpu(), xo.grad) < 1e-2 and relerr(wd.grad.cpu(), wo.grad) < 1e-2

    # --- rope (with and without position_ids) + flash attention + reshape
    q, k, v, do = leaf(b, s, nh, d), leaf(b, s, kvh, d), leaf(b, s, kvh, d), leaf(b, s, nh * d)
    rot = F.LlamaRotaryEmbedding(d, max_position_embeddings=512, base=500000.0, device=DEV)
    cos, sin = R.rope_tables(d, 512, 500000.0)
    for pos in (None, torch.arange(s).flip(0)[None, :].expand(b, s).contiguous()):
        qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
        q2, k2 = F.fusion_rope(qd, kd, vd, None, None if pos is None else pos.to(DEV), None, rot)
        if pos is not None:          # permuted positions only exercise RoPE (causality needs ordered positions)
            qo = R.apply_rope(q.float(), cos, sin, "fp32", pos)
            assert maxerr(q2.cpu(), qo) < 1e-2
            continue
        out = F.fusion_flash_attention(q2, LlamaConfig(), k2, vd, None, False)
        assert out.shape == (b, s, nh * d)
        out.backward(do.to(DEV))
        qo, ko, vo = (t.float().requires_grad_() for t in (q, k, v))
        oo = R.attention(R.apply_rope(qo, cos, sin, "fp32"), R.apply_rope(ko, cos, sin, "fp32"), vo, "fp32")
        oo.backward(do.float())
        assert maxerr(out.cpu(), oo) < 2e-2
        for name, a, r in (("dq", qd.grad, qo.grad), ("dk", kd.grad, ko.grad), ("dv", vd.grad, vo.grad)):
            assert relerr(a.cpu(), r) < 2e-2, (name, relerr(a.cpu(), r))
    with pytest.raises(NotImplementedError):
        F.fusion_flash_attention(q2, LlamaConfig(), k2, vd, torch.ones(1, device=DEV), False)
    with pytest.raises(AssertionError):
        F.fusion_rope(qd, kd, vd, None, None, (kd, vd), rot)

    # --- swiglu: both call forms of llama/modeling.py:38-45
    gt, up, dz = leaf(b, s, inter), leaf(b, s, inter), leaf(b, s, inter)
    gd, ud = gt.to(DEV).requires_grad_(), up.to(DEV).requires_grad_()
    z = F.swiglu(gd, ud)
    z.backward(dz.to(DEV))
    go, uo = gt.float().requires_grad_(), up.float().requires_grad_()
    zo = R.swiglu(go, uo, "fp32")
    zo.backward(dz.float())
    assert maxerr(z.cpu(), zo) < 1e-2 and relerr(gd.grad.cpu(), go.grad) < 1e-2 and relerr(ud.grad.cpu(), uo.grad) < 1e-2
    z2 = F.swiglu(torch.cat([gt, up], -1).to(DEV))
    assert torch.equal(z2, z.detach())
