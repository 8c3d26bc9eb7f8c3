"""Bit-exact checks of the wgmma GEMM's shared-memory / TMA-store epilogue (64- and 128-row tiles).

Reference: the kernel's own fp32 accumulators, from b200_gemm_bf16_splitk with split_k = 1 and C = NULL (the same tiles in the
same k order; its reduce-add into a zeroed workspace is exact).  The epilogue is then applied in torch with the kernel's
rounding points:
  mode 0: bf16(acc + bias)      mode 1: bf16((acc + bias) + C_old)      mode 2: bf16(bf16(acc + bias) + R)
The fused SwiGLU GEMMs must equal the unfused GEMM followed by swiglu_fwd / swiglu_bwd, bit for bit.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BF16 = torch.bfloat16


def _ops():
    from paddlenlp_b200 import ops

    return ops


def _acc(a, b, trans_a, trans_b):
    """fp32 accumulators of op(a) @ op(b), as the GEMM kernel forms them."""
    from paddlenlp_b200 import _lib

    K, M = a.shape if trans_a else a.shape[::-1]
    N = b.shape[0] if trans_b else b.shape[1]
    ws = torch.zeros(M, N, dtype=torch.float32, device=DEV)
    _lib.call("b200_gemm_bf16_splitk", _lib.ptr(a), _lib.ptr(b), None, None, _lib.ptr(ws), M, N, K, a.stride(0), b.stride(0),
              N, 1 if trans_a else 0, 0 if trans_b else 1, 1, _lib.stream_ptr())
    return ws


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(BF16)


def _mat(rows, cols, scale, seed):
    """[rows, cols] view whose leading dimension is padded to a multiple of 8 elements, as the GEMM requires."""
    return _rand(rows, -(-cols // 8) * 8, scale=scale, seed=seed)[:, :cols]


def _operands(M, N, K, trans_a, trans_b, seed):
    a = _mat(*((K, M) if trans_a else (M, K)), scale=0.5, seed=seed)
    b = _mat(*((N, K) if trans_b else (K, N)), scale=0.5, seed=seed + 1)
    return a, b


def _check(M, N, K, trans_a, trans_b, mode, bias=False, max_ctas=0, out_pad=0, seed=0):
    ops = _ops()
    a, b = _operands(M, N, K, trans_a, trans_b, seed)
    bias_t = torch.randn(N, generator=torch.Generator(device=DEV).manual_seed(seed + 2), device=DEV) if bias else None
    acc = _acc(a, b, trans_a, trans_b)
    f = acc + bias_t if bias else acc
    out = torch.full((M, N + out_pad), float("nan"), dtype=BF16, device=DEV)[:, :N]
    residual = None
    if mode == 0:
        want = f.to(BF16)
    elif mode == 1:
        out.copy_(_rand(M, N, scale=4.0, seed=seed + 3))
        want = (f + out.float()).to(BF16)
    else:
        residual = torch.empty(M, N + out_pad, dtype=BF16, device=DEV)[:, :N]
        residual.copy_(_rand(M, N, scale=4.0, seed=seed + 3))
        want = (f.to(BF16).float() + residual.float()).to(BF16)
    got = ops.gemm(a, b, out, trans_a=trans_a, trans_b=trans_b, accumulate=mode == 1, bias=bias_t, residual=residual,
                   max_ctas=max_ctas)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()


# Every training GEMM of the Llama-3.2-3B (h 3072, I 8192, q|k|v 5120, V 128256, 4096 tokens) and Qwen2-1.5B (h 1536, I 8960,
# q|k|v 2048 with bias, V 151936, 4 x 2048 tokens) steps in its real layout and epilogue: (M, N, K, trans_a, trans_b, mode, bias).
# Forward and dX GEMMs are token-major; weight gradients are op(X^T) dY accumulated into the gradient buffer.
def _step_gemms(T, h, inter, qkv, V, qkv_bias):
    return [
        ("qkv", T, qkv, h, False, False, 0, qkv_bias),
        ("o", T, h, h, False, False, 2, False),
        ("down", T, h, inter, False, False, 2, False),
        ("head", T, V, h, False, False, 0, False),
        ("dx_head", T, h, V, False, True, 0, False),
        ("dx_qkv", T, h, qkv, False, True, 0, False),
        ("dx_o", T, h, h, False, True, 0, False),
        ("dx_gate_up", T, h, 2 * inter, False, True, 0, False),
        ("dw_qkv", h, qkv, T, True, False, 1, False),
        ("dw_o", h, h, T, True, False, 1, False),
        ("dw_gate_up", h, 2 * inter, T, True, False, 1, False),
        ("dw_down", inter, h, T, True, False, 1, False),
        ("dw_head", h, V, T, True, False, 1, False),
    ]


STEP_GEMMS = ([("llama3b_" + c[0],) + c[1:] for c in _step_gemms(4096, 3072, 8192, 5120, 128256, False)]
              + [("qwen2_" + c[0],) + c[1:] for c in _step_gemms(8192, 1536, 8960, 2048, 151936, True)])


@pytest.mark.parametrize("case", STEP_GEMMS, ids=[c[0] for c in STEP_GEMMS])
def test_step_gemm_bit_exact(case):
    _, M, N, K, ta, tb, mode, bias = case
    _check(M, N, K, ta, tb, mode, bias=bias)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("trans", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("M", [4095, 5, 33, 48, 64])
def test_ragged_edges(M, mode, trans):
    """M and N not multiples of the tile: TMA clips the last boxes (5112 = 19 x 256 + 248, 4095 = 31 x 128 + 127).
    M <= 64 runs 64-row tiles (the decode step's and small prefills' GEMMs)."""
    _check(M, 5112, 1000, trans[0], trans[1], mode, bias=mode != 1, seed=11)


@pytest.mark.parametrize("max_ctas", [1, 7, 0])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("M,N", [(1100, 1400), (48, 3000)])
def test_max_ctas_buffer_recycling(M, N, max_ctas, mode):
    """One CTA walking every tile, 7 CTAs (a partial last raster group; 5 of them run two of the 12 64-row tiles), and all
    SMs."""
    _check(M, N, 192, False, False, mode, bias=True, max_ctas=max_ctas, seed=21)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_strided_views(mode):
    _check(700, 520, 256, False, True, mode, out_pad=72, seed=31)


@pytest.mark.parametrize("offset", [4, 8])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_misaligned_output_rejected(mode, offset):
    """A view starting 4 or 8 bytes past a 16-byte boundary cannot be a TMA base: an output (modes 0, 1) or residual (mode 2)
    view like that is an argument error, and nothing is written."""
    from paddlenlp_b200._lib import B200Error

    ops = _ops()
    M, N, K = 600, 512, 256
    a, b = _operands(M, N, K, False, False, 41)
    e = offset // 2
    buf = torch.full((M, N + 8), float("nan"), dtype=BF16, device=DEV)
    out, residual = buf[:, e:N + e], None
    if mode == 2:
        out = buf[:, :N]
        residual = _rand(M, N + 8, seed=43)[:, e:N + e]
    with pytest.raises(B200Error, match="residual must be 16-byte aligned" if mode == 2 else "C must be 16-byte aligned"):
        ops.gemm(a, b, out, accumulate=mode == 1, residual=residual)
    torch.cuda.synchronize()
    assert torch.isnan(buf.float()).all()


def test_in_place_accumulate_into_live_gradient_buffer():
    """Two accumulating weight-gradient GEMMs into a slice of one flat buffer; its neighbours stay untouched."""
    ops = _ops()
    h, N, T = 1536, 2048, 2048
    flat = _rand(3 * h * N, seed=51)
    before = flat.clone()
    g = flat[h * N: 2 * h * N].view(h, N)
    want = g.float()
    for s in range(2):
        x, dy = _rand(T, h, seed=52 + 2 * s), _rand(T, N, seed=53 + 2 * s)
        want = (_acc(x, dy, True, False) + want).to(BF16).float()
        ops.gemm(x, dy, g, trans_a=True, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(g.float(), want)
    assert torch.equal(flat[: h * N], before[: h * N]) and torch.equal(flat[2 * h * N:], before[2 * h * N:])


@pytest.mark.parametrize("M,h,inter", [(4096, 3072, 8192), (8192, 1536, 8960), (4095, 1000, 4160), (5, 4096, 14336),
                                       (64, 1000, 4160)])
def test_swiglu_fwd_fused_equals_unfused(M, h, inter):
    """Mode 4: gate|up and m equal the plain GEMM followed by swiglu_fwd (4160 channels: the last n-tile has 64; M <= 64: 64-row
    tiles, as the decode step's ffn1, which stores m only)."""
    ops = _ops()
    x, w = _rand(M, h, seed=61), _rand(h, 2 * inter, scale=0.05, seed=62)
    gu = torch.full((M, 2 * inter), float("nan"), dtype=BF16, device=DEV)
    m = torch.full((M, inter), float("nan"), dtype=BF16, device=DEV)
    ops.gemm_swiglu(x, w, gu, m)
    gu_ref = ops.gemm(x, w)
    m_ref = ops.swiglu_fwd(gu_ref)
    _, m_only = ops.gemm_swiglu(x, w, store_gate_up=False)
    torch.cuda.synchronize()
    assert torch.equal(gu, gu_ref)
    assert torch.equal(m, m_ref)
    assert torch.equal(m_only, m_ref)


@pytest.mark.parametrize("M,h,inter", [(4096, 3072, 8192), (8192, 1536, 8960), (4095, 1000, 4160), (5, 3072, 8192),
                                       (64, 1000, 4160)])
def test_swiglu_bwd_fused_equals_unfused(M, h, inter):
    """Mode 5: d(gate)|d(up) equals the plain dX GEMM followed by swiglu_bwd."""
    ops = _ops()
    dy, w_down = _rand(M, h, seed=71), _rand(inter, h, scale=0.05, seed=72)
    gu = _rand(M, 2 * inter, seed=73)
    dgu = torch.full((M, 2 * inter), float("nan"), dtype=BF16, device=DEV)
    ops.gemm_swiglu_bwd(dy, w_down, gu, dgu)
    dm = ops.gemm(dy, w_down, trans_b=True)
    dgu_ref = ops.swiglu_bwd(gu, dm)
    torch.cuda.synchronize()
    assert torch.equal(dgu, dgu_ref)

