"""Weight-only int8 without a GPU: the restatement's properties (oracle/weight_only_ref.py), FusedMultiTransformerConfig's
quant_type validation, the C-ABI's argument errors (returned before any device work) and the ptxas log of weight_only.cu."""
import ctypes
import os
import re

import pytest
import torch

from oracle import weight_only_ref as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _w(K=64, N=48, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (0.02 * torch.randn(K, N, generator=g)).to(torch.bfloat16)


def test_quantised_values_bounded_and_within_half_a_step():
    w = _w(256, 96)
    w[:, 5] *= 40                                          # an outlier column
    q, s = W.quantize(w)
    assert q.dtype == torch.int8 and s.dtype == torch.bfloat16 and s.shape == (96,)
    assert int(q.abs().max()) <= 127
    assert bool((q.abs().amax(dim=0) >= 126).all())        # every column uses (nearly) the whole range
    err = (w.double() - q.double() * s.double()).abs()
    assert bool((err <= s.double() / 2 * (1 + 2 ** -20)).all())


def test_scale_is_bf16_of_absmax_over_127():
    w = _w(32, 16, seed=1)
    _, s = W.quantize(w)
    a = w.float().abs().amax(dim=0)
    assert torch.equal(s, (a / 127.0).to(torch.bfloat16))


def test_zero_column_gives_zero_scale_and_zero_q():
    w = _w()
    w[:, 3] = 0
    q, s = W.quantize(w)
    assert float(s[3]) == 0 and int(q[:, 3].abs().max()) == 0


def test_half_way_quotients_round_to_even():
    s = 2.0 ** -10
    col = torch.tensor([127, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.5] * 2, dtype=torch.float64) * s
    q, sc = W.quantize(col.to(torch.bfloat16)[:, None])
    assert float(sc[0]) == s
    assert q[:, 0].tolist() == [127, 0, 2, 2, 0, -2, -2, 4] * 2


def test_clamp_column():
    """A subnormal-range scale: bf16(189 2^-133 / 127) = 2^-133, so the largest quotient is 189 and clamps to 127 (for a normal
    scale bf16 rounding moves a / scale by at most 2^-8 relative: it stays below 127.5)."""
    col = torch.tensor([189, -189, 100, -3, 0, 150, 120, 1] * 2, dtype=torch.float64) * 2.0 ** -133
    w = col.to(torch.bfloat16)[:, None]
    a = w.float().abs().amax()
    q, s = W.quantize(w)
    assert float(s[0]) == 2.0 ** -133 and float(a / s.float()[0]) > 127.5
    assert q[:, 0].tolist()[:8] == [127, -127, 100, -3, 0, 127, 120, 1]


def test_pack_layout():
    """Lane l of unit (g, s) holds q[16s + c + {0, 1, 8, 9}][8g + l/4] with c = 2 (l % 4)."""
    K, N = 32, 16
    q = torch.arange(K * N, dtype=torch.int64).view(K, N) % 251 - 125
    p = W.pack(q.to(torch.int8)).view(-1)
    for g in range(N // 8):
        for s in range(K // 16):
            for lane in range(32):
                n, c = 8 * g + lane // 4, 2 * (lane % 4)
                base = ((g * (K // 16) + s) * 32 + lane) * 4
                want = [q[16 * s + c + d, n] for d in (0, 1, 8, 9)]
                assert p[base:base + 4].tolist() == [int(v) for v in want]


def test_config_quant_type_validation():
    from paddlenlp_b200.experimental.transformers import FusedMultiTransformerConfig

    kw = dict(embed_dim=256, num_heads=2, dim_feedforward=512)
    assert FusedMultiTransformerConfig(**kw).quant_type == ""
    assert FusedMultiTransformerConfig(quant_type="weight_only_int8", **kw).quant_type == "weight_only_int8"
    for qt in ("weight_only_int4", "a8w8", "a8w8c8", "a8w8_fp8", "fp8"):
        with pytest.raises(NotImplementedError):
            FusedMultiTransformerConfig(quant_type=qt, **kw)
    for qt in ("int8", "weight_only", "wint8"):
        with pytest.raises(ValueError):
            FusedMultiTransformerConfig(quant_type=qt, **kw)


def test_weight_only_classes_are_exported_under_the_paddlenlp_alias():
    import paddlenlp  # noqa: F401
    from paddlenlp.experimental.transformers import FusedBlockMultiTransformerWeightOnly, FusedMultiTransformerWeightOnly
    from paddlenlp_b200.experimental.transformers import fused_transformer_layers as F

    assert FusedMultiTransformerWeightOnly is F.FusedMultiTransformerWeightOnly
    assert issubclass(FusedBlockMultiTransformerWeightOnly, F.FusedBlockMultiTransformer)
    assert issubclass(FusedMultiTransformerWeightOnly, F.WeightOnlyInt8Mixin)


def test_abi_argument_errors():
    """Rejected with an argument error (< 0) before any device work, so no GPU is needed."""
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    a = ctypes.c_void_p(0x10000)                           # 16-byte aligned, never dereferenced
    odd = ctypes.c_void_p(0x10008)

    def gemm(M=4, N=64, K=64, ldx=64, ldc=64, X=a, Q=a, C=a, ws=None, split=0):
        return lib.b200_weight_only_gemm_bf16(X, Q, a, None, C, ws, M, N, K, ldx, ldc, split, None)

    def gemm_f32(M=4, N=64, K=64, X=a, Q=a, ws=a):
        return lib.b200_weight_only_gemm_f32(X, Q, a, ws, M, N, K, K, 0, None)

    quant = lib.b200_weight_quantize_int8
    cases = [(lambda: gemm(K=40, ldx=40), "multiple of 16"), (lambda: gemm(N=60, ldc=64), "multiple of 8"),
             (lambda: gemm(M=0), "non-positive"), (lambda: gemm(M=-3), "non-positive"), (lambda: gemm(X=odd), "16-byte"),
             (lambda: gemm(Q=odd), "16-byte"), (lambda: gemm(C=odd), "16-byte"), (lambda: gemm(split=4), "workspace"),
             (lambda: gemm(ldx=60), "ldx"), (lambda: gemm_f32(K=24), "multiple of 16"), (lambda: gemm_f32(N=4), "multiple of 8"),
             (lambda: gemm_f32(M=0), "non-positive"), (lambda: gemm_f32(ws=odd), "16-byte"), (lambda: gemm_f32(ws=None), "workspace"),
             (lambda: quant(a, a, a, 40, 64, 64, None), "multiple of 16"), (lambda: quant(a, a, a, 64, 12, 64, None), "multiple of 8"),
             (lambda: quant(a, a, a, 0, 64, 64, None), "non-positive")]
    for fn, msg in cases:
        assert fn() < 0, msg
        assert msg in lib.b200_last_error().decode(), (msg, lib.b200_last_error())


def test_weight_only_ptxas_log():
    """No instantiation of the W8 GEMM (or the quantise kernel) spills or uses a stack, and ptxas serialised no wgmma (C7510)."""
    log = os.path.join(ROOT, "paddlenlp_b200", "build", "weight_only.o.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log: the library was not built in this tree")
    text = open(log).read()
    assert "C7510" not in text
    found = re.findall(r"Compiling entry function '(\w+)'.*\n.*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", text)
    gemms = [f for f in found if "w8_gemm_kernel" in f[0]]
    assert len(gemms) == 5, found                         # token tiles 8, 16, 32, 64, 128
    for name, stack, stores, loads in found:
        assert (stack, stores, loads) == ("0", "0", "0"), (name, stack, stores, loads)
