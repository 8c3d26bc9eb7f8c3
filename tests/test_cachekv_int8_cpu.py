"""Static int8 KV cache without a GPU: the restatement's properties (oracle/cachekv_int8_ref.py), the scale file's loading,
config validation, the C-ABI's argument errors (returned before any device work) and the ptxas log of the new instantiations."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from oracle import cachekv_int8_ref as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16


def test_ties_after_the_bf16_product_go_to_even():
    """Half-way products built from exactly representable bf16 values: s = 1, x = k + 0.5 (bf16 holds every half integer up
    to 128), and s = 0.5 with x = odd integers."""
    x = torch.tensor([0.5, 1.5, 2.5, 3.5, -0.5, -1.5, -2.5, 64.5, 65.5, 100.5, 125.5, 126.5], dtype=BF16)
    assert torch.equal(x.double(), torch.tensor([0.5, 1.5, 2.5, 3.5, -0.5, -1.5, -2.5, 64.5, 65.5, 100.5, 125.5, 126.5],
                                                dtype=torch.float64))
    u = C.quantize(x, torch.tensor(1.0, dtype=BF16)).int() - 128
    assert u.tolist() == [0, 2, 2, 4, 0, -2, -2, 64, 66, 100, 126, 126]
    y = torch.tensor([1, 3, 5, 7, -1, -3, 129, 131, 251], dtype=BF16)
    u = C.quantize(y, torch.tensor(0.5, dtype=BF16)).int() - 128
    assert u.tolist() == [0, 2, 2, 4, 0, -2, 64, 66, 126]


def test_bf16_rounding_of_the_product_comes_first():
    """The product is rounded to bf16 before the integer rounding.  x = 3.140625 and 3.171875 are bf16; s = 32.25 (bf16):
    s x = 101.2851... and 102.2968..., which bf16 (spacing 0.5 in [64, 128)) rounds to 101.5 and 102.5, and those ties go to
    the even integers 102 and 102; rounding the exact products would give 101 and 102."""
    x = torch.tensor([3.140625, 3.171875], dtype=BF16)
    s = torch.tensor(32.25, dtype=BF16)
    assert x.double().tolist() == [3.140625, 3.171875] and float(s) == 32.25
    exact = x.double() * 32.25
    assert (x.float() * s.float()).to(BF16).float().tolist() == [101.5, 102.5]
    u = C.quantize(x, s).int() - 128
    assert u.tolist() == [102, 102]
    assert torch.round(exact).int().tolist() == [101, 102]


def test_clamp_at_127():
    x = torch.tensor([126.0, 127.0, 128.0, 1000.0, -127.0, -128.0, -3e38, 3e38], dtype=BF16)
    u = C.quantize(x, torch.tensor(1.0, dtype=BF16)).int() - 128
    assert u.tolist() == [126, 127, 127, 127, -127, -127, -127, 127]
    assert int(C.quantize(x, torch.tensor(1.0, dtype=BF16)).min()) == 1          # byte 0 is never produced


def test_offset_128_round_trips_integers_and_zero():
    k = torch.arange(-127, 128, dtype=torch.float64)
    u = C.quantize(k.to(BF16), torch.tensor(1.0, dtype=BF16))
    assert torch.equal(u.int(), (k + 128).int())
    assert torch.equal(C.dequantize(u, torch.tensor(1.0, dtype=BF16)), k)
    assert int(C.quantize(torch.zeros(3, dtype=BF16), torch.tensor(0.37, dtype=BF16))[0]) == 128


def test_round_trip_error_within_half_a_step():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(4, 2, 64, generator=g) * 3).to(BF16)
    a = x.double().abs().amax(dim=(0, 2))
    s, o = C.scales_from_absmax(a)
    u = C.quantize(x, s.view(1, 2, 1))
    xh = C.dequantize(u, o.view(1, 2, 1))
    step = o.double().view(1, 2, 1)
    # half a step of the integer rounding, a quarter step of the bf16 product rounding (spacing 0.5 in [64, 128)), and the
    # bf16 scales: s * o is 1 within 2^-8, up to half a step at |s x| = 127
    assert bool(((xh - x.double()).abs() <= step * (0.5 + 0.25 + 127 * 2.0 ** -8) + 1e-12).all())


def _json(L, nh, seed=0, prefix="llama"):
    g = torch.Generator().manual_seed(seed)
    d = {}
    for i in range(L):
        for kind in ("k", "v"):
            d[f"{prefix}.layers.{i}.self_attn.cache{kind}_matmul.activation_quanter"] = (torch.rand(nh, generator=g) * 9 + 0.5).tolist()
    return d


@pytest.mark.parametrize("nh,kvh", [(4, 4), (8, 2), (6, 1)])
def test_scale_json_keeps_every_group_th_value(nh, kvh):
    d = _json(3, nh)
    k, v = C.absmax_from_json(d, "llama", 3, nh, kvh)
    g = nh // kvh
    for i in range(3):
        assert k[i].tolist() == d[f"llama.layers.{i}.self_attn.cachek_matmul.activation_quanter"][::g]
        assert v[i].tolist() == d[f"llama.layers.{i}.self_attn.cachev_matmul.activation_quanter"][::g]
    s, o = C.scales_from_absmax(k)
    assert s.dtype == BF16 and o.dtype == BF16
    assert torch.equal(s, (127.0 / k).to(BF16)) and torch.equal(o, (k / 127.0).to(BF16))


def test_bad_absmax_is_refused():
    for bad in ([1.0, 0.0], [1.0, -2.0], [float("nan"), 1.0], [float("inf"), 1.0]):
        with pytest.raises(ValueError):
            C.scales_from_absmax(bad)


def test_calibration_absmax_ignores_zero_pages():
    cache = torch.zeros(6, 2, 32, 16, dtype=BF16)
    cache[2, 0, 3, 5] = -7.5
    cache[4, 1, 0, 0] = 0.25
    assert C.absmax_of_cache(cache).tolist() == [7.5, 0.25]


def test_config_validation():
    from paddlenlp_b200.experimental.transformers import FusedMultiTransformerConfig

    kw = dict(embed_dim=256, num_heads=2, dim_feedforward=512)
    assert FusedMultiTransformerConfig(**kw).cachekv_int8_type is None
    assert FusedMultiTransformerConfig(cachekv_int8_type="static", **kw).cachekv_int8_type == "static"
    with pytest.raises(NotImplementedError, match="dynamic"):
        FusedMultiTransformerConfig(cachekv_int8_type="dynamic", **kw)
    with pytest.raises(ValueError):
        FusedMultiTransformerConfig(cachekv_int8_type="int8", **kw)


def test_static_on_the_dense_cache_names_block_attn():
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel
    from paddlenlp_b200.transformers import LlamaConfig

    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=2,
                      num_key_value_heads=1)
    with pytest.raises(NotImplementedError, match="block_attn=True"):
        LlamaForCausalLMInferenceModel(cfg, cachekv_int8_type="static")
    with pytest.raises(NotImplementedError, match="dynamic"):
        LlamaForCausalLMInferenceModel(cfg, cachekv_int8_type="dynamic")
    cfg.cachekv_int8_type = "static"                      # read from the config when the argument is None
    with pytest.raises(NotImplementedError, match="block_attn=True"):
        LlamaForCausalLMInferenceModel(cfg)


def test_abi_argument_errors():
    """Each new entry point refuses null scales, bad shapes and bad block sizes with an argument error (< 0) before any
    device work, so no GPU is needed."""
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    a = ctypes.c_void_p(0x10000)

    def write(ks=a, vs=a, bs=64, d=128, kvh=2):
        return lib.b200_write_cache_kv_paged_c8(a, a, a, a, ks, vs, a, 2, 4, 4, kvh, d, bs, 4, (4 + 2 * kvh) * d, None)

    def rope(ks=a, vs=a, bs=64, d=128, kvh=2):
        return lib.b200_decode_rope_append_paged_c8(a, None, None, a, a, a, ks, vs, a, a, a, 2, 4, kvh, d, bs, 4,
                                                    (4 + 2 * kvh) * d, None)

    def dec(ko=a, vo=a, bs=64, d=128, kvh=2, nh=4):
        return lib.b200_decode_attention_paged_c8(a, a, a, a, ko, vo, a, a, None, 2, nh, kvh, d, 16, bs, 4, (nh + 2 * kvh) * d,
                                                  0.1, 1, None)

    def app(ks=a, vs=a, ko=a, vo=a, bs=64, d=128, kvh=2, nh=4, qkv=a):
        return lib.b200_append_attention_c8(qkv, a, a, ks, vs, ko, vo, a, a, a, a, a, a, a, a, a, 2, 8, 4, nh, kvh, d, 16, bs, 4,
                                            256, (nh + 2 * kvh) * d, nh * d, 0.1, 1, None)

    cases = [(lambda: write(ks=None), "cache_k_scale"), (lambda: write(vs=None), "cache_k_scale"),
             (lambda: write(bs=16), "block_size"), (lambda: write(d=72), "multiple of 16"),
             (lambda: rope(ks=None), "cache_k_scale"), (lambda: rope(bs=256), "block_size"),
             (lambda: dec(ko=None), "out_scale"), (lambda: dec(vo=None), "out_scale"), (lambda: dec(bs=48), "block_size"),
             (lambda: dec(d=96), "head_dim"), (lambda: dec(nh=18), "GQA"),
             (lambda: app(ks=None), "cache_k_scale"), (lambda: app(vo=None), "out_scale"), (lambda: app(bs=8), "block_size"),
             (lambda: app(d=96), "head_dim"), (lambda: app(qkv=None), "null pointer")]
    for fn, msg in cases:
        assert fn() < 0, msg
        assert msg in lib.b200_last_error().decode(), (msg, lib.b200_last_error())


def _ptxas(name):
    log = os.path.join(ROOT, "paddlenlp_b200", "build", name + ".o.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log: the library was not built in this tree")
    text = open(log).read()
    found = re.findall(r"Compiling entry function '(\w+)'.*\n(?:.*\n)?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\n.*Used (\d+) registers", text)
    names = subprocess.run(["c++filt"], input="\n".join(f[0] for f in found), capture_output=True, text=True).stdout.split("\n")
    return [(n,) + tuple(int(x) for x in f[1:]) for n, f in zip(names, found)]


# registers per thread of the uint8 decode kernel at d = 128, G = 1..8, as ptxas (CUDA 12.9) reported them
DECODE_C8_REGS_D128 = {1: 71, 2: 100, 3: 128, 4: 152, 5: 177, 6: 207, 7: 238, 8: 254}


def test_c8_decode_kernel_ptxas_log():
    """Every uint8 instantiation of the bulk decode kernel: no spills and no stack frame beyond the bf16 twin's (16 bytes, the
    mbarrier wait loop); at G <= 4 it fits the 2-CTA budget (<= 204 registers)."""
    found = _ptxas("decode_attn_tc")
    c8 = [f for f in found if "decode_attention_bulk_kernel" in f[0] and "unsigned char" in f[0]]
    bf = {re.sub(r"unsigned char", "__nv_bfloat16", f[0]): f for f in c8}
    twins = {f[0]: f for f in found if f[0] in bf}
    assert len(c8) == 16, c8                                   # d 64 / 128 x G 1..8, paged only
    for name, stack, stores, loads, regs in c8:
        twin = twins[re.sub(r"unsigned char", "__nv_bfloat16", name)]
        assert (stores, loads) == (0, 0), name
        assert stack <= twin[1], (name, stack, twin[1])
        g = int(re.search(r"<(\d+), (\d+), true", name).group(2))
        if g <= 4:
            assert regs <= 204, (name, regs)
        if "<128," in name:
            assert regs == DECODE_C8_REGS_D128[g], (name, regs)


def test_c8_prefill_and_writer_ptxas_log():
    fa = [f for f in _ptxas("fa_fwd") if "fa_fwd_kernel" in f[0]]
    c8 = [f for f in fa if re.search(r"fa_fwd_kernel<\d+, 3>", f[0])]
    assert len(c8) == 2, fa
    gen = [f for f in _ptxas("generation") if "unsigned char" in f[0]]
    assert len(gen) == 3, gen                                  # write_cache_kv, decode_rope_append, append_rope_write
    for name, stack, stores, loads, regs in c8 + gen:
        assert (stack, stores, loads) == (0, 0, 0), name
