"""Weight-only int8 generation on the H100: weight_quantize bit-exact against its restatement (oracle/weight_only_ref.py), the W8
GEMM against fp64 scale * (x @ q) at every preset's layer shapes, and the int8 models: lossless weights reproduce the bf16
model, the fused decode step equals the unfused composition, CUDA graphs equal eager, continuous batching equals each request
alone, no bf16 copy of a layer matrix is kept, and the error of real quantisation stays where it was measured."""
import functools

import pytest
import torch

from oracle import weight_only_ref as W
from test_continuous_batching_gpu import _compare, _oracle, _pages, _requests, _tiny, _weights
from test_decode_step_gpu import (DEFAULT_SPLIT_ROW_TOL, PRESETS, _gen, _lens, _nan, _seed, _with_pdl, assert_same_bits,
                                  assert_workspace_zero)
from test_kernels_at_scale_gpu import bf16_ulp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16

# Per-element allowance of the W8 GEMM's fp32 sums, times scale * (|x| @ |q|) (plus one bf16 ulp for the bf16 form).
# Measured on an H100 80GB HBM3 (700 W power limit) over every preset, matrix, row count, form and split below:
# c_need <= 1.09e-6.  c is ~5x the worst (the value SPLITK_C gives the bf16 split-K sums).
W8_C = 5.5e-6
# Relative error of the prefill logits of an int8 model against the bf16 model of the same random weights (init_random, std
# 0.02, two layers at the Llama-3.2-1B width), per row, measured on the same card: 4.4e-2 at worst.  The bound is ~4x that.
REAL_QUANT_LOGIT_REL = 0.18


def _ops():
    from paddlenlp_b200 import ops

    return ops


def _shapes(p):
    """(K, N) of the four fused layer matrices in [in, out] layout."""
    qkv_n = (p["nh"] + 2 * p["kvh"]) * p["d"]
    return {"qkv": (p["h"], qkv_n), "linear": (p["nh"] * p["d"], p["h"]), "ffn1": (p["h"], 2 * p["I"]), "ffn2": (p["I"], p["h"])}


def _planted_weight(K, N, seed):
    """bf16 W [K, N] ~ N(0, 0.02) with planted columns: outliers (x50 and one 3.0), an all-zero column, one whose quotients sit
    half way between integers (a = 127 s, values (j + 1/2) s), and a clamp column.  For a normal scale bf16 rounding moves
    a / scale by at most 2^-8 relative (a / scale <= 127.496); in the subnormal range the spacing is 2^-133 and a = 189 2^-133
    gives scale = bf16(1.488 2^-133) = 2^-133, so a / scale = 189 and q clamps to 127."""
    g = _gen(seed)
    w = (0.02 * torch.randn(K, N, generator=g, device=DEV)).to(BF16)
    cols = torch.randperm(N, generator=torch.Generator().manual_seed(seed))[:8].tolist()
    w[:, cols[0]] *= 50
    w[K // 3, cols[1]] = 3.0
    w[:, cols[2]] = 0
    # half-way column: s = 2^-10, a = 127 s (max entry), other entries (j + 1/2) s, all exact in bf16
    s = 2.0 ** -10
    j = torch.randint(-120, 120, (K,), generator=g, device=DEV).float()
    hw = ((j + 0.5) * s)
    hw[0] = 127 * s
    w[:, cols[3]] = hw.to(BF16)
    tiny = torch.randint(-189, 190, (K,), generator=g, device=DEV).double() * 2.0 ** -133
    tiny[1], tiny[2] = 189 * 2.0 ** -133, -189 * 2.0 ** -133
    w[:, cols[4]] = tiny.to(BF16)
    return w, cols


def _onehot_check(q_packed, scale, q_ref, s_ref, K, N):
    """The packed weights, read back through the fp32 GEMM form with one-hot rows of x: y[k] = scale * q[k, :] exactly."""
    x = torch.eye(K, dtype=BF16, device=DEV)
    ws = torch.zeros(K, N, dtype=torch.float32, device=DEV)
    _ops().call("b200_weight_only_gemm_f32", _ops().ptr(x), _ops().ptr(q_packed), _ops().ptr(scale), _ops().ptr(ws), K, N, K, K,
                0, _ops().stream_ptr())
    want = q_ref.float() * s_ref.float()[None, :]
    assert torch.equal(ws, want), f"one-hot rows: {int((ws != want).sum())} elements differ"


_QUANT = {}


def _quantized(preset, name):
    """W, packed q and scales of one preset matrix, with the oracle's q and scales (cached)."""
    key = (preset, name)
    if key not in _QUANT:
        K, N = _shapes(PRESETS[preset])[name]
        w, cols = _planted_weight(K, N, _seed(preset, name))
        q, s = _ops().weight_quantize(w)
        q_ref, s_ref = W.quantize(w)
        _QUANT[key] = (w, q, s, q_ref, s_ref, cols)
    return _QUANT[key]


@pytest.mark.parametrize("name", ["qkv", "linear", "ffn1", "ffn2"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_quantize_bit_exact(preset, name):
    w, q, s, q_ref, s_ref, cols = _quantized(preset, name)
    K, N = w.shape
    assert q.dtype == torch.int8 and q.shape == (N, K) and s.dtype == BF16 and s.shape == (N,)
    assert_same_bits(s, s_ref, f"{preset} {name}: scales")
    assert torch.equal(q.cpu(), W.pack(q_ref.cpu())), f"{preset} {name}: packed bytes"
    assert int(s_ref[cols[2]].float()) == 0 and int(q_ref[:, cols[2]].abs().max()) == 0           # zero column
    assert int(q_ref[:, cols[3]].abs().max()) == 127                                             # half-way column, to even
    hw = (q_ref[1:, cols[3]].int() % 2 != 0).sum()
    assert int(hw) == 0, "half-way quotients must round to even"
    assert int(q_ref[:, cols[4]].abs().max()) == 127 and float(s_ref[cols[4]]) == 2.0 ** -133       # clamped
    _onehot_check(q, s, q_ref, s_ref, K, N)


def _gemm_ref(x, q_ref, s_ref, bias):
    return W.linear_f64(x, q_ref, s_ref, bias), W.error_allowance(x, q_ref, s_ref)


# The TMA reduce-add of the fp32 partials flushes a subnormal sum to zero (the planted clamp column has a 2^-133 scale).
FLUSH = 2.0 ** -126


def _check(got, ref, mag, what, bf16_form):
    err = (got.double() - ref).abs()
    fixed = FLUSH + (bf16_ulp(ref) if bf16_form else 0)
    allow = W8_C * mag + fixed
    bad = ~(err <= allow)
    c_need = ((err - fixed).clamp_min(0) / (mag + 1e-300)).max().item()
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond c = {W8_C:.1e}, first at {i}: "
                             f"{got[tuple(i)].item()} vs {ref[tuple(i)].item()} (c_need {c_need:.2e})")


ROWS = (1, 5, 64, 128, 300, 4096)


@pytest.mark.parametrize("name", ["qkv", "qkv_bias", "linear", "ffn1", "ffn2"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_gemm_against_fp64(preset, name):
    _gemm_rows_against_fp64(preset, name, ROWS)


# pick_nt() in weight_only.cu takes token tiles of 8, 16, 32, 64 and 128 rows: every row count through 40 (each 8-, 16- and
# 32-row instantiation, full and partial), the partial 64- and 128-row tiles on both sides of their edges, and the first
# two-tile counts above 128 and 256.  Continuous batching feeds the GEMM every row count up to max_batch_size.
TILE_ROWS = tuple(range(1, 41)) + (63, 64, 65, 96, 127, 128, 129, 255, 256, 257)


@pytest.mark.parametrize("preset,name", [("llama3-8b", "ffn2"), ("qwen2-0.5b", "ffn2"), ("qwen2-0.5b", "qkv_bias")])
def test_gemm_every_token_tile(preset, name):
    """Llama-3-8B ffn2 has the longest K (14 336), Qwen2-0.5B ffn2 the narrowest N (896); its qkv carries a bias."""
    _gemm_rows_against_fp64(preset, name, TILE_ROWS)


def _gemm_rows_against_fp64(preset, name, rows):
    """Both forms at each row count, splits 0, 1 and 64 where K may split, against fp64: the bf16 form into a NaN-filled
    output whose 8 padding columns stay NaN, the fp32 form into a zero workspace whose spare bytes stay zero, and the split-K
    workspace zero after every bf16 call that may split."""
    o = _ops()
    mat = "qkv" if name == "qkv_bias" else name
    w, q, s, q_ref, s_ref, _ = _quantized(preset, mat)
    K, N = w.shape
    q_ref = q_ref.to(DEV)
    g = _gen(_seed(preset, name, "x"))
    bias = (0.5 * torch.randn(N, generator=g, device=DEV)) if name == "qkv_bias" else None
    for M in rows:
        x = torch.randn(M, K, generator=g, device=DEV).to(BF16)
        ref, mag = _gemm_ref(x, q_ref, s_ref, bias)
        splits = (0, 1, 64) if M <= o.SKINNY_M else (0,)
        for split in splits:
            what = f"{preset} {name} M={M} split={split}"
            # bf16 form into a NaN-filled output with 8 padding columns that must stay NaN
            out = _nan(M, N + 8)
            o.weight_only_linear(x, q, bias=bias, weight_scale=s, out=out[:, :N], split_k=split)
            _check(out[:, :N], ref, mag, what + " bf16", True)
            assert bool(out[:, N:].isnan().all()), what + ": wrote past N"
            if M <= o.SKINNY_M:
                assert_workspace_zero(o._workspaces[(x.device, "splitk")], what + ": splitk workspace")
        for split in (0, 1, 64):
            # fp32 form: a zero workspace with spare bytes past [M, N] that must stay zero
            ws = torch.zeros(M * N + 4096, dtype=torch.float32, device=DEV)
            o.call("b200_weight_only_gemm_f32", o.ptr(x), o.ptr(q), o.ptr(s), o.ptr(ws), M, N, K, K, split, o.stream_ptr())
            f32_ref = ref if bias is None else W.linear_f64(x, q_ref, s_ref)
            _check(ws[: M * N].view(M, N), f32_ref, mag, f"{preset} {name} M={M} split={split} f32", False)
            assert_workspace_zero(ws[M * N:], f"{preset} {name} M={M} split={split}: past [M, N]")


def test_weight_only_linear_argument_errors():
    o = _ops()
    x = torch.randn(4, 64, device=DEV).to(BF16)
    q, s = o.weight_quantize(torch.randn(64, 32, device=DEV).to(BF16))
    with pytest.raises(NotImplementedError):
        o.weight_quantize(torch.randn(64, 32, device=DEV).to(BF16), algo="weight_only_int4")
    with pytest.raises(ValueError):
        o.weight_quantize(torch.randn(64, 32, device=DEV).to(BF16), algo="int8")
    with pytest.raises(NotImplementedError):
        o.weight_only_linear(x, q, weight_scale=s, weight_dtype="int4")
    with pytest.raises(ValueError):
        o.weight_only_linear(torch.randn(4, 48, device=DEV).to(BF16), q, weight_scale=s)
    with pytest.raises(ValueError):
        o.weight_only_linear(torch.randn(300, 64, device=DEV).to(BF16), q, weight_scale=s, split_k=4)
    with pytest.raises(o._lib.B200Error, match="multiple of 16"):
        o.weight_quantize(torch.randn(40, 32, device=DEV).to(BF16))
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------
# Models
# ----------------------------------------------------------------------------------------------------------
def _config(preset, max_len, layers=2, vocab=256):
    import paddlenlp_b200.transformers as T

    p = PRESETS[preset]
    qwen = p["bias"]
    kw = dict(vocab_size=vocab, hidden_size=p["h"], intermediate_size=p["I"], num_hidden_layers=layers, num_attention_heads=p["nh"],
              num_key_value_heads=p["kvh"], rms_norm_eps=1e-6 if qwen else 1e-5, rope_theta=p["theta"],
              max_position_embeddings=max_len)
    return T.Qwen2Config(**kw) if qwen else T.LlamaConfig(**kw)


def _pair(preset, kind, max_len, seed):
    """A bf16 model and a weight_only_int8 model holding the same lossless weights w = q 2^-12 (every output channel holds
    +-127 2^-12, so quantisation is exact) and the same embeddings, norms, biases and head."""
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = _config(preset, max_len)
    kw = dict(block_attn=kind != "dense", append_attn=kind == "append_attn")
    mb = LlamaForCausalLMInferenceModel(cfg, **kw)
    mq = LlamaForCausalLMInferenceModel(cfg, quant_type="weight_only_int8", **kw)
    mb.init_random(seed, std=0.05)
    tb, tq = mb.transformer_block, mq.transformer_block
    g = _gen(seed + 1)
    for name in tb.MATRICES:
        for i in range(tb.L):
            rows, cols = tb.layer_matrix_shape(name)
            K, N = (cols, rows) if name == "qkv" else (rows, cols)
            q = torch.randint(-127, 128, (K, N), generator=g, device=DEV)
            at = torch.randint(0, K, (N,), generator=g, device=DEV)
            q[at, torch.arange(N, device=DEV)] = 127 * (1 - 2 * torch.randint(0, 2, (N,), generator=g, device=DEV))
            w = (q.float() * 2.0 ** -12).to(BF16)
            w = w.t() if name == "qkv" else w
            tb.set_layer_matrix(name, i, w)
            tq.set_layer_matrix(name, i, w)
    for i in range(tb.L):
        for s in (tb.ln_scales[i], tb.ffn_ln_scales[i]):
            s.copy_((1 + 0.1 * torch.randn(tb.h, generator=g, device=DEV)).to(BF16))
        if tb.qkv_biases[i] is not None:
            tb.qkv_biases[i].copy_((0.5 * torch.randn(tb.qkv_n, generator=g, device=DEV)).to(BF16))
        tq.ln_scales[i].copy_(tb.ln_scales[i])
        tq.ffn_ln_scales[i].copy_(tb.ffn_ln_scales[i])
        if tb.qkv_biases[i] is not None:
            tq.qkv_biases[i].copy_(tb.qkv_biases[i])
    for a, b in ((mq.embed_tokens, mb.embed_tokens), (mq.norm_weight, mb.norm_weight), (mq.lm_head_weight, mb.lm_head_weight)):
        a.copy_(b)
    tb.weights_changed()
    tq.weights_changed()
    return mb, mq


def _rel_rows(a, b):
    a, b = a.double().reshape(a.shape[0], -1), b.double().reshape(b.shape[0], -1)
    return ((a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-30))


@pytest.mark.parametrize("kind", ["dense", "paged", "append_attn"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_lossless_weights_match_bf16(preset, kind):
    B, S, max_len = 4, 37, 128
    mb, mq = _pair(preset, kind, max_len, seed=_seed(preset, kind) % 1000)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(1, 256, (B, S), generator=g).to(DEV)
    enc = torch.tensor([S, 20, 1, 33], dtype=torch.int32, device=DEV)
    cb, cq = mb.allocate_caches(B, max_len), mq.allocate_caches(B, max_len)
    if kind != "dense":
        mq.block_tables = mb.block_tables.clone()
    lb, lq = mb._prefill(ids, enc, cb), mq._prefill(ids, enc, cq)
    worst = _rel_rows(lq, lb).max().item()
    compared = 0
    lens = enc.clone()
    for step in range(4):
        assert worst <= DEFAULT_SPLIT_ROW_TOL, (preset, kind, step, worst)
        top = lb.float().topk(2, dim=-1)
        margin = (top.values[:, 0] - top.values[:, 1]) / lb.float().abs().amax(dim=-1)
        tok_b, tok_q = lb.float().argmax(-1), lq.float().argmax(-1)
        sure = margin > 2 * DEFAULT_SPLIT_ROW_TOL
        assert torch.equal(tok_b[sure], tok_q[sure]), (preset, kind, step)
        compared += int(sure.sum())
        if step == 3:
            break
        lb, lq = mb._decode(tok_b, lens, cb), mq._decode(tok_b, lens, cq)
        lens = lens + 1
        worst = _rel_rows(lq, lb).max().item()
    assert compared > 0


W8_LAYER_WIDTHS = ("llama3-8b", "qwen2-1.5b")


@pytest.mark.parametrize("pdl", [False, True])
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("preset", W8_LAYER_WIDTHS)
def test_fused_w8_decode_step_equals_unfused(preset, paged, pdl, monkeypatch):
    """split_k = 1: the fused int8 decode step (fp32 workspaces into rope-append, add_rmsnorm and swiglu_fwd_f32) equals
    weight_only_linear -> decode_rope_append -> decode_attention -> ... bit for bit: hidden states and caches."""
    _fused_w8_vs_unfused(preset, paged, pdl, 64, monkeypatch)


@pytest.mark.parametrize("B", [13, 29])
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("preset", W8_LAYER_WIDTHS)
def test_fused_w8_decode_step_equals_unfused_16_and_32_row_tiles(preset, paged, B, monkeypatch):
    """The same at batch 13 and 29, which the W8 GEMM runs in 16- and 32-row token tiles."""
    _fused_w8_vs_unfused(preset, paged, True, B, monkeypatch)


def _fused_w8_vs_unfused(preset, paged, pdl, B, monkeypatch):
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    o = _ops()
    monkeypatch.setattr(o, "weight_only_linear_f32", functools.partial(o.weight_only_linear_f32, split_k=1))
    monkeypatch.setattr(o, "weight_only_linear", functools.partial(o.weight_only_linear, split_k=1))
    max_len = 256
    m = LlamaForCausalLMInferenceModel(_config(preset, max_len), block_attn=paged, quant_type="weight_only_int8")
    m.init_random(7 + paged)
    t = m.transformer_block
    g = _gen(8)
    for i in range(t.L):
        if t.qkv_biases[i] is not None:
            t.qkv_biases[i].copy_((0.5 * torch.randn(t.qkv_n, generator=g, device=DEV)).to(BF16))
    t.weights_changed()
    caches = m.allocate_caches(B, max_len)
    for c in caches:
        c.copy_(torch.randn(c.shape, generator=g, device=DEV).to(BF16))
    lens = _lens(B, max_len, 11)
    src = torch.randn(B, t.h, generator=_gen(12), device=DEV).to(BF16)
    kw = m._cache_kw()
    fused_c, unf_c = [c.clone() for c in caches], [c.clone() for c in caches]
    with _with_pdl(pdl):
        h_fused = t(src, fused_c, B=B, S=1, seq_lens_decoder=lens, time_step=0, **kw)
        # unfused: the same block with the fused branch switched off (decode rows above SKINNY_M take the unfused path)
        monkeypatch.setattr(t, "SKINNY_M", 0)
        h_unf = t(src, unf_c, B=B, S=1, seq_lens_decoder=lens, time_step=0, **kw)
        torch.cuda.synchronize()
    what = f"{preset} {'paged' if paged else 'dense'} pdl={pdl} B={B}"
    assert bool(torch.isfinite(h_unf.float()).all())
    assert_same_bits(h_fused, h_unf, f"{what}: hidden states")
    for j, (a, b) in enumerate(zip(fused_c, unf_c)):
        assert_same_bits(a, b, f"{what}: cache tensor {j}")
    for tag in ("splitk_qkv", "splitk_h", "splitk_ffn1"):
        assert_workspace_zero(o._workspaces[(src.device, tag)], f"{what}: {tag}")


def _lossless_sd(w):
    """The reference weights with every layer matrix made exactly representable by int8 + bf16 scale: per output column,
    q = rint(w / 2^e) with its largest entry set to +-127, w = q 2^e."""
    out = dict(w)
    for k, v in w.items():
        if ".layers." in k and k.endswith("proj.weight"):
            a = v.abs().amax(dim=0).clamp_min(1e-30)
            e = torch.ceil(torch.log2(a / 127))
            q = torch.round(v / 2 ** e).clamp(-127, 127)
            at = v.abs().argmax(dim=0)
            cols = torch.arange(v.shape[1])
            q[at, cols] = 127 * torch.sign(v[at, cols])
            out[k] = q * 2 ** e
    return out


_LOSSLESS = {}


def _w8_tiny(model_type, block_attn=True, append_attn=True, block_size=32):
    """The continuous-batching suite's tiny model with its weights made lossless, as a weight_only_int8 model whose config
    carries the quant_type (as the reference predictor sets it)."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = _tiny(model_type)
    if model_type not in _LOSSLESS:
        _LOSSLESS[model_type] = _lossless_sd(_weights(cfg))
    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    c = T.Qwen2Config(**kw) if model_type == "qwen2" else T.LlamaConfig(**kw)
    c.quant_type = "weight_only_int8"
    m = LlamaForCausalLMInferenceModel(c, block_attn=block_attn, append_attn=append_attn, block_size=block_size)
    assert m.transformer_block.config.quant_type == "weight_only_int8"
    m.set_state_dict(_LOSSLESS[model_type])
    return cfg, m


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_continuous_generate_matches_each_request_alone(model_type, monkeypatch):
    """A mixed queue through continuous batching gives every request the greedy tokens the uncached oracle gives it alone
    (lossless int8 weights: the oracle's weights are the model's)."""
    import test_continuous_batching_gpu as cb

    cfg, m = _w8_tiny(model_type)
    reqs = _requests()
    monkeypatch.setattr(cb, "_weights", lambda c: _LOSSLESS[model_type])
    ref = _oracle(model_type, reqs, "w8-lossless")
    nb = 4 * 11 * _pages(reqs, 32)
    outs, stats = m.continuous_generate(reqs, max_batch_size=4, num_blocks=nb)
    assert _compare(outs, reqs, ref) >= 20
    assert stats["mixed_steps"] >= 2


@pytest.mark.parametrize("block_attn", [False, True])
def test_generate_graph_equals_eager(block_attn):
    _, m = _w8_tiny("qwen2", block_attn=block_attn, append_attn=False)
    ids = torch.randint(1, 512, (3, 17), generator=torch.Generator().manual_seed(1)).to(DEV)
    a = m.generate(ids, max_length=24, use_cuda_graph=True)[0]
    b = m.generate(ids, max_length=24, use_cuda_graph=False)[0]
    assert torch.equal(a, b)


def test_memory_int8_only_and_set_state_dict_peak():
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    preset = "llama3-8b"
    cfg = _config(preset, 128)
    m = LlamaForCausalLMInferenceModel(cfg, quant_type="weight_only_int8")
    t = m.transformer_block
    for name in t.MATRICES:
        rows, cols = t.layer_matrix_shape(name)
        for i in range(t.L):
            wq, sc = getattr(t, name + "_weights")[i], getattr(t, name + "_weights_scale")[i]
            assert wq.dtype == torch.int8 and wq.numel() == rows * cols
            assert sc.dtype == BF16 and sc.numel() == wq.shape[0]
    sizes = {t.layer_matrix_shape(n) for n in t.MATRICES} | {t.layer_matrix_shape(n)[::-1] for n in t.MATRICES}
    for k, v in vars(t).items():
        for x in (v if isinstance(v, (list, tuple)) else [v]):
            if isinstance(x, torch.Tensor) and x.dtype == BF16:
                assert tuple(x.shape) not in sizes, f"bf16 layer matrix reachable as {k}"
    # a training-format state dict on the host; the device stages one bf16 fused matrix at a time
    g = torch.Generator().manual_seed(0)
    p = PRESETS[preset]
    h, I, kvd = p["h"], p["I"], p["kvh"] * p["d"]
    sd = {"llama.embed_tokens.weight": torch.randn(256, h, generator=g).to(BF16), "llama.norm.weight": torch.ones(h, dtype=BF16),
          "lm_head.weight": torch.randn(h, 256, generator=g).to(BF16)}
    for i in range(t.L):
        lp = f"llama.layers.{i}."
        for n, shape in (("self_attn.q_proj", (h, h)), ("self_attn.k_proj", (h, kvd)), ("self_attn.v_proj", (h, kvd)),
                         ("self_attn.o_proj", (h, h)), ("mlp.gate_proj", (h, I)), ("mlp.up_proj", (h, I)), ("mlp.down_proj", (I, h))):
            sd[lp + n + ".weight"] = (0.02 * torch.randn(*shape, generator=g)).to(BF16)
        sd[lp + "input_layernorm.weight"] = torch.ones(h, dtype=BF16)
        sd[lp + "post_attention_layernorm.weight"] = torch.ones(h, dtype=BF16)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m.set_state_dict(sd)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    largest = max(r * c for r, c in (t.layer_matrix_shape(n) for n in t.MATRICES)) * 2
    assert extra < 2 * largest, (extra, largest)


def test_real_quantisation_error():
    """Random (not lossless) weights: the int8 model's prefill logits against the bf16 model of the same seed."""
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = _config("llama3.2-1b", 128)
    mb = LlamaForCausalLMInferenceModel(cfg)
    mq = LlamaForCausalLMInferenceModel(cfg, quant_type="weight_only_int8")
    mb.init_random(3)
    mq.init_random(3)
    assert torch.equal(mb.embed_tokens, mq.embed_tokens) and torch.equal(mb.lm_head_weight, mq.lm_head_weight)
    ids = torch.randint(1, 256, (4, 64), generator=torch.Generator().manual_seed(2)).to(DEV)
    rel = _rel_rows(mq.forward_logits_prefill(ids).flatten(0, 1), mb.forward_logits_prefill(ids).flatten(0, 1)).max().item()
    assert 0 < rel <= REAL_QUANT_LOGIT_REL, rel
