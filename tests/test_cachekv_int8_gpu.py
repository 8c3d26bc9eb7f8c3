"""Static int8 paged KV cache on the H100: every cache writer bit-exact against the restatement (oracle/cachekv_int8_ref.py)
applied to the bf16 values its bf16 twin stores, decode attention and append_attention's prompt rows against fp64 attention over
the dequantised pages, and the int8-cache models: fused decode step against the append_attention step, CUDA graph against
eager, continuous batching against each request alone, half the cache bytes, and the logit error of a calibrated int8 cache."""
import math

import pytest
import torch

from oracle import cachekv_int8_ref as C
from test_continuous_batching_gpu import _requests, _tiny, _weights
from test_decode_attention_at_scale_gpu import (DECODE_C, HEAD_TOL, PREFILL_C, PREFILL_HEAD_TOL, assert_attention_close)
from test_decode_step_gpu import DEFAULT_SPLIT_ROW_TOL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16
U8 = torch.uint8
# Relative error of the decode logits of a two-layer tiny model with a calibrated int8 cache against the same model with a
# bf16 cache, per row, teacher-forced over 24 decode steps after a 40-token prompt.  Measured on an H100 80GB HBM3 (700 W
# power limit): at most 4.85e-2 (llama) and 4.27e-2 (qwen2).  The bound is ~3x that.
INT8_CACHE_LOGIT_REL = 0.15
# The attention checks reuse the bf16 kernels' tolerances (tests/test_decode_attention_at_scale_gpu.py).  Measured on the same
# card over every case below: decode c_need <= 2.5e-7 (DECODE_C 4e-7), (sequence, head) error <= 2.2e-3 (HEAD_TOL 4e-3);
# append_attention prompt rows c_need <= 2.3e-3 (PREFILL_C 1e-2), (row, head) error <= 3.3e-3 (PREFILL_HEAD_TOL 6e-3).
# Continuous batching against each request alone is compared token for token with bf16 layer weights.  With int8 weights
# the W8 GEMM splits K by the number of rows, so rows batched differently are summed in another order and a near-tie can
# flip a token (measured: requests diverged after as few as 13 equal tokens); that composition is checked through the
# fused step, CUDA graphs and the pool's bookkeeping instead.


def _ops():
    from paddlenlp_b200 import ops

    return ops


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _scales(kvh, seed, absmax=None):
    """Per-head scales from absmax values in [2, 6) (or the given ones): s, o bf16 [kvh]."""
    if absmax is None:
        absmax = 2 + 4 * torch.rand(kvh, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    s, o = C.scales_from_absmax(absmax)
    return s.to(DEV), o.to(DEV)


def _tables(B, per_seq, nb, seed):
    """Block tables of distinct pages in shuffled order (pages out of order exercise the table lookup)."""
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))[:B * per_seq]
    return perm.view(B, per_seq).to(torch.int32).to(DEV)


def _planted_v(qkv, nh, kvh, d, rows):
    """Plant ties (k + 0.5 at s = 1), clamps (+-300) and zeros into the V columns of kv head 0 of the given token rows."""
    col0 = (nh + kvh) * d
    vals = torch.tensor([0.5, 1.5, 2.5, -2.5, 100.5, 101.5, 126.5, 127.5, 300.0, -300.0, 0.0, -0.0, 64.5, -65.5, 3.5, 4.5],
                        dtype=BF16, device=DEV)
    for r in rows:
        qkv[r, col0:col0 + d] = vals.repeat(d // 16)


def _unit_head0(s, o):
    s[0], o[0] = 1.0, 1.0                                  # head 0: the planted products are the planted values


def _check_quantised(c8, bf, s, what):
    """The uint8 cache equals the restatement's quantisation of the bf16 twin's cache, everywhere."""
    want = C.quantize(bf.cpu(), s.cpu().view(1, -1, 1, 1))
    got = c8.cpu()
    diff = got != want
    if bool(diff.any()):
        i = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} bytes differ, first at {i}: {int(got[tuple(i)])} vs {int(want[tuple(i)])} "
                             f"(bf16 {bf[tuple(i)].item()}, s {s[i[1]].item()})")


def _pair_caches(nb, kvh, bs, d, s_k, s_v, seed):
    """A random bf16 cache pair and its quantisation: the state both writers start from."""
    g = _g(seed)
    kb = torch.randn(nb, kvh, bs, d, generator=g, device=DEV).to(BF16)
    vb = torch.randn(nb, kvh, bs, d, generator=g, device=DEV).to(BF16)
    k8 = C.quantize(kb.cpu(), s_k.cpu().view(1, -1, 1, 1)).to(DEV)
    v8 = C.quantize(vb.cpu(), s_v.cpu().view(1, -1, 1, 1)).to(DEV)
    return kb, vb, k8, v8


@pytest.mark.parametrize("d,bs", [(128, 64), (64, 32), (128, 128)])
def test_writers_bit_exact(d, bs):
    """write_cache_kv_paged, decode_rope_append_paged (bf16 and fp32-workspace forms) and append_attention on a batch that
    mixes a fresh prompt, a chunk over a cached prefix, decode rows and an idle slot: the uint8 cache is the restatement of the
    bf16 values the bf16 twin writes, byte for byte, with planted ties, clamps and zeros."""
    o = _ops()
    nh, kvh = 4, 2
    ld = (nh + 2 * kvh) * d
    B, per_seq = 4, 6
    nb = B * per_seq + 3
    bt = _tables(B, per_seq, nb, 1)
    s_k, o_k = _scales(kvh, 2)
    s_v, o_v = _scales(kvh, 3)
    _unit_head0(s_v, o_v)
    cos, sin = o.rope_tables(d, per_seq * bs + 8, 10000.0, DEV)
    g = _g(4)

    # prefill fill
    S = 70
    qkv = (3 * torch.randn(B * S, ld, generator=g, device=DEV)).to(BF16)
    _planted_v(qkv, nh, kvh, d, range(0, B * S, 7))
    lens = torch.tensor([70, 1, 33, 64], dtype=torch.int32, device=DEV)
    kb, vb, k8, v8 = _pair_caches(nb, kvh, bs, d, s_k, s_v, 5)
    o.write_cache_kv_paged(qkv, kb, vb, bt, lens, B, S, nh)
    o.write_cache_kv_paged(qkv, k8, v8, bt, lens, B, S, nh, cache_k_scale=s_k, cache_v_scale=s_v)
    torch.cuda.synchronize()
    _check_quantised(k8, kb, s_k, "write_cache_kv_paged K")
    _check_quantised(v8, vb, s_v, "write_cache_kv_paged V")

    # decode append, bf16 form and fp32-workspace form
    pos = torch.tensor([0, 63, 64, per_seq * bs - 1], dtype=torch.int32, device=DEV)
    for form in ("bf16", "f32"):
        kb, vb, k8, v8 = _pair_caches(nb, kvh, bs, d, s_k, s_v, 6)
        if form == "bf16":
            x = (3 * torch.randn(B, ld, generator=g, device=DEV)).to(BF16)
            _planted_v(x, nh, kvh, d, range(B))
            xa, xb = x.clone(), x.clone()
            o.decode_rope_append_paged(xa, kb, vb, bt, cos, sin, pos, nh)
            o.decode_rope_append_paged(xb, k8, v8, bt, cos, sin, pos, nh, cache_k_scale=s_k, cache_v_scale=s_v)
        else:
            acc = 3 * torch.randn(B, ld, generator=g, device=DEV)
            acc[:, (nh + kvh) * d:(nh + kvh) * d + 16] = torch.tensor([0.5, 1.5, 2.5, 126.5, 127.5, 300.0, 0.0, -2.5] * 2,
                                                                      device=DEV)
            bias = torch.randn(ld, generator=g, device=DEV).to(BF16).float()
            bias[(nh + kvh) * d:(nh + kvh) * d + 16] = 0
            a1, a2 = acc.clone(), acc.clone()
            xa = o.decode_rope_append_paged(None, kb, vb, bt, cos, sin, pos, nh, acc_f32=a1, bias=bias)
            xb = o.decode_rope_append_paged(None, k8, v8, bt, cos, sin, pos, nh, acc_f32=a2, bias=bias, cache_k_scale=s_k,
                                            cache_v_scale=s_v)
            torch.cuda.synchronize()
            assert not bool(a2.any()), "the fp32 workspace is handed back zeroed"
        torch.cuda.synchronize()
        assert torch.equal(xa, xb), f"decode_rope_append_paged ({form}): the rotated projection differs"
        _check_quantised(k8, kb, s_k, f"decode_rope_append_paged ({form}) K")
        _check_quantised(v8, vb, s_v, f"decode_rope_append_paged ({form}) V")

    # append_attention over a mixed batch: fresh prompt, chunk over a cached prefix, decode row, idle slot
    B2 = 4
    enc = torch.tensor([45, 30, 0, 0], dtype=torch.int32, device=DEV)
    dec = torch.tensor([0, 100, 77, 0], dtype=torch.int32, device=DEV)
    this = torch.tensor([45, 30, 1, 0], dtype=torch.int32, device=DEV)
    cu = torch.tensor([0, 45, 75, 76, 76], dtype=torch.int32, device=DEV)
    T = 76
    x = (3 * torch.randn(T, ld, generator=g, device=DEV)).to(BF16)
    _planted_v(x, nh, kvh, d, range(0, T, 5))
    kb, vb, k8, v8 = _pair_caches(nb, kvh, bs, d, s_k, s_v, 7)
    xa, xb = x.clone(), x.clone()
    o.append_attention(xa, kb, vb, enc, dec, this, cu, bt[:B2].contiguous(), cos, sin, nh, max_q_len=45)
    o.append_attention(xb, k8, v8, enc, dec, this, cu, bt[:B2].contiguous(), cos, sin, nh, max_q_len=45, cache_k_scale=s_k,
                       cache_v_scale=s_v, cache_k_out_scale=o_k, cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    assert torch.equal(xa, xb), "append_attention: the rotated projection differs"
    _check_quantised(k8, kb, s_k, "append_attention K")
    _check_quantised(v8, vb, s_v, "append_attention V")


def _random_c8(nb, kvh, bs, d, seed):
    g = torch.Generator().manual_seed(seed)
    k8 = torch.randint(1, 256, (nb, kvh, bs, d), generator=g, dtype=torch.int32).to(U8)
    v8 = torch.randint(1, 256, (nb, kvh, bs, d), generator=g, dtype=torch.int32).to(U8)
    return k8.to(DEV), v8.to(DEV)


@pytest.mark.parametrize("splits", ["one", "auto"])
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("G", [1, 2, 3, 4, 5, 6, 7, 8])
def test_decode_attention_against_fp64(G, d, bs, splits):
    """Per (sequence, head) against fp64 attention over K = (u - 128) o_k, V = (u - 128) o_v: lengths 1 (no history), ending
    inside a chunk and spanning pages, split-KV on and off."""
    o = _ops()
    kvh = 2
    nh = kvh * G
    B, per_seq = 12, (1100 + bs - 1) // bs
    nb = B * per_seq + 2
    bt = _tables(B, per_seq, nb, 11 + G)
    k8, v8 = _random_c8(nb, kvh, bs, d, 12 + G + d)
    s_k, o_k = _scales(kvh, 13, absmax=torch.tensor([2.0, 5.5], dtype=torch.float64))
    s_v, o_v = _scales(kvh, 14, absmax=torch.tensor([3.0, 0.75], dtype=torch.float64))
    lens = torch.tensor([0, 1, 30, 31, 33, 63, 64, 65, 127, 500, 1000, 1098], dtype=torch.int32)
    ld = (nh + 2 * kvh) * d
    qkv = torch.randn(B, ld, generator=_g(15), device=DEV).to(BF16)
    out = torch.full((B, nh * d), float("nan"), dtype=BF16, device=DEV)
    ns = 1 if splits == "one" else 0
    o.decode_attention_paged(qkv, k8, v8, bt, lens.to(DEV), nh, out=out, num_splits=ns, cache_k_out_scale=o_k,
                             cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    if splits == "auto":
        assert o._decode_splits(B, kvh, per_seq * bs) > 1
    kd, vd = C.dequantize(k8, o_k.view(1, -1, 1, 1)), C.dequantize(v8, o_v.view(1, -1, 1, 1))
    q = qkv[:, :nh * d].view(B, nh, d)

    def rows(n):
        L = int(lens[n]) + 1
        return C.gather_pages(kd, bt[n], L), C.gather_pages(vd, bt[n], L)

    assert_attention_close(out, q, rows, c=DECODE_C, head_tol=HEAD_TOL, what=f"c8 decode G={G} d={d} bs={bs} {splits}")


@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("d,G", [(128, 4), (64, 8), (128, 1)])
def test_append_attention_prefill_rows_against_fp64(d, G, bs):
    """append_attention_c8's prompt rows (a fresh prompt and a chunk over a cached prefix) and decode row against fp64
    attention over the dequantised pages the call leaves."""
    o = _ops()
    kvh = 2
    nh = kvh * G
    ld = (nh + 2 * kvh) * d
    B, per_seq = 4, (400 + bs - 1) // bs
    nb = B * per_seq + 1
    bt = _tables(B, per_seq, nb, 21)
    k8, v8 = _random_c8(nb, kvh, bs, d, 22)
    s_k, o_k = _scales(kvh, 23)
    s_v, o_v = _scales(kvh, 24)
    enc = torch.tensor([150, 90, 0, 0], dtype=torch.int32, device=DEV)
    dec = torch.tensor([0, 200, 300, 0], dtype=torch.int32, device=DEV)
    this = torch.tensor([150, 90, 1, 0], dtype=torch.int32, device=DEV)
    cu = torch.tensor([0, 150, 240, 241, 241], dtype=torch.int32, device=DEV)
    T = 241
    x = (2 * torch.randn(T, ld, generator=_g(25), device=DEV)).to(BF16)
    cos, sin = o.rope_tables(d, per_seq * bs, 10000.0, DEV)
    out = torch.full((T, nh * d), float("nan"), dtype=BF16, device=DEV)
    o.append_attention(x, k8, v8, enc, dec, this, cu, bt, cos, sin, nh, max_q_len=150, out=out, cache_k_scale=s_k,
                       cache_v_scale=s_v, cache_k_out_scale=o_k, cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    kd, vd = C.dequantize(k8, o_k.view(1, -1, 1, 1)), C.dequantize(v8, o_v.view(1, -1, 1, 1))
    q = x[:, :nh * d].view(T, nh, d)                       # rotated in place by the call
    seq = [0] * 150 + [1] * 90 + [2]
    pos = list(range(150)) + [200 + i for i in range(90)] + [300]

    def rows(n):
        return C.gather_pages(kd, bt[seq[n]], pos[n] + 1), C.gather_pages(vd, bt[seq[n]], pos[n] + 1)

    assert_attention_close(out[:240], q[:240], rows, c=PREFILL_C, head_tol=PREFILL_HEAD_TOL,
                           what=f"c8 append prompt rows d={d} G={G} bs={bs}")
    assert_attention_close(out[240:], q[240:], lambda n: rows(240 + n), c=DECODE_C, head_tol=HEAD_TOL,
                           what=f"c8 append decode row d={d} G={G} bs={bs}")


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _model(model_type, *, append_attn, cache_int8=True, quant_type=None, block_size=32):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = _tiny(model_type)
    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    c = T.Qwen2Config(**kw) if model_type == "qwen2" else T.LlamaConfig(**kw)
    m = LlamaForCausalLMInferenceModel(c, block_attn=True, append_attn=append_attn, block_size=block_size, quant_type=quant_type,
                                       cachekv_int8_type="static" if cache_int8 else None)
    m.set_state_dict(_weights(cfg))
    return m


def _calib_ids():
    return torch.randint(1, 512, (4, 48), generator=torch.Generator().manual_seed(31))


def _rel_rows(a, b):
    a, b = a.double().reshape(a.shape[0], -1), b.double().reshape(b.shape[0], -1)
    return (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-30)


def test_generate_without_scales_raises():
    m = _model("llama", append_attn=False)
    with pytest.raises(ValueError, match="scales"):
        m.generate(torch.ones(1, 4, dtype=torch.int64), max_length=4)
    m = _model("llama", append_attn=True)
    with pytest.raises(ValueError, match="scales"):
        m.continuous_generate([(torch.ones(4, dtype=torch.int64), 4)], max_batch_size=1, num_blocks=4)


def test_set_cache_scales_from_json_matches_calibration_format():
    m = _model("llama", append_attn=False)
    t = m.transformer_block
    nh, kvh = m.config.num_attention_heads, t.kvh
    g = torch.Generator().manual_seed(5)
    d = {}
    for i in range(t.L):
        for kind in ("k", "v"):
            d[f"llama.layers.{i}.self_attn.cache{kind}_matmul.activation_quanter"] = (torch.rand(nh, generator=g) + 0.5).tolist()
    m.set_cache_scales(d)
    k, v = C.absmax_from_json(d, "llama", t.L, nh, kvh)
    for i in range(t.L):
        for name, a in (("k", k), ("v", v)):
            s, o = C.scales_from_absmax(a[i])
            assert torch.equal(getattr(t, f"cache_{name}_scales")[i].cpu(), s)
            assert torch.equal(getattr(t, f"cache_{name}_out_scales")[i].cpu(), o)
    bad = dict(d)
    bad["llama.layers.0.self_attn.cachek_matmul.activation_quanter"] = [0.0] * nh
    with pytest.raises(ValueError):
        m.set_cache_scales(bad)


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_calibration_and_cache_memory(model_type):
    mb = _model(model_type, append_attn=True, cache_int8=False)
    m8 = _model(model_type, append_attn=True)
    ka, va = m8.calibrate_cache_scales(_calib_ids())
    # the absmax of the bf16 cache of the same prefill
    caches = mb.allocate_block_caches(4, 48)
    ids = _calib_ids().to(DEV)
    mb._prefill(ids, torch.full((4,), 48, dtype=torch.int32, device=DEV), caches)
    t = m8.transformer_block
    for i in range(t.L):
        assert torch.equal(ka[i], C.absmax_of_cache(caches[2 * i].cpu()))
        assert torch.equal(va[i], C.absmax_of_cache(caches[2 * i + 1].cpu()))
    c8, cb = m8.allocate_block_caches(8, 256), mb.allocate_block_caches(8, 256)
    bytes8, bytesb = sum(c.numel() * c.element_size() for c in c8), sum(c.numel() * c.element_size() for c in cb)
    assert all(c.dtype == U8 for c in c8) and 2 * bytes8 == bytesb


@pytest.mark.parametrize("quant_type", [None, "weight_only_int8"])
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_fused_decode_step_close_to_append_attention_step(model_type, quant_type):
    """The fused split-K decode step (decode_rope_append_c8 + decode_attention_c8) against the append_attention_c8 step on the
    same int8 cache: logits at the bf16 twin test's tolerance (the two paths round the qkv projection at different points, so
    their caches may differ by a quantisation step here and there)."""
    mf = _model(model_type, append_attn=False, quant_type=quant_type)
    ma = _model(model_type, append_attn=True, quant_type=quant_type)
    mf.calibrate_cache_scales(_calib_ids())
    for name in ("cache_k_scales", "cache_v_scales", "cache_k_out_scales", "cache_v_out_scales"):
        for a, b in zip(getattr(mf.transformer_block, name), getattr(ma.transformer_block, name)):
            b.copy_(a)
    ma.transformer_block.cache_scales_set = True
    B, S = 8, 40
    ids = torch.randint(1, 512, (B, S), generator=torch.Generator().manual_seed(41)).to(DEV)
    enc = torch.full((B,), S, dtype=torch.int32, device=DEV)
    caches = mf.allocate_block_caches(B, 128)
    ma.block_tables = mf.block_tables
    mf._prefill(ids, enc, caches)
    cf, ca = [c.clone() for c in caches], [c.clone() for c in caches]
    dec = enc.clone()
    tgt = torch.randint(1, 512, (B,), generator=torch.Generator().manual_seed(42)).to(DEV)
    for step in range(4):
        lf = mf._decode(tgt, dec, cf)
        la = ma._decode(tgt, dec, ca)
        torch.cuda.synchronize()
        err = _rel_rows(lf, la).max().item()
        print(f"[{model_type}] step {step}: fused vs append_attention logits row rel. error {err:.2e}")
        assert err <= DEFAULT_SPLIT_ROW_TOL, (step, err)
        tgt = la.float().argmax(-1)
        dec = dec + 1


@pytest.mark.parametrize("quant_type", [None, "weight_only_int8"])
@pytest.mark.parametrize("append_attn", [False, True])
def test_generate_graph_equals_eager(append_attn, quant_type):
    m = _model("qwen2", append_attn=append_attn, quant_type=quant_type)
    m.calibrate_cache_scales(_calib_ids())
    ids = torch.randint(1, 512, (3, 17), generator=torch.Generator().manual_seed(1)).to(DEV)
    a = m.generate(ids, max_length=24, use_cuda_graph=True)[0]
    b = m.generate(ids, max_length=24, use_cuda_graph=False)[0]
    assert torch.equal(a, b)


@pytest.mark.parametrize("quant_type", [None, "weight_only_int8"])
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_continuous_generate_matches_each_request_alone(model_type, quant_type):
    """A mixed queue through continuous batching over an int8 cache: every request runs to its length and the pool gets every
    page back; with bf16 layer weights each request's tokens equal those it gets alone (a run of that request only, same
    pool, same scales)."""
    m = _model(model_type, append_attn=True, quant_type=quant_type)
    m.calibrate_cache_scales(_calib_ids())
    reqs = _requests(n=8)
    nb = 3 * max(math.ceil((ids.numel() + mx) / 32) + 1 for ids, mx in reqs)
    outs, stats = m.continuous_generate(reqs, max_batch_size=4, num_blocks=nb)
    assert stats["mixed_steps"] >= 2 and stats["free_blocks_at_exit"] == nb
    assert [o.numel() for o in outs] == [mx for _, mx in reqs]
    if quant_type is not None:
        return
    for r, rq in enumerate(reqs):
        alone, _ = m.continuous_generate([rq], max_batch_size=4, num_blocks=nb)
        assert torch.equal(outs[r], alone[0]), (r, outs[r].tolist(), alone[0].tolist())


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_int8_cache_logit_error(model_type):
    """Calibrated int8 cache against the bf16 cache at the same weights, teacher-forced decode steps (append_attention path
    for the prompt, the fused decode step after it)."""
    mb = _model(model_type, append_attn=False, cache_int8=False)
    m8 = _model(model_type, append_attn=False)
    B, S, steps = 4, 40, 24
    ids = torch.randint(1, 512, (B, S), generator=torch.Generator().manual_seed(51))
    m8.calibrate_cache_scales(ids)
    ids = ids.to(DEV)
    enc = torch.full((B,), S, dtype=torch.int32, device=DEV)
    cb = mb.allocate_block_caches(B, S + steps)
    c8 = m8.allocate_block_caches(B, S + steps)
    lb, l8 = mb._prefill(ids, enc, cb), m8._prefill(ids, enc, c8)
    worst = _rel_rows(l8, lb).max().item()                  # the prefill attends over the projection's bf16 K / V
    dec = enc.clone()
    tgt = lb.float().argmax(-1)
    for _ in range(steps):
        lb, l8 = mb._decode(tgt, dec, cb), m8._decode(tgt, dec, c8)
        worst = max(worst, _rel_rows(l8, lb).max().item())
        tgt = lb.float().argmax(-1)
        dec = dec + 1
    print(f"[{model_type}] int8 cache vs bf16 cache: worst logit row relative error {worst:.3e}")
    assert 0 < worst <= INT8_CACHE_LOGIT_REL, worst
