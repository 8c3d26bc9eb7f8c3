"""head_dim 64 (Llama-3.2-1B 32/8, Qwen2-0.5B 14/2, TinyLlama 32/4) through every attention kernel and the models built on them.

Attention forward (both q-tile sizes) and backward (the wgmma kernel and the mma.sync cross-check) against the fp32 oracle
and each other, with the metrics and tolerances tests/test_fa_bwd_wgmma_gpu.py applies at head_dim 128; decode attention
(bulk-copy and CUDA-core kernels, dense and paged caches) and append_attention per (sequence, head) against fp64 with the
checker and constants of tests/test_decode_attention_at_scale_gpu.py; two-layer models at the Llama-3.2-1B and Qwen2-0.5B
widths against the tied oracle; generation with every KV cache; an HF-layout checkpoint round trip.
"""
import pytest
import torch

from oracle import llama_ref as R
from test_decode_attention_at_scale_gpu import (DECODE_C, HEAD_TOL, PREFILL_C, PREFILL_HEAD_TOL, PREFILL_LOGITS_TOL,
                                                assert_attention_close, attention_reference)
from test_fa_bwd_wgmma_gpu import doc_mask, relerr, worst_tile_relerr
from test_tied_embeddings_gpu import batch, check_logits, reordered_grads
from tied_oracle import embed_key, tied_forward, tied_loss_and_grads

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BF16 = torch.bfloat16
D = 64


# ----------------------------------------------------------------------------------------------------------
# training attention: forward and backward
# ----------------------------------------------------------------------------------------------------------
def _packed_qkv(B, S, nh, kvh, g):
    """q, k, v as strided views into one packed projection [B, S, (nh + 2 kvh) * 64]."""
    qkv = torch.randn(B, S, (nh + 2 * kvh) * D, device=DEV, generator=g).to(BF16)
    q = qkv[..., :nh * D].unflatten(-1, (nh, D))
    k = qkv[..., nh * D:(nh + kvh) * D].unflatten(-1, (kvh, D))
    v = qkv[..., (nh + kvh) * D:].unflatten(-1, (kvh, D))
    return q, k, v


def _forward(impl, q, k, v, ms):
    from paddlenlp_b200 import _lib, ops

    lib = _lib.load()
    old = lib.b200_set_fa_fwd_impl(impl)
    try:
        return ops.flash_attn_fwd(q, k, v, mask_start=ms)
    finally:
        lib.b200_set_fa_fwd_impl(old)


def _backward(impl, q, k, v, out, dout, lse, ms, pad):
    """dq / dk / dv as views into NaN-filled buffers `pad` columns wider than the gradient."""
    from paddlenlp_b200 import _lib, ops

    lib = _lib.load()
    B, S, nh, _ = q.shape
    kvh = k.shape[2]
    bufs = [torch.full((B, S, h * D + pad), float("nan"), dtype=BF16, device=DEV) for h in (nh, kvh, kvh)]
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


ATTN_CASES = [
    # B, S, nh, kvh, documents per batch row (None: plain causal)
    (1, 4096, 32, 8, None),                                           # Llama-3.2-1B
    (4, 2048, 14, 2, None),                                           # Qwen2-0.5B SFT micro-batch
    (1, 2048, 32, 4, None),                                           # TinyLlama
    (1, 4096, 32, 8, [[1000, 64, 128, 2904]]),
    (4, 2048, 14, 2, [[1, 511, 1024, 512], [2048], [64, 65, 1919], [700, 900, 448]]),
    (1, 1, 1, 1, None),                                               # S at the tile edges, GQA groups 1, 3, 5, 6, 7
    (1, 63, 3, 1, None),
    (1, 64, 5, 1, None),
    (1, 65, 6, 1, None),
    (2, 127, 7, 1, None),
    (1, 128, 2, 2, None),
    (3, 129, 6, 2, [[1, 128], [64, 65], [129]]),
    (2, 200, 10, 2, [[100, 100], [37, 163]]),
]


@pytest.mark.parametrize("B,S,nh,kvh,docs", ATTN_CASES)
def test_attention_head_dim_64(B, S, nh, kvh, docs):
    g = torch.Generator(device=DEV).manual_seed(S * 131 + nh)
    q, k, v = _packed_qkv(B, S, nh, kvh, g)
    ms = None if docs is None else torch.stack([doc_mask(dl, S) for dl in docs]).to(DEV)
    out, lse = _forward(2, q, k, v, ms)
    out1, lse1 = _forward(1, q, k, v, ms)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert relerr(out1, out) < 1e-3 and relerr(lse1, lse) < 1e-5
    dout = torch.randn(B, S, nh, D, device=DEV, generator=g).to(BF16)
    new = _backward(2, q, k, v, out, dout, lse, ms, pad=256)
    old = _backward(1, q, k, v, out, dout, lse, ms, pad=0)
    worst = {}
    for name, a, b in zip(("dq", "dk", "dv"), new, old):
        if name == "dv" or S > 1:   # one row: dS = dP - rowsum(dO o O) = 0 up to rounding, so dq = dk = 0
            assert relerr(a, b) < 1e-3, (name, relerr(a, b))
    for b in range(B):
        qf, kf, vf = (t[b:b + 1].float().detach().requires_grad_(True) for t in (q, k, v))
        ref = R.attention(qf, kf, vf, "fp32", mask_start=None if ms is None else ms[b:b + 1].cpu())
        for impl, o in ((2, out), (1, out1)):
            assert relerr(o[b:b + 1].reshape(1, S, -1), ref) < 2e-2
            e = worst_tile_relerr(o[b], ref[0].reshape(S, nh, D), 64)
            worst[f"o{impl}"] = max(worst.get(f"o{impl}", 0.0), e)
            assert e < 1e-2, ("out", impl, b, e)
        ref.backward(dout[b:b + 1].float().reshape(1, S, -1))
        for impl, grads in ((2, new), (1, old)):
            for name, a, r, tile in (("dq", grads[0], qf.grad, 64), ("dk", grads[1], kf.grad, 128), ("dv", grads[2], vf.grad, 128)):
                if name != "dv" and S == 1:
                    continue
                assert relerr(a[b:b + 1], r) < 2e-2, (name, impl, b, relerr(a[b:b + 1], r))
                e = worst_tile_relerr(a[b], r[0], tile)
                worst[f"{name}{impl}"] = max(worst.get(f"{name}{impl}", 0.0), e)
                assert e < 1e-2, (name, impl, b, e)
        del ref, qf, kf, vf
    print(f"[attention d=64 B={B} S={S} {nh}/{kvh} docs={docs is not None}] worst 64/128-row tile rel. errors "
          + ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


# ----------------------------------------------------------------------------------------------------------
# decode attention and append_attention per (sequence, head) against fp64
# ----------------------------------------------------------------------------------------------------------
GQA = [(32, 32), (16, 8), (24, 8), (32, 8), (40, 8), (12, 2), (14, 2), (32, 4)]      # G = 1 .. 8


def _dense(B, kvh, seq_lens, cap, g):
    cache = torch.randn(2, B, kvh, cap, D, generator=g, device=DEV).to(BF16)
    T = [max(0, min(int(x) + 1, cap)) for x in seq_lens]
    past = torch.arange(cap, device=DEV)[None, :] >= torch.tensor(T, device=DEV)[:, None]
    cache.masked_fill_(past[None, :, None, :, None], float("nan"))
    return cache, lambda b: (cache[0, b, :, :T[b]], cache[1, b, :, :T[b]])


def _paged(B, kvh, seq_lens, bs, mb, g, spare=7):
    """Scattered pages; rows past a sequence's length and pages no table references hold NaN."""
    T = [max(0, min(int(x) + 1, mb * bs)) for x in seq_lens]
    need = [(t + bs - 1) // bs for t in T]
    nb = sum(need) + spare
    kc = torch.full((nb, kvh, bs, D), float("nan"), dtype=BF16, device=DEV)
    vc = torch.full((nb, kvh, bs, D), float("nan"), dtype=BF16, device=DEV)
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(nb)).tolist()
    tables = torch.full((B, mb), -1, dtype=torch.int32)
    i = 0
    for b in range(B):
        for j in range(need[b]):
            p, n = perm[i], min(bs, T[b] - j * bs)
            tables[b, j] = p
            kc[p, :, :n] = torch.randn(kvh, n, D, generator=g, device=DEV).to(BF16)
            vc[p, :, :n] = torch.randn(kvh, n, D, generator=g, device=DEV).to(BF16)
            i += 1

    def rows(b):
        pages = tables[b, :need[b]].long().to(DEV)
        return (kc[pages].transpose(0, 1).reshape(kvh, -1, D)[:, :T[b]], vc[pages].transpose(0, 1).reshape(kvh, -1, D)[:, :T[b]])
    return kc, vc, tables.to(DEV), rows


def _decode_case(cache_kind, nh, kvh, seq_lens, cap, seed, splits=0, what=""):
    from paddlenlp_b200 import ops

    B = len(seq_lens)
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = (nh + 2 * kvh) * D
    qkv = torch.randn(B, n + 3 * D, generator=g, device=DEV).to(BF16)[:, :n]          # strided view
    lens = torch.tensor(seq_lens, dtype=torch.int32, device=DEV)
    out = torch.full((B, nh * D), float("nan"), dtype=BF16, device=DEV)
    if cache_kind.startswith("paged"):
        bs = int(cache_kind[5:])
        kc, vc, tables, rows = _paged(B, kvh, seq_lens, bs, (cap + bs - 1) // bs, g)
        ops.decode_attention_paged(qkv, kc, vc, tables, lens, nh, out=out, num_splits=splits)
    else:
        cache, rows = _dense(B, kvh, seq_lens, cap, g)
        ops.decode_attention(qkv, cache, lens, nh, kvh, D, out=out, num_splits=splits, impl="simt" if cache_kind == "simt" else "tc")
    return assert_attention_close(out, qkv[:, :nh * D].reshape(B, nh, D), rows,
                                  what=f"d=64 {what} {cache_kind} nh={nh} kvh={kvh} splits={splits}")


KINDS = ["dense", "simt", "paged32", "paged64", "paged128"]


@pytest.mark.parametrize("cache_kind", KINDS)
@pytest.mark.parametrize("nh,kvh", GQA)
def test_decode_every_gqa_group(nh, kvh, cache_kind):
    cap = 1100
    seq_lens = [0, cap - 1, cap + 40, 31, 32, 63, 64, 65, 127, 128, 700]
    for splits in (0, 3):
        _decode_case(cache_kind, nh, kvh, seq_lens, cap, seed=nh * 100 + kvh, splits=splits, what="gqa")


@pytest.mark.parametrize("splits", [0, 1, 2, 3, 7, 64])
@pytest.mark.parametrize("cache_kind", KINDS)
def test_decode_length_sweep(cache_kind, splits):
    """Every length 0 .. 131 attended rows, a full cache and a clamped one."""
    cap = 192
    _decode_case(cache_kind, 32, 8, list(range(-1, 131)) + [cap - 1, cap + 9], cap, seed=splits + 5, splits=splits, what="sweep")


@pytest.mark.parametrize("splits", [0, 1, 64])
@pytest.mark.parametrize("cache_kind", KINDS)
def test_decode_long_cache(cache_kind, splits):
    """32k - 1, 32k and 32k + 1 attended rows."""
    _decode_case(cache_kind, 14, 2, [32766, 32767, 32768], 32768 + 128, seed=splits + 9, splits=splits, what="long")


@pytest.mark.parametrize("cache_kind", ["dense", "simt", "paged64"])
def test_decode_llama3_2_1b_benchmark_shape(cache_kind):
    _decode_case(cache_kind, 32, 8, torch.linspace(127, 2046, 64).round().int().tolist(), 2048, seed=8, what="bench")


@pytest.mark.parametrize("block_size", [32, 64, 128])
@pytest.mark.parametrize("nh,kvh", [(32, 8), (14, 2), (32, 4)])
def test_append_attention_mixed_batch(nh, kvh, block_size):
    """A 300-row prompt, a 200-row chunk on a 150-row prefix, decode rows, a one-token prompt and an idle slot that was a
    decode row in the call before, checked per (token row, head) against fp64 over the rows the op appended."""
    from paddlenlp_b200 import ops

    B, max_len = 7, 640
    mb = max_len // block_size
    ld = (nh + 2 * kvh) * D
    nb = B * mb + 5
    g = torch.Generator(device=DEV).manual_seed(nh + block_size)
    tables = torch.randperm(nb, generator=torch.Generator().manual_seed(nh))[: B * mb].to(torch.int32).view(B, mb).contiguous().to(DEV)
    kc = torch.full((nb, kvh, block_size, D), float("nan"), dtype=BF16, device=DEV)
    vc = torch.full((nb, kvh, block_size, D), float("nan"), dtype=BF16, device=DEV)
    cos, sin = ops.rope_tables(D, max_len, 10000.0, DEV)

    def call(chunks):
        n = [e - s for s, e in chunks]
        qkv = torch.randn(sum(n), ld, generator=g, device=DEV).to(BF16)
        cu = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
        enc = torch.tensor([ni if (ni > 1 or s == 0) and ni > 0 else 0 for ni, (s, e) in zip(n, chunks)], dtype=torch.int32,
                           device=DEV)
        dec = torch.tensor([s for s, e in chunks], dtype=torch.int32, device=DEV)
        this = torch.tensor(n, dtype=torch.int32, device=DEV)
        out = torch.full((sum(n), nh * D), float("nan"), dtype=BF16, device=DEV)
        ops.append_attention(qkv, kc, vc, enc, dec, this, cu, tables, cos, sin, nh, max_q_len=max(n), out=out)
        return qkv, out, cu.tolist()

    call([(0, 0), (0, 150), (0, 77), (0, 40), (0, 0), (0, 255), (0, 126)])
    call([(0, 0), (150, 150), (77, 77), (40, 41), (0, 0), (255, 255), (126, 127)])
    chunks = [(0, 300), (150, 350), (77, 78), (41, 41), (0, 1), (255, 256), (127, 128)]
    qkv, out, cu = call(chunks)
    kinds = ["prompt", "prompt", "decode", "idle", "prompt", "decode", "decode"]
    for kind, c, tol in (("decode", DECODE_C, HEAD_TOL), ("prompt", PREFILL_C, PREFILL_HEAD_TOL)):
        idx, where = [], []
        for b, (s, e) in enumerate(chunks):
            if kinds[b] == kind:
                idx += [cu[b] + i for i in range(e - s)]
                where += [(b, s + i) for i in range(e - s)]
        seqs = {b: (kc[tables[b].long()].transpose(0, 1).reshape(kvh, -1, D), vc[tables[b].long()].transpose(0, 1).reshape(kvh, -1, D))
                for b in {w[0] for w in where}}

        def rows(n):
            b, pos = where[n]
            return seqs[b][0][:, :pos + 1], seqs[b][1][:, :pos + 1]
        sel = torch.tensor(idx, device=DEV)
        assert_attention_close(out[sel], qkv[sel, :nh * D].reshape(len(idx), nh, D), rows, c=c, head_tol=tol,
                               what=f"d=64 append_attention {kind} rows nh={nh} kvh={kvh} block_size={block_size}")
    assert cu[3] == cu[4]


def test_attention_reference_is_head_dim_agnostic():
    q = torch.randn(4, D, dtype=torch.float64)
    K, V = torch.randn(2, 5, D, dtype=torch.float64), torch.randn(2, 5, D, dtype=torch.float64)
    ref, _ = attention_reference(q, K, V)
    p = torch.softmax(q[0] @ K[0].t() / D ** 0.5, -1)
    assert torch.allclose(ref[0], p @ V[0])


# ----------------------------------------------------------------------------------------------------------
# models at the released widths
# ----------------------------------------------------------------------------------------------------------
WIDTHS = {
    "llama3_2_1b": dict(model_type="llama", hidden_size=2048, intermediate_size=8192, num_attention_heads=32,
                        num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0),
    "qwen2_0_5b": dict(model_type="qwen2", hidden_size=896, intermediate_size=4864, num_attention_heads=14,
                       num_key_value_heads=2, rms_norm_eps=1e-6, rope_theta=1000000.0),
}


def _ref_cfg(width, vocab, max_pos, layers=2):
    spec = dict(WIDTHS[width])
    mt = spec.pop("model_type")
    return R.RefConfig(vocab_size=vocab, num_hidden_layers=layers, max_position_embeddings=max_pos, qkv_bias=mt == "qwen2",
                       model_type=mt, **spec)


def _tied_weights(cfg, seed, scale=8):
    w = R.init_weights(cfg, seed=seed)
    w.pop("lm_head.weight")
    E = embed_key(cfg)
    w[E] = (w[E] * scale).to(BF16).float()                                # decisive logits at the 0.02 init scale
    if cfg.qkv_bias:                                                       # non-zero q / k / v biases
        g = torch.Generator().manual_seed(seed + 1)
        for k in w:
            if k.endswith("_proj.bias"):
                w[k] = (0.1 * torch.randn(w[k].shape, generator=g)).to(BF16).float()
    return w


def _model(cfg, w, **extra):
    import paddlenlp_b200.transformers as T

    C = T.Qwen2Config if cfg.model_type == "qwen2" else T.LlamaConfig
    M = T.Qwen2ForCausalLM if cfg.model_type == "qwen2" else T.LlamaForCausalLM
    model = M(C(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                max_position_embeddings=cfg.max_position_embeddings, tie_word_embeddings=True, **extra))
    model.set_state_dict(w)
    return model


@pytest.mark.parametrize("width,S", [("llama3_2_1b", 4096), ("qwen2_0_5b", 2048)])
def test_two_layer_tied_model_real_vocab(width, S):
    """Two layers, the released tied head and vocabulary: logits, loss and every weight gradient against the tied oracle on
    the device, gradient tolerance max(3e-2, 2 x the oracle's own re-ordering floor)."""
    vocab = 128256 if width == "llama3_2_1b" else 151936
    cfg = _ref_cfg(width, vocab, S)
    w = _tied_weights(cfg, seed=71)
    model = _model(cfg, w)
    ids, labels = batch(cfg, 1, S, 72)
    model.engine.clear_grad()
    loss, logits = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    logits = logits.float().clone()
    loss.backward()
    wd = {k: v.to(DEV) for k, v in w.items()}
    ids_d, lab_d = ids.to(DEV), labels.to(DEV)
    with torch.no_grad():
        ref32 = tied_forward(ids_d, wd, cfg, "fp32")
    ref_loss, ref16, gref = tied_loss_and_grads(ids_d, lab_d, wd, cfg, "bf16")
    check_logits(f"{width} 2 layers tied S={S}", logits, ref16, ref32)
    assert abs(float(loss) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    del ref16, ref32, logits
    gref2 = reordered_grads(ids_d, lab_d, wd, cfg)
    grads = model.engine.named_views(grads=True)
    assert set(gref) <= set(grads), set(gref) - set(grads)
    for k in sorted(gref):
        e, floor = relerr(grads[k], gref[k]), relerr(gref2[k], gref[k])
        print(f"[{width} 2 layers tied S={S}] grad {k}: rel err {e:.2e}; oracle re-ordering floor {floor:.2e}")
        assert e < max(3e-2, 2.0 * floor), (k, e, floor)


@pytest.mark.parametrize("width", list(WIDTHS))
def test_packing_and_recompute(width):
    """Three documents packed into one row under FlashMask give the logits of the documents run one by one (the first bit
    for bit: same tiles, same order); recompute gives bit-identical loss and logits and gradients within the attention
    backward's reduce-add ordering noise."""
    cfg = _ref_cfg(width, 4096, 512)
    w = _tied_weights(cfg, seed=81, scale=4)
    model = _model(cfg, w)
    lens = [150, 37, 201]
    g = torch.Generator().manual_seed(11)
    docs = [torch.randint(1, cfg.vocab_size, (n,), generator=g) for n in lens]
    ids = torch.cat(docs + [torch.zeros(512 - sum(lens), dtype=torch.int64)])[None].to(DEV)
    pos = torch.cat([torch.arange(n) for n in lens] + [torch.arange(512 - sum(lens))])[None].to(DEV)
    ms = torch.cat([torch.full((n,), s + n, dtype=torch.int32) for s, n in zip([0, 150, 187], lens)]
                   + [torch.zeros(512 - sum(lens), dtype=torch.int32)])[None].to(DEV)
    with torch.no_grad():
        packed = model(input_ids=ids, position_ids=pos, attn_mask_startend_row_indices=ms)[0].float().clone()
        start = 0
        for d in docs:
            one = model(input_ids=d[None].to(DEV))[0].float()
            e = ((packed[0, start:start + len(d)] - one[0]).abs().max() / one.abs().max()).item()
            assert e < 2e-2, (start, e)
            if start == 0:
                assert torch.equal(packed[0, :len(d)], one[0])
            start += len(d)
    tok = torch.randint(0, cfg.vocab_size, (2, 257), generator=torch.Generator().manual_seed(9))
    i2, l2 = tok[:, :-1].contiguous().to(DEV), tok[:, 1:].contiguous().to(DEV)
    model.engine.clear_grad()
    loss_a, logits_a = model(input_ids=i2, labels=l2)
    logits_a = logits_a.clone()
    loss_a.backward()
    g_a = model.engine.flat_grads.clone()
    model.recompute_enable()
    model.engine.clear_grad()
    loss_b, logits_b = model(input_ids=i2, labels=l2)
    assert torch.equal(loss_a.detach(), loss_b.detach()) and torch.equal(logits_a, logits_b)
    loss_b.backward()
    e = relerr(model.engine.flat_grads, g_a)
    print(f"[{width}] recompute: loss and logits bit-identical, gradient rel. difference {e:.2e}")
    assert e < 2e-3
    model.recompute_disable()


@pytest.mark.parametrize("width", list(WIDTHS))
def test_generation_every_cache_and_graph(width):
    """Greedy tokens identical across the dense, paged and append_attention caches, with and without the CUDA graph; prefill
    and three decode steps against the uncached training-path forward (the tolerances of the head_dim 128 test)."""
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel
    import paddlenlp_b200.transformers as T

    cfg = _ref_cfg(width, 4096, 512)
    w = _tied_weights(cfg, seed=91)
    train = _model(cfg, w)
    C = T.Qwen2Config if cfg.model_type == "qwen2" else T.LlamaConfig
    hf = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings, tie_word_embeddings=True)
    prompt = torch.randint(0, cfg.vocab_size, (8, 130), generator=torch.Generator().manual_seed(42))
    tokens = []
    for cache in ("dense", "paged", "append_attn"):
        inf = LlamaForCausalLMInferenceModel(C(**hf), block_attn=cache != "dense", append_attn=cache == "append_attn")
        inf.set_state_dict(w)
        for graph in (True, False):
            out, _, _ = inf.generate(prompt, max_length=12, use_cuda_graph=graph)
            tokens.append(((cache, graph), out.cpu()))
        B, S = 64, 130
        ids = torch.randint(0, cfg.vocab_size, (B, S), generator=torch.Generator().manual_seed(43)).to(DEV)
        enc = torch.full((B,), S, dtype=torch.int32, device=DEV)
        caches = inf.allocate_caches(B, S + 8)
        lg = inf._prefill(ids, enc, caches)
        full = train.engine.forward_logits(ids)[:, -1].float()
        e0 = ((lg.float() - full).abs().max() / full.abs().max()).item()
        assert e0 < PREFILL_LOGITS_TOL, (cache, e0)
        seq, lens = ids, enc.clone()
        for step in range(3):
            nxt = lg.float().argmax(-1)
            seq = torch.cat([seq, nxt[:, None]], dim=1)
            lg = inf._decode(nxt, lens, caches)
            lens += 1
            ref = train.engine.forward_logits(seq)[:, -1].float()
            err = ((lg.float() - ref).abs().max() / ref.abs().max()).item()
            print(f"[{width} {cache}] prefill {e0:.2e}, decode step {step}: {err:.2e}")
            assert err < 2e-2, (cache, step, err)
        del inf, caches
    for key, t in tokens[1:]:
        assert torch.equal(t, tokens[0][1]), (key, tokens[0][0])


def test_qwen2_0_5b_width_hf_checkpoint_round_trip(tmp_path):
    import paddlenlp_b200.transformers as T

    cfg = _ref_cfg("qwen2_0_5b", 4096, 512)
    model = _model(cfg, _tied_weights(cfg, seed=101))
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(5)).to(DEV)
    with torch.no_grad():
        a = model(input_ids=ids)[0].clone()
    model.save_pretrained(str(tmp_path), hf_format=True)
    loaded = T.Qwen2ForCausalLM.from_pretrained(str(tmp_path))
    assert loaded.engine.tied and loaded.engine.d == 64
    with torch.no_grad():
        b = loaded(input_ids=ids)[0]
    assert torch.equal(a, b)
