"""Decode and append attention per (sequence, head) against fp64, at every shipped preset's GQA ratio.

The decode kernels (the bulk-copy kernel of decode_attn_tc.cu over the dense and the paged cache, and the CUDA-core kernel
in decode_attn_tc.cu that cross-checks it) and append_attention stream the cache in 32-row chunks, clamp the length to
seq_lens + 1 and split long sequences across CTAs.  The bugs such code grows (a dropped partial chunk, rows attended past
the length, the new token left out, a lost split, the wrong kv head) move a long sequence's output by a small amount in
absolute terms, because that output is an average of thousands of V rows (elements ~0.04) while a sequence with no
history returns one V row (elements ~3).  A relative error over the whole batch cannot see them; the checker here works
per element and per (sequence, head), and its own CPU tests (no gpu mark) show that it rejects each of those bugs while
the old whole-batch check accepts the first three.

GQA groups: G = 1 (32/32), 3 (Llama-3.2-3B 24/8), 4 (Llama-3-8B 32/8), 5 (Qwen2.5-14B/32B 40/8), 6 (Qwen2-1.5B 12/2),
7 (Qwen2-7B 28/4) and 8 (16/2).  Rows of the cache that no sequence may read (past a sequence's length, in pages no block
table references) hold NaN, and every output starts as NaN, so a stray read or a missing write fails the finiteness check.
"""
import math

import pytest
import torch

from oracle import llama_ref as R

DEV = "cuda:0"
BF16 = torch.bfloat16
D = 128
BF16_REL = 2.0 ** -8           # one bf16 rounding of the output: at most half an ulp, <= 2^-8 of the value rounded
# Measured on an H100 80GB HBM3 at a 400 W power limit, over every case below.
# Per-element allowance for the fp32 arithmetic of the decode kernels (scores, exp2, P V, the split merge), times
# sum_t p_t |v_t|.  c_need <= 9.6e-8 in every decode case (the worst: the length sweep over 32-row pages); c is ~4x that.
DECODE_C = 4e-7
# Relative Frobenius error of one (sequence, head) output: one bf16 rounding is ~1.6e-3 rms (measured worst 2.3e-3).
HEAD_TOL = 4e-3
# append_attention's prompt rows run the flash-attention kernel, which rounds P to bf16 before the P V product:
# c_need <= 2.5e-3 and (row, head) error <= 3.1e-3 over the three GQA groups and two page sizes.
PREFILL_C = 1e-2
PREFILL_HEAD_TOL = 6e-3
OLD_TOL = 1.5e-2               # the whole-batch check the generation tests use: max|out - ref| / max|ref|
# Prefill logits of the inference stack vs the training-path forward, max|diff| / max|ref|, two layers: the same
# computation with other rounding points and GEMM summation orders; 5.2e-3 .. 8.0e-3 measured at the three widths.
PREFILL_LOGITS_TOL = 1.5e-2


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


# ----------------------------------------------------------------------------------------------------------
# Checker
# ----------------------------------------------------------------------------------------------------------
def attention_reference(q, K, V, scale=None):
    """fp64 softmax(q K^T * scale) V for one query row.  q [nh, d]; K, V [kvh, T, d] (query head h reads kv head
    h // (nh / kvh)).  Returns (ref, mag) [nh, d], mag = sum_t p_t |v_t|; T = 0 gives zeros (the kernels' output for a
    sequence with nothing to attend to)."""
    nh, d = q.shape
    kvh, T = K.shape[0], K.shape[1]
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    if T == 0:
        z = torch.zeros(nh, d, dtype=torch.float64, device=q.device)
        return z, z
    qg = q.double().view(kvh, nh // kvh, d)
    p = torch.softmax(torch.bmm(qg, K.double().transpose(1, 2)) * scale, dim=-1)
    Vd = V.double()
    return torch.bmm(p, Vd).reshape(nh, d), torch.bmm(p, Vd.abs()).reshape(nh, d)


def assert_attention_close(out, q, rows, *, c=DECODE_C, head_tol=HEAD_TOL, scale=None, what="decode"):
    """Check out [N, nh*d] (one query row per entry) against attention_reference, one row at a time.

    q [N, nh, d] are the query rows the kernel read; rows(n) -> (K, V) [kvh, T_n, d] are the cache rows query n attends to.
    Three checks:
      per element        |out - ref| <= 2^-8 |ref| + c * sum_t p_t |v_t|
      per (row, head)    relative Frobenius error <= head_tol (a head whose reference is zero must be exactly zero)
      finite             every output element (callers pre-fill out with NaN, so a row that is never written fails)
    Returns the worst element error/bound ratio, the smallest c the output needs (c_need) and the worst head error."""
    N, nh, d = q.shape
    assert tuple(out.shape) == (N, nh * d), (tuple(out.shape), tuple(q.shape))
    fin = torch.isfinite(out)
    if not bool(fin.all()):
        n, j = (~fin).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~fin).sum())} non-finite (unwritten?) outputs, first at row {n} head {j // d}")
    ratios, needs, heads = [], [], []
    for n in range(N):
        K, V = rows(n)
        ref, mag = attention_reference(q[n], K, V, scale)
        got = out[n].double().view(nh, d)
        err = (got - ref).abs()
        ratios.append((err / (BF16_REL * ref.abs() + c * mag + 1e-300)).max())
        needs.append(((err - BF16_REL * ref.abs()).clamp_min(0) / (mag + 1e-300)).max())
        en, rn = err.norm(dim=-1), ref.norm(dim=-1)
        heads.append(torch.where(rn > 0, en / rn.clamp_min(1e-300), torch.where(en > 0, math.inf, 0.0)))
    ratios, needs, heads = torch.stack(ratios).cpu(), torch.stack(needs).cpu(), torch.stack(heads).cpu()
    k = int(heads.view(-1).argmax())
    worst = dict(ratio=ratios.max().item(), at=int(ratios.argmax()), c_need=needs.max().item(),
                 head=heads.view(-1)[k].item(), head_at=(k // nh, k % nh))
    print(f"[{what}] worst element error / bound {worst['ratio']:.3f} (row {worst['at']}), c_need {worst['c_need']:.2e}, "
          f"worst (row, head) rel. error {worst['head']:.2e} at {worst['head_at']}")
    assert worst["ratio"] <= 1.0, f"{what}: element error exceeds its bound: {worst}"
    assert worst["head"] <= head_tol, f"{what}: (row, head) relative error exceeds {head_tol}: {worst}"
    return worst


def old_global_error(out, ref):
    return ((out.double() - ref).abs().max() / ref.abs().max()).item()


# ----------------------------------------------------------------------------------------------------------
# CPU tests of the checker: the statistics of the decode tests (B = 16, 2 kv heads, G = 3, lengths up to 2 048, a
# sequence with no history in row 0, N(0, 1) q / k / v rounded to bf16); each sabotage changes one sequence
# ----------------------------------------------------------------------------------------------------------
def _table_batch():
    B, kvh, G, cap = 16, 2, 3, 2048
    nh = kvh * G
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(100, cap - 1, (B,), generator=g)
    lens[0], lens[1] = 0, cap - 1                                        # no history; 2 048 rows with the new token
    q = torch.randn(B, nh, D, generator=g).to(BF16)
    K = torch.randn(B, kvh, cap + 8, D, generator=g).to(BF16)            # 8 rows past the longest sequence: garbage
    V = torch.randn(B, kvh, cap + 8, D, generator=g).to(BF16)
    T = [int(x) + 1 for x in lens]
    return q, K, V, T


def _outputs(q, K, V, T, sabotage=None):
    """fp64 reference [B, nh*d] and its bf16 rounding; `sabotage(b) -> (K_b, V_b)` replaces sequence b's rows."""
    ref = []
    for b in range(q.shape[0]):
        kb, vb = K[b, :, :T[b]], V[b, :, :T[b]]
        if sabotage is not None:
            kb, vb = sabotage(b, kb, vb)
        ref.append(attention_reference(q[b], kb, vb)[0].reshape(-1))
    ref = torch.stack(ref)
    return ref, ref.to(BF16)


def _sabotaged(name, T):
    long_partial = max((b for b in range(len(T)) if T[b] % 32 >= 16), key=lambda b: T[b])
    longest = max(range(len(T)), key=lambda b: T[b])
    if name == "partial chunk dropped":
        s = long_partial
        return s, lambda b, k, v, K, V: (k[:, :T[b] // 32 * 32], v[:, :T[b] // 32 * 32]) if b == s else (k, v)
    if name == "5 rows past the length":
        s = longest
        return s, lambda b, k, v, K, V: (K[b, :, :T[b] + 5], V[b, :, :T[b] + 5]) if b == s else (k, v)
    if name == "new token excluded":
        s = 1
        assert T[s] == 2048
        return s, lambda b, k, v, K, V: (k[:, :-1], v[:, :-1]) if b == s else (k, v)
    if name == "one split dropped":
        s = longest
        q4 = T[s] // 4

        def drop(b, k, v, K, V):
            if b != s:
                return k, v
            keep = torch.cat([torch.arange(q4), torch.arange(2 * q4, T[b])])
            return k[:, keep], v[:, keep]
        return s, drop
    if name == "wrong kv head":
        s = longest
        return s, lambda b, k, v, K, V: (k.flip(0), v.flip(0)) if b == s else (k, v)
    raise KeyError(name)


def _rows_of(K, V, T):
    return lambda b: (K[b, :, :T[b]], V[b, :, :T[b]])


def test_checker_accepts_a_correctly_rounded_result():
    q, K, V, T = _table_batch()
    ref, out = _outputs(q, K, V, T)
    w = assert_attention_close(out, q, _rows_of(K, V, T), what="correct")
    assert w["c_need"] == 0.0                                   # one rounding: half an ulp <= 2^-8 |ref|
    assert old_global_error(out, ref) < OLD_TOL


@pytest.mark.parametrize("name,old_passes", [("partial chunk dropped", True), ("5 rows past the length", True),
                                             ("new token excluded", True), ("one split dropped", False),
                                             ("wrong kv head", False)])
def test_checker_rejects_sabotage(name, old_passes):
    q, K, V, T = _table_batch()
    ref, _ = _outputs(q, K, V, T)
    s, fn = _sabotaged(name, T)
    _, bad = _outputs(q, K, V, T, lambda b, k, v: fn(b, k, v, K, V))
    old = old_global_error(bad, ref)
    head = max(((bad[s].double() - ref[s]).view(-1, D).norm(dim=-1) / ref[s].view(-1, D).norm(dim=-1)).tolist())
    print(f"[{name}] sequence {s} (T = {T[s]}): old whole-batch check {old:.1e} (tol {OLD_TOL}), "
          f"worst (sequence, head) rel. error {head:.1e}")
    assert (old < OLD_TOL) == old_passes
    with pytest.raises(AssertionError, match="relative error exceeds|element error exceeds"):
        assert_attention_close(bad, q, _rows_of(K, V, T), what=name)


def test_checker_rejects_an_unwritten_row():
    q, K, V, T = _table_batch()
    ref, out = _outputs(q, K, V, T)
    out[5, 2 * D:3 * D] = float("nan")                                   # one (sequence, head) never written
    with pytest.raises(AssertionError, match="non-finite"):
        assert_attention_close(out, q, _rows_of(K, V, T), what="nan row")


def test_unsupported_gqa_group_is_refused_at_construction():
    """The decode kernels are instantiated for G = nh / kvh in 1..8: a model outside that fails when it is built, not at the
    first decode step after a prefill."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel
    from paddlenlp_b200.experimental.transformers.fused_transformer_layers import (FusedBlockMultiTransformer,
                                                                                   FusedMultiTransformerBase,
                                                                                   FusedMultiTransformerConfig)

    for cls in (FusedMultiTransformerBase, FusedBlockMultiTransformer):
        with pytest.raises(ValueError, match="GQA group size 9"):
            cls(FusedMultiTransformerConfig(embed_dim=18 * D, num_heads=18, kv_num_heads=2, dim_feedforward=256, num_layers=1))
        with pytest.raises(ValueError, match="multiple"):
            cls(FusedMultiTransformerConfig(embed_dim=16 * D, num_heads=16, kv_num_heads=3, dim_feedforward=256, num_layers=1))
    cfg = T.LlamaConfig(vocab_size=512, hidden_size=32 * D, intermediate_size=256, num_hidden_layers=1, num_attention_heads=32,
                        num_key_value_heads=2)
    for block_attn in (False, True):
        with pytest.raises(ValueError, match="GQA group size 16"):
            LlamaForCausalLMInferenceModel(cfg, block_attn=block_attn)


# ----------------------------------------------------------------------------------------------------------
# decode kernels on the GPU
# ----------------------------------------------------------------------------------------------------------
GQA = [(32, 32), (24, 8), (32, 8), (40, 8), (12, 2), (28, 4), (16, 2)]      # G = 1, 3, 4, 5, 6, 7, 8


def _qkv(B, nh, kvh, g, pad=0):
    """Packed projection [B, (nh + 2 kvh) d]; with pad > 0 a view of a wider buffer (stride(0) = width + pad)."""
    n = (nh + 2 * kvh) * D
    return torch.randn(B, n + pad, generator=g, device=DEV).to(BF16)[:, :n]


def _dense(B, kvh, seq_lens, cap, g):
    """Dense cache [2, B, kvh, cap, d] with NaN past every sequence's T = min(seq_lens + 1, cap) rows."""
    cache = torch.randn(2, B, kvh, cap, D, generator=g, device=DEV).to(BF16)
    T = [max(0, min(int(x) + 1, cap)) for x in seq_lens]
    past = torch.arange(cap, device=DEV)[None, :] >= torch.tensor(T, device=DEV)[:, None]
    cache.masked_fill_(past[None, :, None, :, None], float("nan"))
    return cache, T, lambda b: (cache[0, b, :, :T[b]], cache[1, b, :, :T[b]])


def _paged(B, kvh, seq_lens, bs, mb, g, spare=7):
    """Paged pools [nb, kvh, bs, d] with scattered pages: every sequence owns ceil(T / bs) pages (T = min(seq_lens + 1,
    mb * bs)), its table entries past them are -1; rows past T in its last page and every page no table references
    hold NaN."""
    T = [max(0, min(int(x) + 1, mb * bs)) for x in seq_lens]
    need = [(t + bs - 1) // bs for t in T]
    nb = sum(need) + spare
    kc = torch.randn(nb, kvh, bs, D, generator=g, device=DEV).to(BF16)
    vc = torch.randn(nb, kvh, bs, D, generator=g, device=DEV).to(BF16)
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(nb)).tolist()
    tables = torch.full((B, mb), -1, dtype=torch.int32)
    used = torch.zeros(nb, dtype=torch.bool)
    i = 0
    for b in range(B):
        for j in range(need[b]):
            tables[b, j] = perm[i]
            used[perm[i]] = True
            i += 1
        if need[b] and T[b] % bs:
            last = int(tables[b, need[b] - 1])
            kc[last, :, T[b] % bs:] = float("nan")
            vc[last, :, T[b] % bs:] = float("nan")
    kc[~used.to(DEV)] = float("nan")
    vc[~used.to(DEV)] = float("nan")

    def rows(b):
        pages = tables[b, :need[b]].long().to(DEV)
        k = kc[pages].transpose(0, 1).reshape(kvh, -1, D)[:, :T[b]]
        v = vc[pages].transpose(0, 1).reshape(kvh, -1, D)[:, :T[b]]
        return k, v
    return kc, vc, tables.to(DEV), T, rows


def _decode_case(cache_kind, nh, kvh, seq_lens, cap, seed, splits=0, pad=0, what=""):
    """Run one decode kernel on NaN-filled garbage around the data and check it; cache_kind: "dense" (bulk kernel),
    "simt" (CUDA-core kernel, dense cache) or "pagedN" (bulk kernel, N-row pages; cap rounded up to whole pages)."""
    o = ops()
    B = len(seq_lens)
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = _qkv(B, nh, kvh, g, pad)
    lens = torch.tensor(seq_lens, dtype=torch.int32, device=DEV)
    out = torch.full((B, nh * D), float("nan"), dtype=BF16, device=DEV)
    if cache_kind.startswith("paged"):
        bs = int(cache_kind[5:])
        kc, vc, tables, T, rows = _paged(B, kvh, seq_lens, bs, (cap + bs - 1) // bs, g)
        o.decode_attention_paged(qkv, kc, vc, tables, lens, nh, out=out, num_splits=splits)
    else:
        cache, T, rows = _dense(B, kvh, seq_lens, cap, g)
        o.decode_attention(qkv, cache, lens, nh, kvh, D, out=out, num_splits=splits,
                           impl="simt" if cache_kind == "simt" else "tc")
    q = qkv[:, :nh * D].reshape(B, nh, D)
    return assert_attention_close(out, q, rows, what=f"{what} {cache_kind} nh={nh} kvh={kvh} splits={splits}")


@pytest.mark.gpu
@pytest.mark.parametrize("cache_kind", ["dense", "simt", "paged64"])
@pytest.mark.parametrize("nh,kvh", GQA)
def test_decode_every_gqa_ratio(nh, kvh, cache_kind):
    """Every preset's GQA group through each decode kernel, ragged lengths across several 128-row tiles (no history, a
    full cache and one clamped past it), a strided qkv view, automatic splits and a forced 3-way split."""
    cap = 1100
    seq_lens = [0, cap - 1, cap + 40, 31, 32, 127, 128, 700]
    for splits in (0, 3):
        _decode_case(cache_kind, nh, kvh, seq_lens, cap, seed=nh * 100 + kvh, splits=splits, pad=3 * D, what="gqa")


@pytest.mark.gpu
@pytest.mark.parametrize("cache_kind", ["dense", "simt", "paged64"])
def test_decode_benchmark_shape(cache_kind):
    """The decode benchmark's attention: Llama-3-8B 32/8, batch 64, lengths spread over the 128-token prompt plus 1 920
    generated tokens."""
    seq_lens = torch.linspace(127, 2046, 64).round().int().tolist()
    _decode_case(cache_kind, 32, 8, seq_lens, 2048, seed=8, what="benchmark shape")


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [0, 1, 2, 3, 7, 64])
@pytest.mark.parametrize("cache_kind", ["dense", "simt", "paged32", "paged64", "paged128"])
def test_decode_length_sweep(cache_kind, splits):
    """Every length 0 .. 131 attended rows (seq_lens -1 .. 130): each partial 32-row chunk, the first and last row of every
    page and of the first 128-row tile; plus a full and a clamped cache.  With 64 splits most splits are empty."""
    cap = 192
    seq_lens = list(range(-1, 131)) + [cap - 1, cap + 9]
    _decode_case(cache_kind, 24, 8, seq_lens, cap, seed=splits + 3, splits=splits, what="sweep")


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [0, 1, 7, 64])
@pytest.mark.parametrize("B", [1, 3, 5])
@pytest.mark.parametrize("cache_kind", ["dense", "simt", "paged128"])
@pytest.mark.parametrize("nh,kvh", [(12, 2), (32, 8)])
def test_decode_long_cache(nh, kvh, cache_kind, B, splits):
    """32k - 1, 32k and 32k + 1 attended rows, a full cache and one clamped past it, over a 32 896-row cache.  At batch 1
    and 3 the automatic choice asks for many splits (most of a short sequence's would be empty)."""
    cap = 32768 + 128
    seq_lens = [32767, 32766, 32768, cap - 1, cap + 100][:B]
    _decode_case(cache_kind, nh, kvh, seq_lens, cap, seed=B * 10 + splits, splits=splits, what="long")


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["decode_attention", "decode_attention_paged"])
def test_decode_unsupported_gqa_group_is_an_error(fn):
    from paddlenlp_b200._lib import B200Error

    o = ops()
    g = torch.Generator(device=DEV).manual_seed(0)
    nh, kvh = 18, 2
    qkv = _qkv(2, nh, kvh, g)
    lens = torch.tensor([3, 5], dtype=torch.int32, device=DEV)
    with pytest.raises(B200Error, match="GQA group size 9 not instantiated"):
        if fn == "decode_attention":
            o.decode_attention(qkv, torch.zeros(2, 2, kvh, 64, D, dtype=BF16, device=DEV), lens, nh, kvh, D)
        else:
            kc = torch.zeros(4, kvh, 32, D, dtype=BF16, device=DEV)
            o.decode_attention_paged(qkv, kc, kc.clone(), torch.zeros(2, 2, dtype=torch.int32, device=DEV), lens, nh)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------
# append_attention: a mixed batch per (token row, head)
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block_size", [32, 128])
@pytest.mark.parametrize("nh,kvh", [(24, 8), (12, 2), (32, 8)])
def test_append_attention_per_row_and_head(nh, kvh, block_size):
    """One call serves a 300-row prompt (three 128-row q tiles), a 200-row prompt chunk on a 150-row cached prefix (not page
    aligned), three decode rows (T = 78, 128 and 256), a one-token prompt and an idle slot that was a decode row in the
    call before (its stale decode length must not write anything).  The reference is built from the rotated q the op left
    in qkv and the k / v it appended to the pages (test_generation_gpu checks those against the oracle), so this measures
    attention alone."""
    o = ops()
    B, max_len = 7, 640
    mb = max_len // block_size
    ld = (nh + 2 * kvh) * D
    nb = B * mb + 5
    g = torch.Generator(device=DEV).manual_seed(nh + block_size)
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(nh))[: B * mb].to(torch.int32)
    tables = perm.view(B, mb).contiguous().to(DEV)
    kc = torch.full((nb, kvh, block_size, D), float("nan"), dtype=BF16, device=DEV)
    vc = torch.full((nb, kvh, block_size, D), float("nan"), dtype=BF16, device=DEV)
    cos, sin = o.rope_tables(D, max_len, 10000.0, DEV)

    def call(chunks):
        """chunks: per slot (start, stop) rows appended in this call; stop == start: idle; start > 0 and one row: decode."""
        n = [e - s for s, e in chunks]
        assert n[-1] > 0                                              # no trailing idle slot: cu_seqlens_q[B-1] < token_num
        qkv = torch.randn(sum(n), ld, generator=g, device=DEV).to(BF16)
        cu = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
        enc = torch.tensor([ni if (ni > 1 or s == 0) and ni > 0 else 0 for ni, (s, e) in zip(n, chunks)], dtype=torch.int32,
                           device=DEV)
        dec = torch.tensor([s for s, e in chunks], dtype=torch.int32, device=DEV)
        this = torch.tensor(n, dtype=torch.int32, device=DEV)
        out = torch.full((sum(n), nh * D), float("nan"), dtype=BF16, device=DEV)
        o.append_attention(qkv, kc, vc, enc, dec, this, cu, tables, cos, sin, nh, max_q_len=max(n), out=out)
        return qkv, out, cu.tolist()

    # prefixes: slot 1: 150 rows, slot 2: 77, slot 3: 40 (+1 decode row next), slot 5: 255, slot 6: 126 (+1 decode row)
    call([(0, 0), (0, 150), (0, 77), (0, 40), (0, 0), (0, 255), (0, 126)])
    call([(0, 0), (150, 150), (77, 77), (40, 41), (0, 0), (255, 255), (126, 127)])
    chunks = [(0, 300), (150, 350), (77, 78), (41, 41), (0, 1), (255, 256), (127, 128)]
    qkv, out, cu = call(chunks)
    kinds = ["prompt", "prompt", "decode", "idle", "prompt", "decode", "decode"]

    def seq_rows(b):
        pages = tables[b].long()
        return kc[pages].transpose(0, 1).reshape(kvh, -1, D), vc[pages].transpose(0, 1).reshape(kvh, -1, D)

    worst = {}
    for kind, c, tol in (("decode", DECODE_C, HEAD_TOL), ("prompt", PREFILL_C, PREFILL_HEAD_TOL)):
        idx, where = [], []
        for b, (s, e) in enumerate(chunks):
            if kinds[b] == kind:
                for i in range(e - s):
                    idx.append(cu[b] + i)
                    where.append((b, s + i))
        cache = {b: seq_rows(b) for b in {w[0] for w in where}}

        def rows(n):
            b, pos = where[n]
            K, V = cache[b]
            return K[:, :pos + 1], V[:, :pos + 1]
        sel = torch.tensor(idx, device=DEV)
        worst[kind] = assert_attention_close(out[sel], qkv[sel, :nh * D].reshape(len(idx), nh, D), rows, c=c, head_tol=tol,
                                             what=f"append_attention {kind} rows nh={nh} kvh={kvh} block_size={block_size}")
    assert cu[3] == cu[4]                                             # the idle slot owns no row


# ----------------------------------------------------------------------------------------------------------
# end to end at the benchmark models' widths
# ----------------------------------------------------------------------------------------------------------
WIDTHS = {
    "llama3_2_3b": dict(model_type="llama", tied=False, hidden_size=3072, intermediate_size=8192, num_attention_heads=24,
                        num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0),
    "llama3_2_3b_tied": dict(model_type="llama", tied=True, hidden_size=3072, intermediate_size=8192, num_attention_heads=24,
                             num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0),
    "qwen2_1_5b": dict(model_type="qwen2", tied=False, hidden_size=1536, intermediate_size=8960, num_attention_heads=12,
                       num_key_value_heads=2, rms_norm_eps=1e-6, rope_theta=1000000.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cache", ["dense", "paged", "append_attn"])
@pytest.mark.parametrize("width", list(WIDTHS))
def test_benchmark_width_decode_matches_uncached_forward(width, cache):
    """As test_generation_gpu.test_full_width_decode_matches_uncached_forward, at the widths of the two benchmark models
    (two layers, a 4 096-token vocabulary, batch 64, a 130-token prompt): prefill logits match the training-path forward,
    and three decode steps reproduce the uncached forward of the grown sequence within bf16 noise, with identical decisive
    arg-max."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    spec = dict(WIDTHS[width])
    model_type, tied = spec.pop("model_type"), spec.pop("tied")
    kw = dict(vocab_size=4096, num_hidden_layers=2, max_position_embeddings=512, **spec)
    cfg = R.RefConfig(qkv_bias=model_type == "qwen2", model_type=model_type, **kw)
    w = R.init_weights(cfg, seed=41)
    if tied:
        w.pop("lm_head.weight")
        E = f"{model_type}.embed_tokens.weight"
        w[E] = (w[E] * 8).to(BF16).float()
    else:
        w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(BF16).float()
    C = T.Qwen2Config if model_type == "qwen2" else T.LlamaConfig
    M = T.Qwen2ForCausalLM if model_type == "qwen2" else T.LlamaForCausalLM
    train = M(C(tie_word_embeddings=tied, **kw))
    train.set_state_dict(w)
    inf = LlamaForCausalLMInferenceModel(C(tie_word_embeddings=tied, **kw), block_attn=cache != "dense",
                                         append_attn=cache == "append_attn")
    inf.set_state_dict(w)
    B, S = 64, 130
    ids = torch.randint(0, cfg.vocab_size, (B, S), generator=torch.Generator().manual_seed(42)).to(DEV)
    enc = torch.full((B,), S, dtype=torch.int32, device=DEV)
    caches = inf.allocate_caches(B, S + 8)
    lg = inf._prefill(ids, enc, caches)
    full = train.engine.forward_logits(ids)[:, -1].float()
    e0 = ((lg.float() - full).abs().max() / full.abs().max()).item()
    print(f"[{width} {cache}] prefill logits vs training path: {e0:.2e}")
    assert e0 < PREFILL_LOGITS_TOL, e0
    seq, lens = ids, enc.clone()
    for step in range(3):
        nxt = lg.float().argmax(-1)
        seq = torch.cat([seq, nxt[:, None]], dim=1)
        lg = inf._decode(nxt, lens, caches)
        lens += 1
        ref = train.engine.forward_logits(seq)[:, -1].float()
        err = ((lg.float() - ref).abs().max() / ref.abs().max()).item()
        top2 = ref.topk(2, dim=-1).values
        decisive = (top2[:, 0] - top2[:, 1]) > 4 * err * ref.abs().max()
        print(f"[{width} {cache}] decode step {step}: {err:.2e}, decisive {decisive.float().mean().item():.2f}")
        assert err < 2e-2, (step, err)
        assert bool((lg.float().argmax(-1) == ref.argmax(-1))[decisive].all())
        assert decisive.float().mean().item() >= 0.4
