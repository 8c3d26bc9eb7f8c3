"""The static int8 paged KV cache at serving scale, against fp64 and against a fake-quantised reference forward.

The uint8 form of the bulk decode-attention kernel has its own chunk geometry (4 KB chunks in an 8-stage ring: 32-row chunks
at d = 128, 64-row chunks spanning two 32-row pages at d = 64) and its own scale folding (o_k into the query scale, o_v on
the merged output and on every split partial).  It is checked per (sequence, head) against fp64 attention over the
dequantised pages at every preset GQA ratio, over every length 0 .. 131 (0 .. 200 at d = 64) with 0 .. 64 splits, at 32k rows,
at the decode benchmark's shape and at 256 and 1 024 slots.  Every kv head has its own scales, from absmax ~1e-3 to ~1e3;
the queries of a group are scaled against its K scale so that its scores stay O(1) (a score of size 1e3 would make fp32
rounding, not the kernel, the error).  A uint8 pool cannot hold NaN: rows past each length and pages no table references
hold random bytes, which the per-element bound rejects if read (the checker's CPU tests show it for bf16 garbage).

The cache writers are checked byte for byte against the restatement of their bf16 twins' values at every preset's head
layout and at batch 1 .. 1 024, with ties and clamps planted in every kv head; every byte outside the rows a call writes
must keep its value (assert_pool_bytes, the uint8 stand-in for the NaN checks; its CPU test shows it catches one byte).
append_attention_c8 is checked per (row, head) over many 128-row kv tiles and a long unaligned prefix, and on a 256-slot
serving step (a uint8 port of the bf16 serving-step test) with recycled pages, idle slots and 7 forced splits; the rows
each call appends equal its bf16 twin's rows quantised, byte for byte, and no other byte changes.

Two-layer models at the benchmark widths run prefill and three decode steps against oracle/llama_ref.model_forward with
kv_quant (the fake-quantised forward), with calibrated scales times distinct per-(layer, head) factors in [0.5, 4]; the same
tolerance must reject four sabotaged references.  continuous_generate runs at serving widths, teacher-forced against the same
reference, with every row it must not read set to 0xFF before every append_attention call.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, over every case below (the tests print these):
  decode attention   worst element error / bound 0.996 (the half-ulp term), c_need <= 1.2e-7 (the d = 64 length sweep;
                     3.6e-8 at 32k rows, 8.4e-8 at 1 024 slots), worst (sequence, head) rel. error 2.5e-3: the bf16 kernels'
                     DECODE_C = 4e-7 and HEAD_TOL = 4e-3 hold, with no larger c at 32k rows or 1 024 slots
  append_attention   prompt rows c_need <= 3.5e-3, (row, head) error <= 4.0e-3 (the serving step; PREFILL_C 1e-2,
                     PREFILL_HEAD_TOL 6e-3); decode rows c_need <= 7.9e-8, (row, head) error <= 2.5e-3
  models             max|diff| / max|ref| against the fake-quantised reference <= 1.61e-2 (Llama-3.2-3B width, append_attn);
                     the sabotaged references miss by 4.2e-2 at least (layer scales swapped, tied Llama-3.2-3B width) and
                     by 8.7e-2 or more at every untied width.  Per width, worst / MODEL_TOL is 0.21 .. 0.65 and the
                     nearest sabotage / MODEL_TOL 1.68 (tied Llama-3.2-3B) .. 4.07; the test prints both
  continuous_generate  worst gap / TAU 0.79 (Llama-3.2-1B width, 192 slots, 1 pre-emption and recovery) and 0.64
                     (Qwen2-1.5B width, 64 slots, 32 pre-emptions), graph or eager run, over two runs; decisive fraction
                     0.81 and 0.76
The whole file takes about 2 minutes there.
"""
import math
import time

import pytest
import torch

from oracle import cachekv_int8_ref as C
from oracle import llama_ref as R
from test_continuous_batching_at_scale_gpu import (APPEND_CASES, GEN_WIDTHS, TAU, _gen_requests, _serving_layout,
                                                  teacher_forced_check)
from test_decode_attention_at_scale_gpu import (DECODE_C, GQA, HEAD_TOL, PREFILL_C, PREFILL_HEAD_TOL, WIDTHS,
                                                assert_attention_close)
from test_decode_step_gpu import PRESETS

DEV = "cuda:0"
BF16 = torch.bfloat16
U8 = torch.uint8
# Model logits against the fake-quantised reference, max|diff| / max|ref| over prefill and three decode steps: measured worst
# 1.61e-2 (bf16 rounding points and GEMM summation orders, as in the bf16-cache width test, plus the odd cache byte that a
# one-ulp difference in K moves by one step).  The smallest error of a sabotaged reference is 4.2e-2, so the bound sits
# between them (1.55x the worst, 0.6x the nearest sabotage) rather than at 3-5x: the sabotage assertions show it is tight.
MODEL_TOL = 2.5e-2


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


def _g(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ----------------------------------------------------------------------------------------------------------
# Pool snapshot check (CPU-tested below)
# ----------------------------------------------------------------------------------------------------------
def assert_pool_bytes(after, before, live, want, what):
    """A uint8 pool after a call: at the live rows (bool [nb, bs], every kv head and column) the bytes `want`, everywhere
    else the bytes of the snapshot `before`.  after / before / want [nb, kvh, bs, d]."""
    m = live[:, None, :, None].expand_as(after)
    expect = torch.where(m, want, before)
    diff = after != expect
    if bool(diff.any()):
        i = diff.nonzero()[0].tolist()
        where = "a live row" if bool(m[tuple(i)]) else "outside the live rows"
        raise AssertionError(f"{what}: {int(diff.sum())} bytes differ ({int((diff & ~m).sum())} outside the live rows), first "
                             f"at {i} ({where}): {int(after[tuple(i)])} vs {int(expect[tuple(i)])}")


def test_pool_check_catches_one_stray_byte():
    g = torch.Generator().manual_seed(3)
    before = torch.randint(0, 256, (6, 2, 32, 64), generator=g, dtype=torch.int32).to(U8)
    live = torch.zeros(6, 32, dtype=torch.bool)
    live[2, :17] = True
    live[4, 31] = True
    want = torch.randint(0, 256, before.shape, generator=g, dtype=torch.int32).to(U8)
    after = torch.where(live[:, None, :, None], want, before)
    assert_pool_bytes(after, before, live, want, "correct")
    for at in [(2, 1, 17, 0), (4, 0, 30, 63), (0, 0, 0, 0), (5, 1, 31, 63)]:        # the row after a run, the row before, ...
        bad = after.clone()
        bad[at] ^= 1
        with pytest.raises(AssertionError, match="outside the live rows"):
            assert_pool_bytes(bad, before, live, want, "stray byte")
    bad = after.clone()
    bad[2, 1, 16, 5] ^= 0x80                                                          # a live byte written wrong
    with pytest.raises(AssertionError, match="a live row"):
        assert_pool_bytes(bad, before, live, want, "live byte")


# ----------------------------------------------------------------------------------------------------------
# Scales and pools
# ----------------------------------------------------------------------------------------------------------
# Powers of two: s = 2^e, o = 2^-e exactly, so a tie (k + 1/2) 2^-e and a clamp 300 2^-e are exact bf16 values of every head.
# absmax = 127 2^-e: 2^17 ~ 9.7e-4, 2^-3 ~ 1016.
K_EXP = [17, -3, 0, 5, -1, 2, 9, -2]
V_EXP = [-3, 17, 3, -2, 6, 0, -5, 1]


def _pow2_scales(exps, kvh, shift=0):
    e = torch.tensor([exps[(h + shift) % len(exps)] for h in range(kvh)], dtype=torch.float64)
    return (2.0 ** e).to(BF16).to(DEV), (2.0 ** -e).to(BF16).to(DEV)


def _absmax(s):
    return 127.0 / s.double()


def _random_pool(nb, kvh, bs, d, seed):
    g = _g(seed)
    return (torch.randint(0, 256, (nb, kvh, bs, d), generator=g, device=DEV, dtype=torch.int32).to(U8),
            torch.randint(0, 256, (nb, kvh, bs, d), generator=g, device=DEV, dtype=torch.int32).to(U8))


def _c8_paged(seq_lens, kvh, d, bs, mb, seed, spare=7):
    """Random-byte pools with shuffled tables: sequence b owns ceil(T / bs) pages (T = min(seq_lens + 1, mb bs)), its table
    entries past them are -1; every other byte (rows past T, unreferenced pages) is random too."""
    B = len(seq_lens)
    T = [max(0, min(int(x) + 1, mb * bs)) for x in seq_lens]
    need = [(t + bs - 1) // bs for t in T]
    nb = sum(need) + spare
    k8, v8 = _random_pool(nb, kvh, bs, d, seed)
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed)).tolist()
    tables = torch.full((B, mb), -1, dtype=torch.int32)
    i = 0
    for b in range(B):
        tables[b, :need[b]] = torch.tensor(perm[i:i + need[b]], dtype=torch.int32)
        i += need[b]
    return k8, v8, tables.to(DEV), T


def _decode_c8_case(nh, kvh, d, seq_lens, cap, bs, seed, splits=0, what=""):
    """decode_attention_paged over uint8 pages with per-head scales, per (sequence, head) against fp64."""
    o = ops()
    B = len(seq_lens)
    mb = (cap + bs - 1) // bs
    k8, v8, tables, T = _c8_paged(seq_lens, kvh, d, bs, mb, seed)
    s_k, o_k = _pow2_scales(K_EXP, kvh, seed)
    s_v, o_v = _pow2_scales(V_EXP, kvh, seed)
    G = nh // kvh
    qkv = torch.randn(B, (nh + 2 * kvh) * d, generator=_g(seed + 1), device=DEV)
    # scores O(1) whatever the K scale: query heads of kv head h scaled by 2 / absmax_k[h]
    qs = (2.0 / _absmax(s_k)).float().repeat_interleave(G * d)
    qkv[:, :nh * d] *= qs
    qkv = qkv.to(BF16)
    lens = torch.tensor(seq_lens, dtype=torch.int32, device=DEV)
    out = torch.full((B, nh * d), float("nan"), dtype=BF16, device=DEV)
    o.decode_attention_paged(qkv, k8, v8, tables, lens, nh, out=out, num_splits=splits, cache_k_out_scale=o_k,
                             cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    ok, ov = o_k.view(1, -1, 1, 1), o_v.view(1, -1, 1, 1)

    def rows(b):
        if T[b] == 0:
            z = torch.zeros(kvh, 0, d, dtype=torch.float64, device=DEV)
            return z, z
        pages = tables[b, :(T[b] + bs - 1) // bs].long()
        kk = C.dequantize(k8[pages], ok).transpose(0, 1).reshape(kvh, -1, d)[:, :T[b]]
        vv = C.dequantize(v8[pages], ov).transpose(0, 1).reshape(kvh, -1, d)[:, :T[b]]
        return kk, vv
    q = qkv[:, :nh * d].reshape(B, nh, d)
    return assert_attention_close(out, q, rows, c=DECODE_C, head_tol=HEAD_TOL,
                                  what=f"c8 {what} d={d} nh={nh} kvh={kvh} bs={bs} splits={splits}")


# ----------------------------------------------------------------------------------------------------------
# 1. decode attention over uint8 pages
# ----------------------------------------------------------------------------------------------------------
C8_GQA = [(nh, kvh, 128) for nh, kvh in GQA] + [(32, 8, 64), (14, 2, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("nh,kvh,d", C8_GQA)
def test_c8_decode_every_gqa_ratio(nh, kvh, d):
    """Ragged lengths over several chunks: no row at all, no history, a full table and one clamped past it; auto and 3 splits."""
    cap = 1100
    seq_lens = [-1, 0, cap - 1, cap + 40, 31, 32, 63, 64, 127, 128, 700]
    for splits in (0, 3):
        _decode_c8_case(nh, kvh, d, seq_lens, cap, 64, seed=nh * 100 + kvh + d + splits, splits=splits, what="gqa")


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [0, 1, 2, 3, 7, 64])
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("nh,kvh,d", [(24, 8, 128), (32, 8, 64)])
def test_c8_decode_length_sweep(nh, kvh, d, bs, splits):
    """Every attended length 0 .. 131 at d = 128 (32-row chunks) and 0 .. 201 at d = 64 (64-row chunks over 32-row pages),
    plus a full and a clamped cache."""
    top = 131 if d == 128 else 201
    cap = 256
    seq_lens = list(range(-1, top)) + [cap - 1, cap + 9]
    _decode_c8_case(nh, kvh, d, seq_lens, cap, bs, seed=splits * 7 + bs + d, splits=splits, what="sweep")


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [0, 1, 7, 64])
@pytest.mark.parametrize("B", [1, 3, 5])
@pytest.mark.parametrize("nh,kvh", [(12, 2), (32, 8)])
def test_c8_decode_long_cache(nh, kvh, B, splits):
    """32k - 1, 32k and 32k + 1 attended rows, a full cache and one clamped past it, over 128-row pages."""
    cap = 32768 + 128
    seq_lens = [32767, 32766, 32768, cap - 1, cap + 100][:B]
    _decode_c8_case(nh, kvh, 128, seq_lens, cap, 128, seed=B * 10 + splits + nh, splits=splits, what="long")


@pytest.mark.gpu
def test_c8_decode_benchmark_shape():
    seq_lens = torch.linspace(127, 2046, 64).round().int().tolist()
    _decode_c8_case(32, 8, 128, seq_lens, 2048, 64, seed=8, what="benchmark shape")


@pytest.mark.gpu
@pytest.mark.parametrize("B,d", [(256, 128), (1024, 128), (1024, 64)])
def test_c8_decode_serving_widths(B, d):
    """256 and 1 024 slots at kvh = 8 (grids of up to 8 192 CTAs); lengths up to 2 047 (1 023 at 1 024 slots, which keeps
    the pools near 1 GiB), some slots empty."""
    top = 2047 if B == 256 else 1023
    seq_lens = torch.linspace(-1, top, B).round().int().tolist()
    seq_lens[5] = seq_lens[B // 2] = -1
    _decode_c8_case(32, 8, d, seq_lens, top + 1, 64, seed=B + d, what="serving")


# ----------------------------------------------------------------------------------------------------------
# 2. the cache writers, byte for byte, with the pool snapshot rule
# ----------------------------------------------------------------------------------------------------------
TIES = [0.5, 1.5, 2.5, -2.5, 100.5, 101.5, 126.5, 127.5, 300.0, -300.0, 0.0, -0.0, 64.5, -65.5, 3.5, 4.5]


def _projection(rows, nh, kvh, d, s_k, s_v, seed, plant_k=False):
    """Packed projection whose K and V columns of kv head h have std ~ absmax_h / 3 (head 1's V: 2 absmax_h, so it clamps),
    with ties and clamps (TIES / s_h) planted into the V columns of every kv head (and the K columns with plant_k) every
    7th row."""
    g = _g(seed)
    x = torch.randn(rows, (nh + 2 * kvh) * d, generator=g, device=DEV)
    for part, s in ((1, s_k), (2, s_v)):
        a = _absmax(s).float()
        std = a / 3
        if part == 2 and kvh > 1:
            std[1] = 2 * a[1]
        c0 = (nh + (part - 1) * kvh) * d
        x[:, c0:c0 + kvh * d] *= std.repeat_interleave(d)
        if part == 2 or plant_k:
            ties = torch.tensor(TIES, device=DEV).repeat(d // 16)
            for h in range(kvh):
                x[::7, c0 + h * d:c0 + (h + 1) * d] = ties / s[h].float()
    return x.to(BF16)


def _tables_for(B, mb, nb, seed):
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))[:B * mb]
    return perm.view(B, mb).to(torch.int32).to(DEV)


def _live(tables, starts, stops, nb, bs):
    """bool [nb, bs]: rows starts[b] .. stops[b]-1 of sequence b (rows past the table are not written)."""
    live = torch.zeros(nb, bs, dtype=torch.bool)
    tl = tables.cpu()
    mb = tl.shape[1]
    for b, (a, e) in enumerate(zip(starts, stops)):
        for p in range(a, min(e, mb * bs)):
            live[int(tl[b, p // bs]), p % bs] = True
    return live.to(DEV)


def _writer_pools(nb, kvh, bs, d, seed):
    g = _g(seed)
    kb = torch.randn(nb, kvh, bs, d, generator=g, device=DEV).to(BF16)
    vb = torch.randn(nb, kvh, bs, d, generator=g, device=DEV).to(BF16)
    k8, v8 = _random_pool(nb, kvh, bs, d, seed + 1)
    return kb, vb, k8, v8, k8.clone(), v8.clone()


def _check_writer(k8, v8, k8_0, v8_0, kb, vb, s_k, s_v, live, what):
    assert_pool_bytes(k8, k8_0, live, C.quantize(kb, s_k.view(1, -1, 1, 1)), what + " K")
    assert_pool_bytes(v8, v8_0, live, C.quantize(vb, s_v.view(1, -1, 1, 1)), what + " V")


def _positions(B, mb, bs, seed):
    """Page edges, the table's first and last row, then random rows."""
    special = [mb * bs - 1, 0, bs - 1, bs, 2 * bs - 1, 2 * bs, mb * bs - bs, mb * bs - 2]
    g = torch.Generator().manual_seed(seed)
    rnd = torch.randint(0, mb * bs, (max(0, B - len(special)),), generator=g).tolist()
    return (special + rnd)[:B]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 64, 256, 1024])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_c8_writers_every_head_layout(preset, B):
    """write_cache_kv_paged, decode_rope_append_paged (bf16 and fp32-workspace forms) and append_attention at the preset's
    (nh, kvh, d): each uint8 pool equals C.quantize of the bf16 twin's pool at the rows the call writes and its snapshot
    everywhere else."""
    o = ops()
    p = PRESETS[preset]
    nh, kvh, d = p["nh"], p["kvh"], p["d"]
    ld = (nh + 2 * kvh) * d
    bs, mb = (64, 3) if B <= 64 else (32, 2)
    nb = B * mb + 5
    tables = _tables_for(B, mb, nb, B + nh)
    s_k, o_k = _pow2_scales(K_EXP, kvh, 1)
    s_v, o_v = _pow2_scales(V_EXP, kvh, 2)
    cos, sin = o.rope_tables(d, mb * bs + 8, p["theta"], DEV)
    seed = B * 31 + nh + d

    # prompts: lengths 0 .. S, the whole table among them
    S = mb * bs
    lens = torch.randint(0, S + 1, (B,), generator=torch.Generator().manual_seed(seed)).to(torch.int32)
    lens[0] = S
    if B > 2:
        lens[1], lens[2] = 0, bs
    qkv = _projection(B * S, nh, kvh, d, s_k, s_v, seed, plant_k=True)
    kb, vb, k8, v8, k8_0, v8_0 = _writer_pools(nb, kvh, bs, d, seed)
    o.write_cache_kv_paged(qkv, kb, vb, tables, lens.to(DEV), B, S, nh)
    o.write_cache_kv_paged(qkv, k8, v8, tables, lens.to(DEV), B, S, nh, cache_k_scale=s_k, cache_v_scale=s_v)
    torch.cuda.synchronize()
    live = _live(tables, [0] * B, lens.tolist(), nb, bs)
    _check_writer(k8, v8, k8_0, v8_0, kb, vb, s_k, s_v, live, f"{preset} B={B} write_cache_kv_paged")
    del qkv

    # one decode row per sequence at page edges and the table's last row
    pos = _positions(B, mb, bs, seed)
    live = _live(tables, pos, [x + 1 for x in pos], nb, bs)
    posd = torch.tensor(pos, dtype=torch.int32, device=DEV)
    for form in ("bf16", "f32"):
        kb, vb, k8, v8, k8_0, v8_0 = _writer_pools(nb, kvh, bs, d, seed + 3)
        if form == "bf16":
            x = _projection(B, nh, kvh, d, s_k, s_v, seed + 4)
            xa, xb = x.clone(), x.clone()
            o.decode_rope_append_paged(xa, kb, vb, tables, cos, sin, posd, nh)
            o.decode_rope_append_paged(xb, k8, v8, tables, cos, sin, posd, nh, cache_k_scale=s_k, cache_v_scale=s_v)
        else:
            acc = _projection(B, nh, kvh, d, s_k, s_v, seed + 5).float()
            bias = (0.01 * torch.randn(ld, generator=_g(seed + 6), device=DEV)).to(BF16).float()
            bias[(nh + kvh) * d:] = 0                                  # the planted V values reach the cache unchanged
            a1, a2 = acc.clone(), acc.clone()
            xa = o.decode_rope_append_paged(None, kb, vb, tables, cos, sin, posd, nh, acc_f32=a1, bias=bias)
            xb = o.decode_rope_append_paged(None, k8, v8, tables, cos, sin, posd, nh, acc_f32=a2, bias=bias,
                                            cache_k_scale=s_k, cache_v_scale=s_v)
            torch.cuda.synchronize()
            assert not bool(a2.any()), "the fp32 workspace is handed back zeroed"
        torch.cuda.synchronize()
        assert torch.equal(xa, xb), f"{preset} B={B} decode_rope_append_paged ({form}): the rotated projection differs"
        _check_writer(k8, v8, k8_0, v8_0, kb, vb, s_k, s_v, live, f"{preset} B={B} decode_rope_append_paged ({form})")

    # append_attention: decode rows at the positions above, a prompt chunk in slot 0 and an idle slot 1 with a stale length
    n = [1] * B
    enc, dec = [0] * B, list(pos)
    dec[0] = bs - 2
    n[0] = enc[0] = min(bs + 3, mb * bs - dec[0])
    if B > 2:
        n[1], enc[1], dec[1] = 0, 0, 2 * bs - 1
    this = torch.tensor(n, dtype=torch.int32, device=DEV)
    cu = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    x = _projection(sum(n), nh, kvh, d, s_k, s_v, seed + 7)
    kb, vb, k8, v8, k8_0, v8_0 = _writer_pools(nb, kvh, bs, d, seed + 8)
    encd, decd = torch.tensor(enc, dtype=torch.int32, device=DEV), torch.tensor(dec, dtype=torch.int32, device=DEV)
    xa, xb = x.clone(), x.clone()
    o.append_attention(xa, kb, vb, encd, decd, this, cu, tables, cos, sin, nh, max_q_len=max(n))
    o.append_attention(xb, k8, v8, encd, decd, this, cu, tables, cos, sin, nh, max_q_len=max(n), cache_k_scale=s_k,
                       cache_v_scale=s_v, cache_k_out_scale=o_k, cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    assert torch.equal(xa, xb), f"{preset} B={B} append_attention: the rotated projection differs"
    live = _live(tables, dec, [a + b for a, b in zip(dec, n)], nb, bs)
    _check_writer(k8, v8, k8_0, v8_0, kb, vb, s_k, s_v, live, f"{preset} B={B} append_attention")


def _c8_qkv(T, nh, kvh, d, s_k, s_v, seed):
    """A projection of T rows for append_attention_c8: K / V columns as _projection, q scaled per group as in the decode
    cases (O(1) scores at every K scale)."""
    x = _projection(T, nh, kvh, d, s_k, s_v, seed).float()
    x[:, :nh * d] = torch.randn(T, nh * d, generator=_g(seed + 1), device=DEV) * (
        2.0 / _absmax(s_k).float()).repeat_interleave((nh // kvh) * d)
    return x.to(BF16)


def _c8_append_checked(x, k8, v8, enc, dec, this, cu, tables, cos, sin, nh, max_q_len, scales, splits, live, what):
    """append_attention_c8 on x (rotated in place) into a NaN-filled output, which it returns, with its writes checked: x
    rotated as the bf16 twin (same call on zero bf16 pools) rotates it, the live rows' bytes C.quantize of the rows the twin
    appends, every other byte as before the call."""
    o = ops()
    s_k, o_k, s_v, o_v = scales
    nb, kvh, bs, d = k8.shape
    kb = torch.zeros(k8.shape, dtype=BF16, device=DEV)
    vb = torch.zeros(k8.shape, dtype=BF16, device=DEV)
    k8_0, v8_0 = k8.clone(), v8.clone()
    xb = x.clone()
    o.append_attention(xb, kb, vb, enc, dec, this, cu, tables, cos, sin, nh, max_q_len=max_q_len, num_splits=splits)
    out = torch.full((x.shape[0], nh * d), float("nan"), dtype=BF16, device=DEV)
    o.append_attention(x, k8, v8, enc, dec, this, cu, tables, cos, sin, nh, max_q_len=max_q_len, out=out,
                       num_splits=splits, cache_k_scale=s_k, cache_v_scale=s_v, cache_k_out_scale=o_k,
                       cache_v_out_scale=o_v)
    torch.cuda.synchronize()
    assert torch.equal(x, xb), f"{what}: the rotated projection differs from the bf16 twin's"
    _check_writer(k8, v8, k8_0, v8_0, kb, vb, s_k, s_v, live, what)
    return out


def _dequantized_rows(k8, v8, o_k, o_v, tables, b, L):
    """Rows 0 .. L-1 of sequence b, dequantised to fp64: K, V [kvh, L, d]."""
    nb, kvh, bs, d = k8.shape
    pages = tables[b, :(L + bs - 1) // bs].long()
    return (C.dequantize(k8[pages], o_k.view(1, -1, 1, 1)).transpose(0, 1).reshape(kvh, -1, d)[:, :L],
            C.dequantize(v8[pages], o_v.view(1, -1, 1, 1)).transpose(0, 1).reshape(kvh, -1, d)[:, :L])


# ----------------------------------------------------------------------------------------------------------
# 3. append_attention_c8: prompt rows over many kv tiles and a long unaligned prefix
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("d,nh,kvh", [(64, 32, 8), (64, 14, 2), (128, 24, 8), (128, 12, 2)])
def test_c8_append_attention_long_prompts(d, nh, kvh, bs):
    """One call: a 300-row prompt (three q tiles), a 1 000-row chunk over a 3 000-row cached prefix (aligned to neither 128
    nor the page), an 8 192-row prompt (64 kv tiles) and a decode row on a 2 000-row history.  Every row of the first two,
    the decode row and every 29th row plus the last 130 rows of the long prompt against fp64 over the dequantised pages the
    call leaves.  The bytes of every row the call appends (up to position 8 191) equal C.quantize of the rows its bf16 twin
    appends, and every other byte keeps its value."""
    o = ops()
    chunks = [(0, 300), (3000, 1000), (0, 8192), (2000, 1)]               # (cached, new)
    B = len(chunks)
    mb = (8192 + bs - 1) // bs
    nb = B * mb + 3
    tables = _tables_for(B, mb, nb, bs + d + nh)
    k8, v8 = _random_pool(nb, kvh, bs, d, bs + nh)
    s_k, o_k = _pow2_scales(K_EXP, kvh, 3)
    s_v, o_v = _pow2_scales(V_EXP, kvh, 3)
    ld = (nh + 2 * kvh) * d
    T = sum(n for _, n in chunks)
    x = _c8_qkv(T, nh, kvh, d, s_k, s_v, bs + 5)
    enc = torch.tensor([n if n > 1 else 0 for _, n in chunks], dtype=torch.int32, device=DEV)
    dec = torch.tensor([c for c, _ in chunks], dtype=torch.int32, device=DEV)
    this = torch.tensor([n for _, n in chunks], dtype=torch.int32, device=DEV)
    cu = [0]
    for _, n in chunks:
        cu.append(cu[-1] + n)
    cos, sin = o.rope_tables(d, mb * bs, 10000.0, DEV)
    live = _live(tables, [c for c, _ in chunks], [c + n for c, n in chunks], nb, bs)
    out = _c8_append_checked(x, k8, v8, enc, dec, this, torch.tensor(cu, dtype=torch.int32, device=DEV), tables, cos, sin,
                             nh, 8192, (s_k, o_k, s_v, o_v), 0, live, f"append_attention_c8 d={d} nh={nh} bs={bs}")
    ok, ov = o_k.view(1, -1, 1, 1), o_v.view(1, -1, 1, 1)
    seq = {}

    def seq_rows(b):
        if b not in seq:
            L = chunks[b][0] + chunks[b][1]
            pages = tables[b, :(L + bs - 1) // bs].long()
            seq[b] = (C.dequantize(k8[pages], ok).transpose(0, 1).reshape(kvh, -1, d),
                      C.dequantize(v8[pages], ov).transpose(0, 1).reshape(kvh, -1, d))
        return seq[b]

    q = x[:, :nh * d].reshape(T, nh, d)                                      # rotated in place by the call
    for kind, c, tol in (("prompt", PREFILL_C, PREFILL_HEAD_TOL), ("decode", DECODE_C, HEAD_TOL)):
        idx, where = [], []
        for b, (cached, n) in enumerate(chunks):
            if (n == 1) != (kind == "decode"):
                continue
            picks = range(n) if n <= 1000 else sorted(set(range(0, n, 29)) | set(range(n - 130, n)))
            for i in picks:
                idx.append(cu[b] + i)
                where.append((b, cached + i))

        def rows(m):
            b, pos = where[m]
            K, V = seq_rows(b)
            return K[:, :pos + 1], V[:, :pos + 1]
        sel = torch.tensor(idx, device=DEV)
        assert_attention_close(out[sel], q[sel], rows, c=c, head_tol=tol,
                               what=f"append_attention_c8 {kind} rows d={d} nh={nh} kvh={kvh} bs={bs}")


@pytest.mark.gpu
@pytest.mark.parametrize("d,nh,kvh,bs", APPEND_CASES)
def test_c8_append_attention_serving_step(d, nh, kvh, bs):
    """The uint8 port of test_continuous_batching_at_scale_gpu.test_append_attention_serving_step: one 256-slot step with
    prompts at every q-tile and page edge admitted into pages recycled from retired requests (which still hold those
    requests' bytes), a 100-row chunk on a 150-row prefix, 234 decode rows over histories up to 2 048 rows, and idle slots
    in the middle and at the end with stale decode lengths.  At automatic and 7 splits, every (row, head) against fp64 over
    the dequantised pages, and the pools by the snapshot rule: the appended rows are the bf16 twin's rows quantised, every
    other byte (rows past each length, the recycled pages' stale rows, unreferenced pages) keeps its value."""
    o = ops()
    seed = d + nh + bs
    lay = _serving_layout(bs, seed)
    B = len(lay)
    mb = 2048 // bs + 1
    prev_pages = [math.ceil((c + n) / bs) if k in ("decode", "chunk") else math.ceil(h / bs) for k, c, n, h in lay]
    new_pages = [math.ceil((c + n) / bs) if k == "prompt" else 0 for k, c, n, _ in lay]
    nb = sum(prev_pages) + sum(new_pages) + 9
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed)).tolist()
    tables = torch.full((B, mb), -1, dtype=torch.int32)
    i = 0
    for b in range(B):
        tables[b, :prev_pages[b]] = torch.tensor(perm[i:i + prev_pages[b]], dtype=torch.int32)
        i += prev_pages[b]
    unused = perm[i:]
    k8, v8 = _random_pool(nb, kvh, bs, d, seed)               # every history row, and every other byte, random
    s_k, o_k = _pow2_scales(K_EXP, kvh, seed)
    s_v, o_v = _pow2_scales(V_EXP, kvh, seed + 1)
    cos, sin = o.rope_tables(d, 4096, 10000.0, DEV)

    def args(chunks):
        n = [c[2] for c in chunks]
        enc = torch.tensor([x if k in ("prompt", "chunk") else 0 for k, _, x in chunks], dtype=torch.int32, device=DEV)
        dec = torch.tensor([c[1] for c in chunks], dtype=torch.int32, device=DEV)
        cu = [0]
        for x in n:
            cu.append(cu[-1] + x)
        return n, enc, dec, torch.tensor(n, dtype=torch.int32, device=DEV), cu

    # the step before: decode slots append row (cached - 1), the chunk slot runs its prefix as a prompt, the slots whose
    # request retires after it (prompt slots of the checked step, idle slots) decode their last row
    prev = [("prompt", 0, h) if k == "chunk" else ("decode", h - 1, 1) for k, c, n, h in lay]
    n, enc, dec, this, cu = args(prev)
    o.append_attention(_c8_qkv(sum(n), nh, kvh, d, s_k, s_v, seed + 2), k8, v8, enc, dec, this,
                       torch.tensor(cu, dtype=torch.int32, device=DEV), tables.to(DEV), cos, sin, nh, max_q_len=max(n),
                       num_splits=7, cache_k_scale=s_k, cache_v_scale=s_v, cache_k_out_scale=o_k, cache_v_out_scale=o_v)
    # retire: the retired slots' pages keep their bytes and go to the admitted prompts first
    recycled = []
    for b, (k, c, n_, h) in enumerate(lay):
        if k in ("prompt", "idle"):
            recycled += [int(x) for x in tables[b] if x >= 0]
            tables[b] = -1
    pool = recycled + unused
    for b, (k, c, n_, h) in enumerate(lay):
        if k == "prompt":
            tables[b, :new_pages[b]] = torch.tensor(pool[:new_pages[b]], dtype=torch.int32)
            pool = pool[new_pages[b]:]
    assert len(recycled) > sum(new_pages) // 2
    chunks = [(k, c, n_) for k, c, n_, _ in lay]
    n, enc, dec, this, cu = args(chunks)
    tdev = tables.to(DEV)
    cud = torch.tensor(cu, dtype=torch.int32, device=DEV)
    live = _live(tdev, [c for _, c, _ in chunks], [c + x if k != "idle" else c for k, c, x in chunks], nb, bs)
    qkv0 = _c8_qkv(sum(n), nh, kvh, d, s_k, s_v, seed + 3)
    base_k, base_v = k8.clone(), v8.clone()
    for splits in (0, 7):
        k8.copy_(base_k)
        v8.copy_(base_v)
        qkv = qkv0.clone()
        out = _c8_append_checked(qkv, k8, v8, enc, dec, this, cud, tdev, cos, sin, nh, max(n), (s_k, o_k, s_v, o_v), splits,
                                 live, f"c8 serving step d={d} nh={nh} kvh={kvh} bs={bs} splits={splits}")
        seq = {}

        def seq_rows(b):
            if b not in seq:
                seq[b] = _dequantized_rows(k8, v8, o_k, o_v, tdev, b, chunks[b][1] + chunks[b][2])
            return seq[b]

        checked = 0
        for kind, c, tol in (("decode", DECODE_C, HEAD_TOL), ("prompt", PREFILL_C, PREFILL_HEAD_TOL)):
            idx, where = [], []
            for b, (k, cached, x) in enumerate(chunks):
                if k != "idle" and (k == "decode") == (kind == "decode"):
                    for j in range(x):
                        idx.append(cu[b] + j)
                        where.append((b, cached + j))

            def rows(m):
                b, pos = where[m]
                K, V = seq_rows(b)
                return K[:, :pos + 1], V[:, :pos + 1]
            sel = torch.tensor(idx, device=DEV)
            assert_attention_close(out[sel], qkv[sel, :nh * d].reshape(len(idx), nh, d), rows, c=c, head_tol=tol,
                                   what=f"c8 serving step {kind} rows d={d} nh={nh} kvh={kvh} bs={bs} splits={splits}")
            checked += len(idx)
        assert checked == out.shape[0]


# ----------------------------------------------------------------------------------------------------------
# 4. models against the fake-quantised reference forward
# ----------------------------------------------------------------------------------------------------------
MODEL_WIDTHS = dict(WIDTHS)
MODEL_WIDTHS["llama3_2_1b"] = dict(model_type="llama", tied=False, hidden_size=2048, intermediate_size=8192,
                                   num_attention_heads=32, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0)


def _factors(L, kvh, seed):
    """Distinct per-(layer, kv head) factors in [0.5, 4], 0.5 among them (it engages the clamp)."""
    f = torch.linspace(0.5, 4.0, L * kvh, dtype=torch.float64)
    return f[torch.randperm(L * kvh, generator=torch.Generator().manual_seed(seed))].view(L, kvh)


def _width_model(spec, *, append_attn, block_size=64, scale_tied=True):
    """A two-layer model at a preset width with an int8 cache (as test_benchmark_width_decode_matches_uncached_forward builds
    its bf16 twin), and the reference's config and weights on the device."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    spec = dict(spec)
    model_type, tied = spec.pop("model_type"), spec.pop("tied")
    kw = dict(vocab_size=4096, num_hidden_layers=2, max_position_embeddings=512, **spec)
    cfg = R.RefConfig(qkv_bias=model_type == "qwen2", model_type=model_type, **kw)
    w = R.init_weights(cfg, seed=41)
    if tied:
        w.pop("lm_head.weight")
        E = f"{model_type}.embed_tokens.weight"
        if scale_tied:
            w[E] = (w[E] * 8).to(BF16).float()
    else:
        w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(BF16).float()
    Cfg = T.Qwen2Config if model_type == "qwen2" else T.LlamaConfig
    inf = LlamaForCausalLMInferenceModel(Cfg(tie_word_embeddings=tied, **kw), block_attn=True, append_attn=append_attn,
                                         block_size=block_size, cachekv_int8_type="static")
    inf.set_state_dict(w)
    if tied:
        w["lm_head.weight"] = w[f"{model_type}.embed_tokens.weight"].t()
    return cfg, {k: v.to(DEV) for k, v in w.items()}, inf


def _set_scales(inf, calib_ids, calib_lens, seed):
    """Calibrate, then multiply every (layer, kv head) absmax by its own factor; returns the reference's per-layer scales."""
    t = inf.transformer_block
    ka, va = inf.calibrate_cache_scales(calib_ids, calib_lens)
    ka, va = ka * _factors(t.L, t.kvh, seed), va * _factors(t.L, t.kvh, seed + 1)
    t.set_cache_scales(ka, va)
    scales = []
    for i in range(t.L):
        s_k, o_k = C.scales_from_absmax(ka[i])
        s_v, o_v = C.scales_from_absmax(va[i])
        assert torch.equal(t.cache_k_scales[i].cpu(), s_k) and torch.equal(t.cache_v_out_scales[i].cpu(), o_v)
        scales.append((s_k, o_k, s_v, o_v))
    return scales


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def _prompt_rows_at_127(prompt_len):
    """fake_quant_rows of the reference's encoder-side write, for a sabotaged reference: rows at positions below
    prompt_len[b] stored at + 127 and read back at - 128 (one step o lower), later rows as the kernels store them.  The
    reference forward is called without position_ids, so a row's position is its index."""

    def rows(x, s, o):
        s, o = s.to(x.device).view(-1, 1), o.to(x.device).view(-1, 1)
        low = C.dequantize(C.quantize(x, s).to(torch.float64) - 1, o).to(x.dtype)
        early = torch.arange(x.shape[1], device=x.device)[None, :] < prompt_len.to(x.device)[:, None]
        return torch.where(early[:, :, None, None], low, C.fake_quant(x, s, o))
    return rows


def test_prompt_rows_at_127_lowers_exactly_the_prompt_rows():
    g = torch.Generator().manual_seed(2)
    x = (2 * torch.randn(3, 10, 2, 16, generator=g)).to(BF16).float()
    s, o = C.scales_from_absmax(torch.tensor([1.5, 4.0], dtype=torch.float64))
    plen = torch.tensor([0, 4, 10])
    got = _prompt_rows_at_127(plen)(x, s, o)
    want = R.fake_quant_rows(x, s, o)
    for b in range(3):
        p = int(plen[b])
        assert torch.equal(got[b, p:], want[b, p:])
        assert torch.equal(got[b, :p].double(), want[b, :p].double() - o.double().view(-1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("append_attn", [False, True])
@pytest.mark.parametrize("width", list(MODEL_WIDTHS))
def test_int8_cache_model_matches_fake_quant_reference(width, append_attn):
    """Batch 64, prompts of 120 .. 140 tokens, prefill and three decode steps of a two-layer int8-cache model against the
    fake-quantised reference forward of the grown sequences: max|diff| / max|ref| within MODEL_TOL and identical decisive
    arg-max.  The fused path attends over the projection's bf16 K / V in its prefill (quant_from = the prompt length),
    append_attention over the cache everywhere (quant_from = 0).  Each sabotaged reference must miss by more than MODEL_TOL:
    no quantisation, the two layers' scales swapped, the kv heads' scales rotated, prompt rows stored at + 127."""
    cfg, w, inf = _width_model(MODEL_WIDTHS[width], append_attn=append_attn)
    B, S = 64, 140
    g = torch.Generator().manual_seed(43)
    enc = torch.randint(120, S + 1, (B,), generator=g)
    enc[0] = S
    ids = torch.randint(0, cfg.vocab_size, (B, S), generator=g)
    scales = _set_scales(inf, ids[:16], enc[:16], seed=len(width))
    qf = torch.zeros(B, dtype=torch.int64) if append_attn else enc.clone()
    refs = {
        "int8 cache": R.KvQuant(scales, qf),
        "no quantisation": None,
        "layer scales swapped": R.KvQuant(scales[::-1], qf),
        "kv-head scales rotated": R.KvQuant([(s_k.roll(1), o_k.roll(1), s_v.roll(1), o_v.roll(1))
                                             for s_k, o_k, s_v, o_v in scales], qf),
        "prompt rows at +127": R.KvQuant(scales, qf),                  # with _prompt_rows_at_127 below
    }
    steps = 3
    caches = inf.allocate_caches(B, S + steps + 8)
    encd = enc.to(torch.int32).to(DEV)
    lg = inf._prefill(ids.to(DEV), encd, caches)
    seqs = [ids[b, :int(enc[b])].tolist() for b in range(B)]
    lens = encd.clone()
    errs = {k: [] for k in refs}
    fracs = []
    for step in range(steps + 1):
        L = max(len(s) for s in seqs)
        full = torch.tensor([s + [0] * (L - len(s)) for s in seqs], dtype=torch.int64, device=DEV)
        last = torch.tensor([len(s) - 1 for s in seqs], device=DEV)
        for name, kq in refs.items():
            with torch.no_grad(), pytest.MonkeyPatch.context() as mp:
                if name == "prompt rows at +127":
                    mp.setattr(R, "fake_quant_rows", _prompt_rows_at_127(enc))
                ref = R.model_forward(full, w, cfg, kv_quant=kq)[torch.arange(B, device=DEV), last].float()
            errs[name].append(_rel(lg.float(), ref))
            if name == "int8 cache":
                # a top-1 / top-2 margin above 2 max|diff| cannot be overturned by the measured error
                top2 = ref.topk(2, dim=-1).values
                decisive = (top2[:, 0] - top2[:, 1]) > 2 * errs[name][-1] * ref.abs().max()
                assert bool((lg.float().argmax(-1) == ref.argmax(-1))[decisive].all()), (width, step)
                fracs.append(decisive.float().mean().item())
        print(f"[{width} append_attn={append_attn}] step {step}: decisive {fracs[-1]:.2f}, "
              + ", ".join(f"{k} {v[-1]:.2e}" for k, v in errs.items()))
        if step == steps:
            break
        nxt = lg.float().argmax(-1)
        for b in range(B):
            seqs[b].append(int(nxt[b]))
        lg = inf._decode(nxt, lens, caches)
        lens += 1
    worst = max(errs["int8 cache"])
    nearest = min(max(v) for k, v in errs.items() if k != "int8 cache")
    print(f"[{width} append_attn={append_attn}] worst {worst:.2e} (tol {MODEL_TOL}); sabotaged references, worst step: "
          + ", ".join(f"{k} {max(v):.2e}" for k, v in errs.items() if k != "int8 cache"))
    print(f"[{width} append_attn={append_attn}] margins: worst / MODEL_TOL {worst / MODEL_TOL:.2f}, nearest sabotage / "
          f"MODEL_TOL {nearest / MODEL_TOL:.2f}")
    assert worst <= MODEL_TOL, errs["int8 cache"]
    assert min(fracs) >= 0.4, fracs
    for name, v in errs.items():
        if name != "int8 cache":
            assert max(v) > MODEL_TOL, f"the tolerance accepts the sabotaged reference '{name}': {v}"


# ----------------------------------------------------------------------------------------------------------
# 5. continuous_generate over an int8 cache at serving widths
# ----------------------------------------------------------------------------------------------------------
def _ff_poisoned(real):
    """append_attention that first sets 0xFF (the largest value, +127 o) into every page of the layer's uint8 cache no block
    table references and every referenced row at or past its slot's seq_lens_decoder + seq_lens_this_time (no host sync: the
    wrapper is captured into the decode graphs with the call)."""

    def wrapper(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q,
                block_tables, cos, sin, nh, max_q_len, **kw):
        nb, _, bs, _ = key_cache.shape
        B, mb = block_tables.shape
        held = block_tables >= 0
        page = torch.where(held, block_tables, nb).long()
        limit = (seq_lens_decoder + seq_lens_this_time).long()
        pos = torch.arange(mb * bs, device=qkv.device).view(1, mb, bs)
        stale = (pos >= limit.view(B, 1, 1)).view(B * mb, bs)
        rows = torch.ones(nb + 1, bs, dtype=torch.bool, device=qkv.device)
        rows.scatter_(0, page.view(-1, 1).expand(-1, bs), stale)
        ref = torch.zeros(nb + 1, dtype=torch.int32, device=qkv.device)
        ref.index_add_(0, page.view(-1), held.view(-1).to(torch.int32))
        rows.masked_fill_((ref == 0).view(-1, 1), True)
        mask = rows[:nb].view(nb, 1, bs, 1)
        key_cache.masked_fill_(mask, 0xFF)
        value_cache.masked_fill_(mask, 0xFF)
        return real(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q,
                    block_tables, cos, sin, nh, max_q_len, **kw)
    return wrapper


@pytest.mark.gpu
@pytest.mark.parametrize("width", list(GEN_WIDTHS))
def test_c8_continuous_generate_matches_fake_quant_reference(width, monkeypatch):
    from paddlenlp_b200 import ops as O

    spec = dict(GEN_WIDTHS[width])
    bs, B, n_req, nb = (spec.pop(k) for k in ("block_size", "max_batch_size", "num_requests", "num_blocks"))
    # the page count of the bf16 test, so the run pre-empts as often; the tied embedding stays as initialised (scaled up, the
    # model would predict its own input token whatever the context)
    cfg, w, inf = _width_model(spec, append_attn=True, block_size=bs, scale_tied=False)
    reqs = _gen_requests(n_req, cfg.vocab_size)
    calib = torch.randint(0, cfg.vocab_size, (8, 128), generator=torch.Generator().manual_seed(3))
    scales = _set_scales(inf, calib, None, seed=11)
    monkeypatch.setattr(O, "append_attention", _ff_poisoned(O.append_attention))
    t0 = time.perf_counter()
    eager, st_e = inf.continuous_generate(reqs, max_batch_size=B, num_blocks=nb, use_cuda_graph=False)
    outs, st_g = inf.continuous_generate(reqs, max_batch_size=B, num_blocks=nb)
    t1 = time.perf_counter()
    print(f"[{width}] stats {st_g}; two runs {t1 - t0:.1f} s")
    assert {k: v for k, v in st_e.items() if k != "decode_step_ms"} == {k: v for k, v in st_g.items() if k != "decode_step_ms"}
    assert st_g["free_blocks_at_exit"] == nb and bool((inf.last_block_tables == -1).all())
    assert st_g["preemptions"] > 0 and st_g["recoveries"] > 0, st_g
    kq = R.KvQuant(scales, torch.zeros(1, dtype=torch.int64))

    def fwd(ids):
        with torch.no_grad():
            return R.model_forward(ids.to(DEV)[None], w, cfg, kv_quant=kq)[0].float()
    parted = 0
    for r, ((prompt, _), a, b) in enumerate(zip(reqs, outs, eager)):
        diff = (a != b).nonzero()
        if diff.numel():
            t = int(diff[0])
            lg = fwd(torch.cat([prompt, a[:t]]))[-1].double()
            top2 = lg.topk(2).values
            assert (top2[0] - top2[1]).item() <= TAU * lg.abs().max().item(), f"request {r}: graph and eager part at {t}"
            parted += 1
    worst, frac, copy, n = teacher_forced_check(fwd, reqs, outs)
    worst_e, _, _, _ = teacher_forced_check(fwd, reqs, eager)
    print(f"[{width}] teacher-forced over {n} positions: worst gap / tau {worst:.3f} (eager {worst_e:.3f}), decisive fraction "
          f"{frac:.3f}, copy {copy:.3f}; {parted} requests part from the eager run at a near-tie; "
          f"check {time.perf_counter() - t1:.1f} s")
    assert frac >= 0.5, frac
