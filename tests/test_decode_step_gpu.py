"""The kernels of one fused decode step, and of the prefill that fills the cache, per element against fp64 and against their
unfused twins, at the decode widths of every shipped preset.

A decode step at up to SKINNY_M = 128 rows runs the fused branch of FusedMultiTransformerBase.forward: each split-K GEMM
(gemm_skinny_f32) leaves fp32 sums in a shared workspace, and the next kernel (decode_rope_append_f32 / the paged append with
acc_f32, add_rmsnorm_f32) rounds them once, adds the bias, rotates or normalises, and hands the workspace back zeroed.  The
end-to-end decode tests accept a logits error of 2e-2 of the largest logit over three steps, which cannot see a bias missing
from v, one cache row written one position late, or one fp32 partial sum left in the workspace for the next step.  The checks
here are per element (bit-exact where the kernel's rounding points are known, within one or two bf16 ulps of fp64 where they
are not), per cache row (every row that was not appended keeps its bits; rows and pages are NaN-filled beforehand) and per
workspace byte.  Outputs start as NaN: an element the kernel never writes fails.

The checkers are plain torch and have CPU tests of their own (no gpu mark): each accepts a correct result and rejects a
planted fault of the kind it exists to catch.

Presets (decode widths):      h     nh/kvh  d    qkv N  I      qkv bias
    Llama-3-8B (benchmark)    4096  32/8    128  6144   14336  no
    Llama-3.2-3B              3072  24/8    128  5120   8192   no
    Llama-3.2-1B              2048  32/8    64   3072   8192   no
    Qwen2-7B                  3584  28/4    128  4608   18944  yes
    Qwen2-1.5B                1536  12/2    128  2048   8960   yes
    Qwen2-0.5B                896   14/2    64   1152   4864   yes   (N = 896 and 1152 leave partial 256-wide tiles)
"""
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import llama_ref as R
from test_kernels_at_scale_gpu import (_rows_with_spread, assert_gemm_close, assert_rows_close, assert_within_ulps,  # noqa: F401
                                       bf16_ulp, fp64_reference)

DEV = "cuda:0"
BF16 = torch.bfloat16
EPS = 1e-5

PRESETS = {
    "llama3-8b": dict(h=4096, nh=32, kvh=8, d=128, I=14336, bias=False, theta=500000.0),
    "llama3.2-3b": dict(h=3072, nh=24, kvh=8, d=128, I=8192, bias=False, theta=500000.0),
    "llama3.2-1b": dict(h=2048, nh=32, kvh=8, d=64, I=8192, bias=False, theta=500000.0),
    "qwen2-7b": dict(h=3584, nh=28, kvh=4, d=128, I=18944, bias=True, theta=1000000.0),
    "qwen2-1.5b": dict(h=1536, nh=12, kvh=2, d=128, I=8960, bias=True, theta=1000000.0),
    "qwen2-0.5b": dict(h=896, nh=14, kvh=2, d=64, I=4864, bias=True, theta=1000000.0),
}
BATCHES = (1, 5, 64, 128)           # 64: the decode benchmark's batch; 128: SKINNY_M, the largest batch of the fused branch

# Per-element allowance for the fp32 split-K sums, times (|A| @ |B|)_ij; no bf16 term (nothing is rounded to bf16).  Measured
# on an H100 80GB HBM3 (700 W power limit) over every preset, GEMM, batch and split below: c_need <= 1.36e-6 (Qwen2-7B ffn2,
# K = 18 944; 1.0e-6 at K = 8192, <= 6.6e-7 for K <= 4096).  c is ~4x the worst.
SPLITK_C = 5.5e-6
# One decode step through the fused branch vs the unfused composition, both at the default split-K: the fp32 partial sums
# reach the workspace in a different order, so a logit of the two can round one bf16 ulp apart and the difference propagates
# through two layers.  Relative error of one hidden-state row, measured on an H100 80GB HBM3 (700 W power limit) over two
# runs (the order of the partial sums changes from run to run): Llama-3-8B 5.3e-3 .. 7.8e-3, Qwen2-1.5B 3.3e-3 .. 4.5e-3.
# The tolerance is ~4x the worst.
DEFAULT_SPLIT_ROW_TOL = 3e-2
# The kernels rotate in fp32, fma(x1, c, -(x2 * s)): two fp32 roundings of at most 2^-24 of |x1 c| + |x2 s| each.  Where the
# two products nearly cancel that is more than one bf16 ulp of the result, so the q / k check allows it on top of the ulp.
ROPE_F32_REL = 2.0 ** -23


def _seed(*parts):
    """A seed that depends only on the test's parameters (str hashes change from one interpreter to the next)."""
    return zlib.crc32(repr(parts).encode()) & 0x7FFFFFFF


def _ops():
    from paddlenlp_b200 import ops

    return ops


def _lib():
    from paddlenlp_b200 import _lib as lib

    return lib


def _gen(seed, device=DEV):
    return torch.Generator(device=device).manual_seed(seed)


def _nan(*shape, dtype=BF16, device=DEV):
    return torch.full(shape, float("nan"), dtype=dtype, device=device)


def _rope_tables(d, max_pos, theta, device):
    """fp32 cos / sin [max_pos, d/2] exactly as the model builds them."""
    return _ops().rope_tables(d, max_pos, theta, device)


# ----------------------------------------------------------------------------------------------------------
# Checkers
# ----------------------------------------------------------------------------------------------------------
def assert_same_bits(got, want, what="tensor"):
    """Bitwise equality of two bf16 tensors (NaN equals NaN); reports the first differing element."""
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    diff = got.view(torch.int16) != want.view(torch.int16)
    if bool(diff.any()):
        i = diff.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at {i}: {got[tuple(i)].item()} vs "
                             f"{want[tuple(i)].item()}")


def assert_workspace_zero(buf, what="workspace"):
    """Every byte of a split-K workspace (the whole buffer, also past the M x N a call used) is zero."""
    b = buf.contiguous().view(torch.uint8).view(-1)
    nz = b != 0
    if bool(nz.any()):
        first = int(nz.nonzero()[0])
        raise AssertionError(f"{what}: {int(nz.sum())} nonzero bytes of {b.numel()}, first at byte {first} "
                             f"(fp32 element {first // 4})")


def assert_f32_sums_close(ws, A, B, c=SPLITK_C, what="split-K sums"):
    """ws [M, N] fp32 against A [M, K] @ B [K, N] in fp64, per element: |ws - ref| <= c * (|A| @ |B|).  Returns c_need."""
    M, K = A.shape
    assert B.shape[0] == K and tuple(ws.shape) == (M, B.shape[1]), (what, tuple(ws.shape), tuple(A.shape), tuple(B.shape))
    a, b = A.double(), B.double()
    ref = a @ b
    mag = a.abs() @ b.abs()
    got = ws.double()
    err = (got - ref).abs()
    bad = ~(err <= c * mag)                              # NaN counts as bad
    c_need = (err / (mag + 1e-300)).max().item()
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond c = {c:.1e}, first at {i}: {got[tuple(i)].item()} vs "
                             f"{ref[tuple(i)].item()} (c_need {c_need:.2e})")
    return c_need


def _rounded_input(acc, bias):
    """bf16(acc + bias): the fp32 sum rounded once, the Linear output rounding of the fused kernels."""
    return (acc + bias if bias is not None else acc).to(BF16)


def assert_rope_append_qkv(qkv, acc, bias, cos, sin, seq_lens, nh, kvh, d, max_len, what="rope append"):
    """The packed projection an fp32-path append returned, against x = bf16(acc + bias):
      v columns                bit-exactly x
      q and k columns          within 1 bf16 ulp of the fp64 rotate-half of x at position seq_lens[b] (cos / sin: the fp32
                               tables the kernel reads), plus ROPE_F32_REL of the two products' magnitudes; a row whose
                               position is outside [0, max_len) is x, not rotated."""
    nq = (nh + kvh) * d
    x = _rounded_input(acc, bias)
    assert_same_bits(qkv[:, nq:], x[:, nq:], f"{what}: v columns")
    pos = seq_lens.long().to(qkv.device)
    ok = (pos >= 0) & (pos < max_len)
    if bool((~ok).any()):
        assert_same_bits(qkv[~ok, :nq], x[~ok, :nq], f"{what}: q|k of rows past the cache")
    if bool(ok.any()):
        xs = x[ok, :nq].double().view(-1, nh + kvh, d)
        c = cos.double()[pos[ok]][:, None, :]
        s = sin.double()[pos[ok]][:, None, :]
        x1, x2 = xs[..., : d // 2], xs[..., d // 2:]
        ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
        mag = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1)
        got = qkv[ok, :nq].view(-1, nh + kvh, d).double()
        err = (got - ref).abs()
        bad = ~(err <= bf16_ulp(ref) + ROPE_F32_REL * mag)             # NaN counts as bad
        if bool(bad.any()):
            i = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: rotated q|k: {int(bad.sum())} elements beyond 1 ulp, first at {i} (row, head, "
                                 f"column): {got[tuple(i)].item()} vs {ref[tuple(i)].item()}")


def expected_cache_after_append(k_before, v_before, qkv, seq_lens, nh, kvh, d, tables=None):
    """k, v caches after every sequence appended its k and v (taken from the projection `qkv` the kernel returned) at row
    seq_lens[b]; nothing is written for a position outside the cache.  Dense: k, v [B, kvh, max_len, d]; paged: pools
    [num_blocks, kvh, block_size, d] addressed through tables [B, max_blocks]."""
    k, v = k_before.clone(), v_before.clone()
    pos = seq_lens.long().to(k.device)
    cap = tables.shape[1] * k.shape[2] if tables is not None else k.shape[2]
    rows = ((pos >= 0) & (pos < cap)).nonzero().view(-1)
    p = pos[rows]
    knew = qkv[rows.to(qkv.device), nh * d:(nh + kvh) * d].reshape(-1, kvh, d).to(k.device)
    vnew = qkv[rows.to(qkv.device), (nh + kvh) * d:(nh + 2 * kvh) * d].reshape(-1, kvh, d).to(k.device)
    if tables is None:
        k[rows, :, p] = knew
        v[rows, :, p] = vnew
    else:
        bs = k.shape[2]
        page = tables.to(k.device).long()[rows, p // bs]
        k[page, :, p % bs] = knew
        v[page, :, p % bs] = vnew
    return k, v


def assert_add_rmsnorm(normed, res_out, x, res, w, eps, what="add_rmsnorm"):
    """r = bf16(x + res) (x alone without a residual): res_out bit-exactly r; normed within 2 bf16 ulps of the fp64 RMSNorm
    of r with the kernel's rounding points (R.rms_norm, "bf16"), at most 1 % of the elements different at all."""
    r = (x.float() + res.float()).to(BF16) if res is not None else x
    if res_out is not None:
        assert_same_bits(res_out, r, f"{what}: residual_out")
    if normed is not None:
        ref = R.rms_norm(r.double(), w.double(), eps, "bf16")
        assert_within_ulps(normed, ref, ulps=2, max_frac=0.01, what=f"{what}: normed")


# ----------------------------------------------------------------------------------------------------------
# 0. The checkers reject the faults they exist to catch (CPU)
# ----------------------------------------------------------------------------------------------------------
def _cpu_append_case(seed=0, B=6, nh=6, kvh=2, d=64, max_len=40):
    g = torch.Generator().manual_seed(seed)
    n = (nh + 2 * kvh) * d
    acc = torch.randn(B, n, generator=g) * 2
    bias = torch.randn(n, generator=g) * 2
    cos, sin = _rope_tables(d, max_len, 10000.0, "cpu")
    seq_lens = torch.tensor([0, max_len - 1, 7, 31, 32, max_len][:B], dtype=torch.int32)
    return acc, bias, cos, sin, seq_lens, nh, kvh, d, max_len


def _cpu_append_result(acc, bias, cos, sin, seq_lens, nh, kvh, d, max_len, k_pos_shift=0, v_bias=True):
    """What a correct append returns (fp64 rotation rounded once), or one with a planted fault."""
    nq = (nh + kvh) * d
    x = _rounded_input(acc, bias)
    out = x.clone()
    if not v_bias:
        out[:, nq:] = acc[:, nq:].to(BF16)
    for b in range(acc.shape[0]):
        p = int(seq_lens[b])
        if not 0 <= p < max_len:
            continue
        xs = x[b, :nq].double().view(nh + kvh, d)
        pp = torch.full((nh + kvh,), p, dtype=torch.long)
        pp[nh:] += k_pos_shift
        pp = pp.clamp_max(max_len - 1)
        c, s = cos.double()[pp], sin.double()[pp]
        x1, x2 = xs[:, : d // 2], xs[:, d // 2:]
        out[b, :nq] = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).to(BF16).view(-1)
    return out


def test_checker_accepts_a_correct_append():
    case = _cpu_append_case()
    assert_rope_append_qkv(_cpu_append_result(*case), *case)


def test_checker_rejects_bias_missing_from_v():
    case = _cpu_append_case(1)
    with pytest.raises(AssertionError, match="v columns"):
        assert_rope_append_qkv(_cpu_append_result(*case, v_bias=False), *case)


def test_checker_rejects_k_rotated_at_the_next_position():
    acc, bias, cos, sin, seq_lens, nh, kvh, d, max_len = case = _cpu_append_case(2)
    seq_lens[:] = torch.tensor([0, 5, 7, 17, 32, 20], dtype=torch.int32)       # every row appended, none at the last row
    with pytest.raises(AssertionError, match="rotated q\\|k"):
        assert_rope_append_qkv(_cpu_append_result(*case, k_pos_shift=1), *case)


@pytest.mark.parametrize("fault", ["row pos + 1", "wrong kv head"])
@pytest.mark.parametrize("layout", ["dense", "paged"])
def test_checker_rejects_a_misplaced_cache_row(layout, fault):
    """One sequence's k lands one row late, or its two kv heads swap places; every other row of the append is right."""
    acc, bias, cos, sin, seq_lens, nh, kvh, d, max_len = case = _cpu_append_case(3)
    qkv = _cpu_append_result(*case)
    B, bs = acc.shape[0], 8
    if layout == "dense":
        tables = None
        k0 = torch.full((B, kvh, max_len, d), float("nan"), dtype=BF16)
    else:
        nb = B * (max_len // bs) + 3
        tables = torch.randperm(nb, generator=torch.Generator().manual_seed(3))[: nb - 3].view(B, -1).to(torch.int32)
        k0 = torch.full((nb, kvh, bs, d), float("nan"), dtype=BF16)
    want_k, _ = expected_cache_after_append(k0, k0.clone(), qkv, seq_lens, nh, kvh, d, tables)
    assert_same_bits(want_k.clone(), want_k)

    def row(pos):          # (index of sequence b's row `pos` in k, without the head) for either layout
        return (b, slice(None), pos) if tables is None else (int(tables[b, pos // bs]), slice(None), pos % bs)

    b = 2
    p = int(seq_lens[b])
    kb = qkv[b, nh * d:(nh + kvh) * d].view(kvh, d)
    bad_k = want_k.clone()
    if fault == "row pos + 1":
        bad_k[row(p)] = k0[row(p)]
        bad_k[row(p + 1)] = kb
    else:
        bad_k[row(p)] = kb.flip(0)                                   # kv head j written into kv head kvh - 1 - j
    with pytest.raises(AssertionError, match="differ"):
        assert_same_bits(bad_k, want_k, "k cache")


def test_checker_rejects_one_nonzero_float_past_the_used_workspace():
    M, N = 64, 1152
    buf = torch.zeros((M * N + 256) * 4, dtype=torch.uint8)
    assert_workspace_zero(buf)
    buf.view(torch.float32)[M * N + 37] = 2.0 ** -30                     # one partial sum left past the M x N a call used
    with pytest.raises(AssertionError, match="nonzero bytes"):
        assert_workspace_zero(buf)


def test_checker_rejects_one_scaled_rmsnorm_row():
    g = torch.Generator().manual_seed(5)
    rows, h = 64, 1032
    x = torch.randn(rows, h, generator=g).to(BF16)
    res = torch.randn(rows, h, generator=g).to(BF16)
    w = (1 + 0.1 * torch.randn(h, generator=g)).to(BF16)
    r = (x.float() + res.float()).to(BF16)
    normed = R.rms_norm(r.double(), w.double(), EPS, "bf16").to(BF16)
    assert_add_rmsnorm(normed, r, x, res, w, EPS)
    bad = normed.clone()
    bad[17] = (bad[17].double() * 1.01).to(BF16)
    with pytest.raises(AssertionError, match="normed"):
        assert_add_rmsnorm(bad, r, x, res, w, EPS)
    with pytest.raises(AssertionError, match="residual_out"):
        assert_add_rmsnorm(normed, x, x, res, w, EPS)                    # residual never added


def test_checker_rejects_a_dropped_split_k_range():
    """One output's sum is missing one of three K ranges: far outside c, though the GEMM is otherwise exact."""
    g = torch.Generator().manual_seed(6)
    M, N, K = 5, 64, 3 * 448
    A = torch.randn(M, K, generator=g).to(BF16)
    B = torch.randn(K, N, generator=g).to(BF16)
    ws = (A.double() @ B.double()).float()
    assert assert_f32_sums_close(ws, A, B) < 1e-7
    ws[3, 40] -= (A[3, 448:896].double() @ B[448:896, 40].double()).float()
    with pytest.raises(AssertionError, match="beyond c"):
        assert_f32_sums_close(ws, A, B)


# ----------------------------------------------------------------------------------------------------------
# 1. Split-K fp32 workspace: gemm_skinny_f32 at the three fused GEMMs of every preset
# ----------------------------------------------------------------------------------------------------------
def _short_last_split(K):
    """A split whose last K range is shorter than the others (ceil(K/64) k-blocks in ranges of ceil(kb / split))."""
    kb = -(-K // 64)
    for s in range(3, kb + 1):
        per = -(-kb // s)
        if kb % per:
            return s
    raise ValueError(K)


def _gemms(p):
    qkv_n = (p["nh"] + 2 * p["kvh"]) * p["d"]
    return {"qkv": (p["h"], qkv_n, True), "out_linear": (p["nh"] * p["d"], p["h"], False), "ffn2": (p["I"], p["h"], False)}


@pytest.mark.gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("gemm", ["qkv", "out_linear", "ffn2"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_gemm_skinny_f32_workspace(preset, gemm, B, fp64_reference):
    """gemm_skinny_f32 with split_k 0 (auto), 1 and a split whose last range is short: the fp32 sums per element against fp64;
    the workspace handed to its real consumer (the qkv GEMM's to the dense and the paged append, the others' to
    add_rmsnorm_f32) and then zero over its whole length; then the same buffer reused at a smaller M with new inputs."""
    o = _ops()
    p = PRESETS[preset]
    K, N, trans_b = _gemms(p)[gemm]
    nh, kvh, d = p["nh"], p["kvh"], p["d"]
    tag = f"test_splitk_{preset}_{gemm}_{B}"
    g = _gen(_seed(preset, gemm, B))
    worst = 0.0
    try:
        o._zero_workspace((B * N + 4096) * 4, torch.device(DEV), tag)   # bytes past M x N from the first call on
        for split in (0, 1, _short_last_split(K)):
            for call, M in enumerate((B, max(1, B // 2 - 1))):
                a = torch.randn(M, K, generator=g, device=DEV).to(BF16)
                w_st = (torch.randn(*((N, K) if trans_b else (K, N)), generator=g, device=DEV) / math.sqrt(K)).to(BF16)
                Bm = w_st.t() if trans_b else w_st
                ws = o.gemm_skinny_f32(a, w_st, trans_b=trans_b, split_k=split, tag=tag)
                what = f"{preset} {gemm} M={M} N={N} K={K} split_k={split} call {call}"
                worst = max(worst, assert_f32_sums_close(ws, a, Bm, what=what))
                if gemm == "qkv":
                    # every position outside the cache: the consumer only rounds, so its output is the GEMM rounded once
                    lens = torch.full((M,), 4, dtype=torch.int32, device=DEV)
                    cos, sin = _rope_tables(d, 4, p["theta"], DEV)
                    if call == 0:
                        cache = torch.zeros(2, M, kvh, 4, d, dtype=BF16, device=DEV)
                        out = o.decode_rope_append_f32(ws, None, cache, cos, sin, lens, nh, kvh, d)
                    else:
                        kc = torch.zeros(M + 1, kvh, 32, d, dtype=BF16, device=DEV)
                        tables = torch.arange(M, dtype=torch.int32, device=DEV).view(M, 1)
                        out = o.decode_rope_append_paged(None, kc, kc.clone(), tables, cos, sin, lens + 28, nh, acc_f32=ws)
                        assert not bool(kc.any())
                else:
                    w = (1 + 0.1 * torch.randn(N, generator=g, device=DEV)).to(BF16)
                    _, out = o.add_rmsnorm_f32(ws, None, w, EPS)
                assert_gemm_close(out, a, Bm, what=f"{what}: rounded by the consumer")
                assert_workspace_zero(o._workspaces[(torch.device(DEV), tag)], f"{what}: workspace after the consumer")
    finally:
        o._workspaces.pop((torch.device(DEV), tag), None)
    print(f"[splitk_f32 {preset} {gemm} B={B}] c_need {worst:.2e}")


# ----------------------------------------------------------------------------------------------------------
# 2. RoPE + append from the fp32 workspace (dense and paged cache)
# ----------------------------------------------------------------------------------------------------------
def _append_positions(B, max_len, bs, g):
    """The last row, the first, one past the cache, page ends and starts, then random rows."""
    special = [max_len - 1, 0, max_len, bs - 1, bs, 2 * bs - 1, 2 * bs, max_len - bs]
    rnd = torch.randint(0, max_len, (max(0, B - len(special)),), generator=g).tolist()
    return torch.tensor((special + rnd)[:B], dtype=torch.int32)


def _paged_pools(B, kvh, d, bs, mb, seed, spare=5):
    """NaN-filled pools [B * mb + spare, kvh, bs, d] and shuffled tables [B, mb] (the spare pages are referenced by none)."""
    nb = B * mb + spare
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))[: B * mb]
    tables = perm.view(B, mb).to(torch.int32).to(DEV)
    kc = _nan(nb, kvh, bs, d)
    return kc, kc.clone(), tables


@pytest.mark.gpu
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("cache_kind", ["dense", "paged32", "paged64", "paged128"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_rope_append_from_f32_workspace(preset, cache_kind, with_bias):
    """decode_rope_append_f32 (dense) and decode_rope_append_paged(acc_f32=, bias=) on a random fp32 accumulation: the
    returned projection against fp64 and bit for bit against the bf16 path fed bf16(acc + bias); the cache row by row; the
    workspace zero afterwards.  Positions include 0, the last row, one past the cache (nothing written, nothing rotated) and
    the first and last rows of pages."""
    o, L = _ops(), _lib()
    p = PRESETS[preset]
    nh, kvh, d = p["nh"], p["kvh"], p["d"]
    n = (nh + 2 * kvh) * d
    max_len = 512
    paged = cache_kind.startswith("paged")
    bs = int(cache_kind[5:]) if paged else 64
    mb = max_len // bs
    cos, sin = _rope_tables(d, max_len, p["theta"], DEV)
    for B in BATCHES:
        seed = _seed(preset, cache_kind, with_bias, B)
        g = _gen(seed)
        lens = _append_positions(B, max_len, bs, torch.Generator().manual_seed(seed)).to(DEV)
        acc = torch.randn(B, n, generator=g, device=DEV) * 2
        bias = torch.randn(n, generator=g, device=DEV) * 2 if with_bias else None
        x = _rounded_input(acc, bias)
        qkv = _nan(B, n)
        ws = acc.clone()
        if paged:
            kc, vc, tables = _paged_pools(B, kvh, d, bs, mb, seed)
            k0, v0 = kc.clone(), vc.clone()
            L.call("b200_decode_rope_append_paged", L.ptr(qkv), L.ptr(ws), L.ptr(bias), L.ptr(kc), L.ptr(vc), L.ptr(tables),
                   L.ptr(cos), L.ptr(sin), L.ptr(lens), B, nh, kvh, d, bs, mb, n, L.stream_ptr())
            twin_qkv, twin_k, twin_v = x.clone(), k0.clone(), v0.clone()
            o.decode_rope_append_paged(twin_qkv, twin_k, twin_v, tables, cos, sin, lens, nh)
            got_k, got_v = kc, vc
        else:
            tables = None
            cache = _nan(2, B, kvh, max_len, d)
            k0, v0 = cache[0].clone(), cache[1].clone()
            L.call("b200_decode_rope_append_f32", L.ptr(qkv), L.ptr(ws), L.ptr(bias), L.ptr(cache), L.ptr(cos), L.ptr(sin),
                   L.ptr(lens), B, nh, kvh, d, max_len, n, L.stream_ptr())
            twin_qkv, twin_cache = x.clone(), torch.stack([k0, v0])
            o.decode_rope_append(twin_qkv, twin_cache, cos, sin, lens, nh, kvh, d)
            got_k, got_v, twin_k, twin_v = cache[0], cache[1], twin_cache[0], twin_cache[1]
        what = f"{preset} {cache_kind} bias={with_bias} B={B}"
        assert_rope_append_qkv(qkv, acc, bias, cos, sin, lens, nh, kvh, d, max_len, what)
        want_k, want_v = expected_cache_after_append(k0, v0, qkv, lens, nh, kvh, d, tables)
        assert_same_bits(got_k, want_k, f"{what}: k cache")
        assert_same_bits(got_v, want_v, f"{what}: v cache")
        assert_same_bits(twin_qkv, qkv, f"{what}: bf16 path vs fp32 path, qkv")
        assert_same_bits(twin_k, got_k, f"{what}: bf16 path vs fp32 path, k cache")
        assert_same_bits(twin_v, got_v, f"{what}: bf16 path vs fp32 path, v cache")
        assert_workspace_zero(ws, f"{what}: acc")
        if B >= 3:
            assert int(lens[2]) == max_len                                     # the row past the cache was in this batch


# ----------------------------------------------------------------------------------------------------------
# 3. Residual RMSNorm: every instantiation of add_rmsnorm / add_rmsnorm_f32 and both sides of each boundary
# ----------------------------------------------------------------------------------------------------------
RMS_ROWS = [1, 64, 70, 1024, 1025, 4099]          # <= 1024: one CTA per row (<2|4|8, 4>); above: four rows per CTA (<4|16|32, 1>)
RMS_H = [896, 1024, 1032, 2048, 2056, 3072, 4096, 4104, 8192]
FORMS = ["full", "no_residual", "no_residual_out", "residual_only"]


def _add_rmsnorm_call(f32, x, res, w, normed, res_out, rows, h):
    L = _lib()
    name = "b200_add_rmsnorm_f32" if f32 else "b200_add_rmsnorm"
    L.call(name, L.ptr(x), L.ptr(res), L.ptr(w), L.ptr(normed), L.ptr(res_out), rows, h, EPS, L.stream_ptr())


@pytest.mark.gpu
@pytest.mark.parametrize("h", RMS_H)
@pytest.mark.parametrize("rows", RMS_ROWS)
def test_add_rmsnorm_every_instantiation(rows, h):
    """bf16 and fp32 (split-K workspace) input in the four forms the stack uses: residual + weight (both outputs), no residual
    (the first norm), no residual output, and no weight with want_normed=False (the last layer).  The outputs a form does not
    produce stay NaN; the fp32 workspace, with 1 024 floats past rows x h, is zero afterwards."""
    g = _gen(rows * 10007 + h)
    for f32 in (False, True):
        for form in FORMS:
            what = f"add_rmsnorm{'_f32' if f32 else ''} [{rows}, {h}] {form}"
            xb = _rows_with_spread(rows, h, g)
            res = torch.randn(rows, h, generator=g, device=DEV).to(BF16) if form != "no_residual" else None
            w = (1 + 0.1 * torch.randn(h, generator=g, device=DEV)).to(BF16)
            want_normed, want_res = form != "residual_only", form != "no_residual_out"
            normed, res_out = _nan(rows, h), _nan(rows, h)
            if f32:
                ws = torch.zeros(rows * h + 1024, device=DEV)
                ws[: rows * h].view(rows, h).copy_(xb.float() * (1 + 2.0 ** -10 * torch.rand(rows, h, generator=g, device=DEV)))
                x = ws[: rows * h].view(rows, h).to(BF16)
                src = ws
            else:
                x = src = xb
            _add_rmsnorm_call(f32, src, res, w if want_normed else None, normed if want_normed else None,
                              res_out if want_res else None, rows, h)
            assert_add_rmsnorm(normed if want_normed else None, res_out if want_res else None, x, res, w, EPS, what)
            if not want_normed:
                assert bool(torch.isnan(normed.float()).all()), f"{what}: normed written"
            if not want_res:
                assert bool(torch.isnan(res_out.float()).all()), f"{what}: residual_out written"
            if f32:
                assert_workspace_zero(ws, f"{what}: workspace")


@pytest.mark.gpu
@pytest.mark.parametrize("h", [1028, 8200])
def test_add_rmsnorm_argument_errors(h):
    """h % 8 != 0 and h > 8192 are refused before any launch, on both paths."""
    o = _ops()
    from paddlenlp_b200._lib import B200Error

    x = torch.randn(4, h, device=DEV).to(BF16)
    w = torch.ones(h, dtype=BF16, device=DEV)
    with pytest.raises(B200Error, match="h <= 8192"):
        o.add_rmsnorm(x, None, w, EPS)
    with pytest.raises(B200Error, match="h <= 8192"):
        o.add_rmsnorm_f32(torch.zeros(4, h, device=DEV), None, w, EPS)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------
# 4. One fused decode layer equals the unfused composition
# ----------------------------------------------------------------------------------------------------------
LAYER_WIDTHS = {"llama3-8b": "llama", "qwen2-1.5b": "qwen2"}


def _decode_model(preset, paged, B, max_len, seed):
    """A two-layer LlamaForCausalLMInferenceModel at the preset's width with random weights, norm scales and (Qwen2) q/k/v
    biases, and caches holding random histories (paged: shuffled tables)."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    p = PRESETS[preset]
    kind = LAYER_WIDTHS[preset]
    kw = dict(vocab_size=256, hidden_size=p["h"], intermediate_size=p["I"], num_hidden_layers=2, num_attention_heads=p["nh"],
              num_key_value_heads=p["kvh"], rms_norm_eps=1e-6 if kind == "qwen2" else 1e-5, rope_theta=p["theta"],
              max_position_embeddings=max_len)
    cfg = T.Qwen2Config(**kw) if kind == "qwen2" else T.LlamaConfig(**kw)
    m = LlamaForCausalLMInferenceModel(cfg, block_attn=paged)
    m.init_random(seed)
    t = m.transformer_block
    g = _gen(seed + 1)
    for i in range(t.L):
        for s in (t.ln_scales[i], t.ffn_ln_scales[i]):
            s.copy_((1 + 0.1 * torch.randn(t.h, generator=g, device=DEV)).to(BF16))
        if t.qkv_biases[i] is not None:
            t.qkv_biases[i].copy_((0.5 * torch.randn(t.qkv_n, generator=g, device=DEV)).to(BF16))
    t.weights_changed()
    caches = m.allocate_caches(B, max_len)
    for c in caches:
        c.copy_(torch.randn(c.shape, generator=g, device=DEV).to(BF16))
    if paged:
        nb = caches[0].shape[0]
        perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))[: m.block_tables.numel()]
        m.block_tables = perm.view(m.block_tables.shape).to(torch.int32).to(DEV)
    return m, caches


def _unfused_step(t, src, caches, seq_lens, tables):
    """The decode step written out from ops calls, without the fp32 workspace hand-offs."""
    o = _ops()
    eps = t.config.epsilon
    cos, sin = t.rope
    residual = src
    ln_out, _ = o.add_rmsnorm(src, None, t.ln_scales[0], eps, want_residual=False)
    for i in range(t.L):
        qkv = o.gemm_skinny(ln_out, t.qkv_weights[i], trans_b=True, bias=t._bias(i))
        if tables is not None:
            kc, vc = caches[2 * i], caches[2 * i + 1]
            o.decode_rope_append_paged(qkv, kc, vc, tables, cos, sin, seq_lens, t.nh)
            attn = o.decode_attention_paged(qkv, kc, vc, tables, seq_lens, t.nh)
        else:
            o.decode_rope_append(qkv, caches[i], cos, sin, seq_lens, t.nh, t.kvh, t.d)
            attn = o.decode_attention(qkv, caches[i], seq_lens, t.nh, t.kvh, t.d)
        out = o.gemm_skinny(attn, t.linear_weights[i])
        ln_out, residual = o.add_rmsnorm(out, residual, t.ffn_ln_scales[i], eps)
        _, act = o.gemm_swiglu(ln_out, t.ffn1_weights[i], store_gate_up=False)
        ffn2 = o.gemm_skinny(act, t.ffn2_weights[i])
        if i != t.L - 1:
            ln_out, residual = o.add_rmsnorm(ffn2, residual, t.ln_scales[i + 1], eps)
        else:
            _, residual = o.add_rmsnorm(ffn2, residual, None, eps, want_normed=False)
    return residual


def _both_steps(m, caches, lens, src):
    """(hidden, caches) of the fused step through transformer_block and of the unfused composition, each on its own copy."""
    t = m.transformer_block
    fused_c = [c.clone() for c in caches]
    unf_c = [c.clone() for c in caches]
    kw = m._cache_kw()
    h_fused = t(src, fused_c, B=src.shape[0], S=1, seq_lens_decoder=lens, time_step=0, **kw)
    h_unf = _unfused_step(t, src, unf_c, lens, kw.get("block_tables"))
    return h_fused, fused_c, h_unf, unf_c


def _with_pdl(on):
    class _Pdl:
        def __enter__(self):
            self.old = _lib().load().b200_set_pdl(1 if on else 0)

        def __exit__(self, *exc):
            _lib().load().b200_set_pdl(self.old)
    return _Pdl()


def _lens(B, max_len, seed):
    lens = torch.randint(0, max_len - 2, (B,), generator=torch.Generator().manual_seed(seed))
    lens[0], lens[1], lens[2] = 0, max_len - 3, 63
    return lens.to(torch.int32).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("pdl", [False, True])
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("preset", list(LAYER_WIDTHS))
def test_fused_decode_step_equals_unfused_composition(preset, paged, pdl, monkeypatch):
    """With split_k = 1 the fp32 sums are deterministic, so the fused branch (split-K GEMMs leaving fp32 sums that the append
    and the norm round) must reproduce gemm_skinny(bias) -> decode_rope_append -> decode_attention -> gemm_skinny ->
    add_rmsnorm -> gemm_swiglu -> gemm_skinny -> add_rmsnorm bit for bit: hidden states and both layers' caches; with
    programmatic dependent launch on and off."""
    import functools

    o = _ops()
    monkeypatch.setattr(o, "gemm_skinny_f32", functools.partial(o.gemm_skinny_f32, split_k=1))
    monkeypatch.setattr(o, "gemm_skinny", functools.partial(o.gemm_skinny, split_k=1))
    B, max_len = 64, 256
    m, caches = _decode_model(preset, paged, B, max_len, seed=7 + paged)
    lens = _lens(B, max_len, 11)
    src = torch.randn(B, m.transformer_block.h, generator=_gen(12), device=DEV).to(BF16)
    with _with_pdl(pdl):
        h_fused, fused_c, h_unf, unf_c = _both_steps(m, caches, lens, src)
        torch.cuda.synchronize()
    what = f"{preset} {'paged' if paged else 'dense'} pdl={pdl}"
    assert bool(torch.isfinite(h_unf.float()).all())
    assert_same_bits(h_fused, h_unf, f"{what}: hidden states")
    for j, (a, b) in enumerate(zip(fused_c, unf_c)):
        assert_same_bits(a, b, f"{what}: cache tensor {j}")
    assert any(not torch.equal(a, c) for a, c in zip(fused_c, caches))       # the step appended something


@pytest.mark.gpu
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("preset", list(LAYER_WIDTHS))
def test_fused_decode_default_split(preset, paged):
    """At the default split-K: both workspaces (splitk_qkv, splitk_h) all zero after each step, and two consecutive steps
    (the second at seq_lens + 1 on the caches the first left) match the unfused composition within the summation-order
    tolerance, row by row."""
    o = _ops()
    B, max_len = 64, 256
    m, caches = _decode_model(preset, paged, B, max_len, seed=21 + paged)
    t = m.transformer_block
    lens = _lens(B, max_len, 22)
    kw = m._cache_kw()
    fused_c = [c.clone() for c in caches]
    unf_c = [c.clone() for c in caches]
    what = f"{preset} {'paged' if paged else 'dense'} default split"
    for step in range(2):
        src = torch.randn(B, t.h, generator=_gen(30 + step), device=DEV).to(BF16)
        h_fused = t(src, fused_c, B=B, S=1, seq_lens_decoder=lens, time_step=0, **kw)
        for tag in ("splitk_qkv", "splitk_h"):
            assert_workspace_zero(o._workspaces[(torch.device(DEV), tag)], f"{what} step {step}: {tag}")
        h_unf = _unfused_step(t, src, unf_c, lens, kw.get("block_tables"))
        err = assert_rows_close(h_fused, h_unf, DEFAULT_SPLIT_ROW_TOL, what=f"{what} step {step}")
        print(f"[{what}] step {step}: worst hidden-state row relative error {err:.2e}")
        lens = lens + 1


# ----------------------------------------------------------------------------------------------------------
# 5. Prefill cache writers
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cache_kind", ["dense", "paged32", "paged64", "paged128"])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_write_cache_kv(preset, cache_kind):
    """write_cache_kv / write_cache_kv_paged at each preset's (kvh, d): B = 5 prompts of S = 300 rows from a row view of a
    wider projection buffer; rows s < seq_lens[b] (all S with seq_lens=None) hold the K and V columns bit for bit, every
    other row and every unreferenced page stays NaN."""
    o = _ops()
    p = PRESETS[preset]
    nh, kvh, d = p["nh"], p["kvh"], p["d"]
    B, S, max_len = 5, 300, 384
    n = (nh + 2 * kvh) * d
    g = _gen(_seed(preset, cache_kind))
    qkv = torch.randn(B * S, n + 40, generator=g, device=DEV).to(BF16)[:, :n]
    assert qkv.stride(0) > n
    K = qkv[:, nh * d:(nh + kvh) * d].reshape(B, S, kvh, d)
    V = qkv[:, (nh + kvh) * d:].reshape(B, S, kvh, d)
    for lens_list in ([0, 1, 127, 128, 300], None):
        lens = None if lens_list is None else torch.tensor(lens_list, dtype=torch.int32, device=DEV)
        n_rows = [S] * B if lens_list is None else lens_list
        what = f"{preset} {cache_kind} seq_lens={lens_list}"
        if cache_kind == "dense":
            cache = _nan(2, B, kvh, max_len, d)
            o.write_cache_kv(qkv, cache, lens, B, S, nh, kvh, d)
            want = _nan(2, B, kvh, max_len, d)
            for b in range(B):
                want[0, b, :, : n_rows[b]] = K[b, : n_rows[b]].transpose(0, 1)
                want[1, b, :, : n_rows[b]] = V[b, : n_rows[b]].transpose(0, 1)
            assert_same_bits(cache, want, what)
        else:
            bs = int(cache_kind[5:])
            mb = max_len // bs
            kc, vc, tables = _paged_pools(B, kvh, d, bs, mb, seed=bs + len(preset))
            o.write_cache_kv_paged(qkv, kc, vc, tables, lens, B, S, nh)
            want_k, want_v = kc.clone(), vc.clone()
            for b in range(B):
                s = torch.arange(n_rows[b], device=DEV)
                page = tables[b].long()[s // bs]
                want_k[page, :, s % bs] = K[b, : n_rows[b]]
                want_v[page, :, s % bs] = V[b, : n_rows[b]]
            assert_same_bits(kc, want_k, f"{what}: k pool")
            assert_same_bits(vc, want_v, f"{what}: v pool")


# ----------------------------------------------------------------------------------------------------------
# 6. The token-choice and state-update tail
# ----------------------------------------------------------------------------------------------------------
def _step_update_reference(next_tokens, stop, step_idx, seq_len, pre_ids, out, *, max_dec_len, eos, col):
    """generate_step_update as the generate loop and oracle/generation_ref.greedy_generate see it, on numpy copies.  A row
    that was stopped before the call emits eos[0] and changes nothing else.  A running row takes one step and records the
    token it chose in pre_ids[step] (when step < pre_len) and in the output log, also when that step reaches max_dec_len or
    the token is an eos id, either of which stops the row; its cache length advances only if it is still running."""
    nt, st, si, sl, pre = next_tokens.copy(), stop.copy(), step_idx.copy(), seq_len.copy(), pre_ids.copy()
    out = out.copy()
    ends = {int(e) for e in eos}
    for b in range(len(nt)):
        if stop[b]:
            tok = int(eos[0])
        else:
            si[b] += 1
            tok = int(nt[b])
            if 0 <= si[b] < pre.shape[1]:
                pre[b, si[b]] = tok
        st[b] = bool(stop[b]) or si[b] >= max_dec_len[b] or tok in ends
        if not st[b]:
            sl[b] += 1
        nt[b] = tok
        if 0 <= col < out.shape[1]:
            out[b, col] = tok
    return (nt, st, si, sl, pre, out), int(st.sum())


@pytest.mark.gpu
def test_generate_step_update():
    """bs = 300 (three CTAs), four calls: rows stopped before the call, a hit on each of three eos ids, max_dec_len reached,
    step >= pre_len, the device output column advancing once per call, an explicit column and one past the log,
    stop_count."""
    o = _ops()
    bs, pre_len, width = 300, 16, 6
    rng = np.random.default_rng(3)
    eos = np.array([2, 1000, 7], np.int64)
    nt = rng.integers(10, 5000, bs).astype(np.int64)
    st = rng.random(bs) < 0.2
    si = rng.integers(0, 12, bs).astype(np.int64)
    md = np.full(bs, 20, np.int64)
    sl = rng.integers(1, 500, bs).astype(np.int32)
    pre = np.full((bs, pre_len), -1, np.int64)
    out = np.full((bs, width), -1, np.int64)
    st[:10] = [True, True, False, False, False, False, False, False, False, True]
    nt[2:5] = eos                                                    # each eos id hit by a running row
    nt[1] = eos[1]                                                   # a stopped row whose token is an eos id other than eos[0]
    si[5], md[5] = 9, 10                                             # reaches max_dec_len in this call
    si[6], md[6] = 15, 40                                            # step == pre_len after the increment: no pre_ids write
    si[7], md[7] = 30, 40                                            # step > pre_len
    si[8], md[8], nt[8] = 19, 20, eos[2]                             # max_dec_len reached and the token is an eos id
    si[9] = 25                                                       # stopped, past max_dec_len and pre_len

    def dev(a, dtype):
        return torch.tensor(a, dtype=dtype, device=DEV)

    state = [dev(nt, torch.int64), dev(st, torch.bool), dev(si, torch.int64), dev(sl, torch.int32), dev(pre, torch.int64),
             dev(out, torch.int64)]
    t_md, t_eos = dev(md, torch.int64), dev(eos, torch.int64)
    t_cnt = torch.full((1,), 12345, dtype=torch.int32, device=DEV)
    t_col = torch.tensor([2], dtype=torch.int64, device=DEV)
    cur = (nt, st, si, sl, pre, out)
    names = ("next_tokens", "stop_flags", "step_idx", "seq_len_decoder", "pre_ids", "out_tokens")
    # (column from the device counter?, the column the call writes)
    for k, (col_dev, col) in enumerate([(True, 2), (True, 3), (False, 0), (False, width)]):
        if k:                                                        # the next step's choices
            fresh = rng.integers(10, 5000, bs).astype(np.int64)
            fresh[10 + k] = eos[k % 3]
            state[0].copy_(dev(fresh, torch.int64))
            cur = (fresh,) + cur[1:]
        o.generate_step_update(state[0], state[1], state[2], t_md, state[3], state[4], t_eos, state[5], t_cnt,
                               out_col=0 if col_dev else col, out_col_dev=t_col if col_dev else None)
        torch.cuda.synchronize()
        cur, count = _step_update_reference(*cur, max_dec_len=md, eos=eos, col=col)
        for name, got, want in zip(names, state, cur):
            got = got.cpu().numpy()
            assert np.array_equal(got, want), (k, name, np.argwhere(got != want)[:5].tolist())
        assert int(t_cnt.item()) == count, (k, int(t_cnt.item()), count)
        if col_dev:
            assert int(t_col.item()) == col + 1                       # advanced once by the call
        if k == 0:                                                   # the cases the reference must get right
            assert cur[0][0] == cur[0][1] == eos[0] and cur[2][0] == si[0] and cur[3][0] == sl[0] and not (cur[4][0] != -1).any()
            assert cur[1][2:6].all() and (cur[3][2:6] == sl[2:6]).all()
            assert cur[0][5] == nt[5] and cur[4][5, 10] == nt[5] and cur[5][5, 2] == nt[5]   # last token kept and recorded
            assert not cur[1][6] and not (cur[4][6] != -1).any() and cur[5][6, 2] == nt[6]


@pytest.mark.gpu
@pytest.mark.parametrize("V", [128256, 151936])
def test_argmax_f32(V):
    """Ties go to the lowest index (within a thread's stride, across warps, across the row); a row of all -inf gives 0;
    rows are read through ld > V, with larger values in the padding than in the row."""
    o = _ops()
    rows, pad = 9, 40
    g = _gen(V)
    buf = torch.randn(rows, V + pad, generator=g, device=DEV)
    buf[:, V:] = 1e30
    lg = buf[:, :V]
    top = 50.0
    lg[0, [V - 1, 5000, 37]] = top                                  # spread across threads
    lg[1, [256, 0]] = top                                           # same thread (stride 256), index 0
    lg[2, [V - 1]] = top                                            # last element
    lg[3, [31, 32, 255]] = top                                      # neighbouring lanes and warps
    lg[4] = -math.inf
    lg[5, 1000:2000] = top                                          # a long run of ties
    lg[6, [V - 2, V - 1]] = top
    out = o.argmax_f32(lg)
    torch.cuda.synchronize()
    want = torch.argmax(lg.cpu(), dim=1)                            # first maximal index
    assert want[:7].tolist() == [37, 0, V - 1, 31, 0, 1000, V - 2]
    assert out.cpu().tolist() == want.tolist()


@pytest.mark.gpu
def test_bf16_rows_to_f32():
    """A row view with ld > cols (the padded logits buffer), more elements than one pass of the grid: exact widening."""
    o = _ops()
    rows, cols, ld = 64, 151936, 151936 + 24
    src = torch.randn(rows, ld, generator=_gen(9), device=DEV).to(BF16)
    src[:, cols:] = float("nan")
    view = src[:, :cols]
    out = torch.full((rows, cols), float("nan"), device=DEV)
    o.bf16_rows_to_f32(view, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, view.float())
