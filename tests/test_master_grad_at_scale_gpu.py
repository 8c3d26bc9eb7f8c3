"""The fp32-gradient kernels of amp_master_grad at the shapes of the two training benchmarks, against fp64, on fp32 inputs
that bf16 cannot represent.

The fp32 forms (the fp32-output weight-gradient GEMM, the RMSNorm backward's fp32 dw, the fp32 column sum of the Qwen2 q/k/v
bias gradient, the fp32 embedding scatter, and the norm and AdamW step over fp32 gradients) exist so that gradients are
never rounded to bf16.  Each test here checks them with a bound that only an fp32 computation meets, and asserts on the
spot that the same result rounded to bf16 would fail it: a kernel that rounded through bf16 cannot pass.

Shapes (tokens per micro-batch T):
    Llama-3.2-3B   T 4096  h 3072  I 8192  24/8 heads             qkv width 5120  V 128 256
    Qwen2-1.5B     T 8192  h 1536  I 8960  12/2 heads, q/k/v bias qkv width 2048  V 151 936

Sums in fp32.  When a sum is evaluated along any tree in which every term passes through at most d roundings, its error is
at most gamma_d * sum |terms|, gamma_d = d u / (1 - d u), u = 2^-24 (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., section 4.2).  reduce_depth() counts d for colsum and the RMSNorm dw from the kernels' summation order.
The embedding scatter adds each token's row with one fp32 atomic: a row hit `count` times meets `count` roundings, in any
order.  The prior content of an accumulated gradient is one more term.

The checkers are plain torch and have CPU tests of their own (no gpu mark): each accepts a correct fp32 result and rejects
the same result rounded to bf16 and the fault it exists to catch.
"""
import math

import pytest
import torch

from oracle import optim_ref
from test_kernels_at_scale_gpu import (HEAD_DIM, MODELS, _rows_with_spread, _tile_sums,  # noqa: F401
                                       fp64_reference, gen, randn, sm_count, units)
from test_master_grad_gpu import _acc

DEV = "cuda:0"
BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
NAN = float("nan")
EPS = 1e-5

U32 = 2.0 ** -24               # fp32 unit roundoff
BF16_REL = 2.0 ** -8           # one bf16 rounding: at most half an ulp, <= 2^-8 of the value rounded
TILE_M, TILE_N = 128, 256      # GEMM output tile
# Per-element allowance for the fp32 accumulation of the tensor cores, times (|A| @ |B|)_ij; no bf16 term (nothing is rounded
# to bf16).  Measured on an H100 80GB HBM3 (700 W power limit) over every weight-gradient shape below with random operands:
# c_need <= 8.9e-7 at K = 4096 and <= 1.07e-6 at K = 8192.  c is ~4x the worst.
GEMM_C32 = 4.5e-6
# The same allowance for the engine's own gradients (test_engine_call_by_call_gpu.py).  Measured there (Qwen2-1.5B width,
# K = 8192 tokens): c_need 8.5e-5 for the lm_head dW and 7.4e-5 for the tied embedding's head term.  In those GEMMs a
# vocabulary column of dlogits holds one term of -1/T at the label and thousands of softmax terms ~1e5 times smaller: the
# accumulator carries the large term and every later k-step adds values that lie below its last bits.  The error then grows
# linearly in K, at about one accumulator ulp per k-step, instead of as a random walk, which is what a truncating (not
# rounding) tensor-core adder gives.  c is ~4x the worst.
ENGINE_GEMM_C32 = 3.5e-4
# Relative Frobenius error of one 128 x 256 output tile.  Measured on the same H100: <= 4.5e-6 at K = 4096, <= 9.3e-6 at
# K = 8192 with random operands, <= 1.8e-5 on the engine's gradients; one bf16 rounding gives ~1.7e-3.  ~4x the worst.
TILE32 = 7e-5
_CHUNK32 = 1 << 25             # fp64 elements per operand chunk of the GEMM reference (256 MB)


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


def gamma(d):
    """gamma_d = d u / (1 - d u): the relative error bound of an fp32 sum whose terms meet at most d roundings."""
    return d * U32 / (1 - d * U32)


def reduce_depth(rows, parts, accumulate):
    """Most fp32 roundings one term meets in colsum and in the RMSNorm dw.  Partial p sums rows p, p + parts, ... from zero
    (the first add is exact: ceil(rows / parts) - 1 roundings); colsum_reduce_kernel's lane l sums partials l, l + 8, ...
    from zero (ceil(parts / 8) - 1); lane 0 adds the other seven lanes (7); accumulate adds the prior content (1)."""
    return (-(-rows // parts) - 1) + (-(-parts // 8) - 1) + 7 + int(accumulate)


def bf16_twin(t):
    return t.to(BF16).to(t.dtype)


# ----------------------------------------------------------------------------------------------------------
# Checkers
# ----------------------------------------------------------------------------------------------------------
def assert_gemm_f32_close(out, A, B, c_old=None, *, adds=1, c=None, tile_tol=None, what="gemm fp32"):
    """Check the fp32 out [M, N] against c_old + sum_i A_i @ B_i in fp64.  A and B are the logical operands [M, K_i] and
    [K_i, N] (pass a.t() for a stored-transposed operand), or lists of them (micro-batches accumulated into one output).
      per element   |out - ref| <= c * mag + gamma_adds * (|c_old| + mag),  mag = sum_i (|A_i| @ |B_i|)
                    c bounds the tensor cores' fp32 accumulation; the second term the `adds` fp32 adds onto c_old
      per tile      relative Frobenius error of every 128 x 256 output tile <= tile_tol
      finite        every element (outputs that are not accumulated into are pre-filled with NaN)
    The reference is formed in row x column chunks of at most _CHUNK32 fp64 elements per operand.  Returns the worst
    error/bound ratio, the smallest c the output needs (c_need), the worst tile error, and the worst element ratio and tile
    error that out rounded to bf16 would have (bf16_ratio, bf16_tile; bf16_rejected: either check would fail it)."""
    c = GEMM_C32 if c is None else c
    tile_tol = TILE32 if tile_tol is None else tile_tol
    As = list(A) if isinstance(A, (list, tuple)) else [A]
    Bs = list(B) if isinstance(B, (list, tuple)) else [B]
    M, N = out.shape
    for a, b in zip(As, Bs):
        assert a.shape[0] == M and b.shape[1] == N and a.shape[1] == b.shape[0], (tuple(out.shape), a.shape, b.shape)
    K = max(a.shape[1] for a in As)
    rows = min(M, max(TILE_M, _CHUNK32 // K // TILE_M * TILE_M))
    cols = min(N, max(TILE_N, min(_CHUNK32 // K, _CHUNK32 // rows) // TILE_N * TILE_N))
    worst = dict(ratio=0.0, at=None, c_need=0.0, tile=0.0, tile_at=None, bf16_ratio=0.0, bf16_tile=0.0, bf16_rejected=None)
    for r0 in range(0, M, rows):
        for c0 in range(0, N, cols):
            ref = mag = None
            for a, b in zip(As, Bs):
                ad, bd = a[r0:r0 + rows].double(), b[:, c0:c0 + cols].double()
                p, m = ad @ bd, ad.abs() @ bd.abs()
                del ad, bd
                ref, mag = (p, m) if ref is None else (ref.add_(p), mag.add_(m))
                del p, m
            slack = 0.0
            if c_old is not None:
                co = c_old[r0:r0 + rows, c0:c0 + cols].double()
                ref += co
                slack = gamma(adds) * (co.abs() + mag)
                del co
            oc = out[r0:r0 + rows, c0:c0 + cols]
            got = oc.double()
            fin = torch.isfinite(got)
            if not bool(fin.all()):
                i, j = (~fin).nonzero()[0].tolist()
                raise AssertionError(f"{what}: {int((~fin).sum())} non-finite (unwritten?) outputs in rows {r0}.. cols {c0}..,"
                                     f" first at ({r0 + i}, {c0 + j})")
            bound = c * mag + slack + 1e-300
            ref2 = _tile_sums(ref * ref, TILE_M, TILE_N).clamp_min(1e-300)
            for twin in (False, True):
                d = (bf16_twin(oc).double() if twin else got) - ref
                err = d.abs()
                ratio = err / bound
                k = int(ratio.argmax())
                r = ratio.view(-1)[k].item()
                trel = (_tile_sums(d * d, TILE_M, TILE_N) / ref2).sqrt()
                kt = int(trel.argmax())
                t = trel.view(-1)[kt].item()
                if twin:
                    worst["bf16_ratio"] = max(worst["bf16_ratio"], r)
                    worst["bf16_tile"] = max(worst["bf16_tile"], t)
                else:
                    if r > worst["ratio"]:
                        worst["ratio"], worst["at"] = r, (r0 + k // ratio.shape[1], c0 + k % ratio.shape[1])
                    worst["c_need"] = max(worst["c_need"], ((err - slack).clamp_min(0) / (mag + 1e-300)).max().item())
                    if t > worst["tile"]:
                        worst["tile"], worst["tile_at"] = t, (r0 // TILE_M + kt // trel.shape[1], c0 // TILE_N + kt % trel.shape[1])
                del d, err, ratio, trel
            del ref, mag, got, bound, ref2, slack
    worst["bf16_rejected"] = worst["bf16_ratio"] > 1 or worst["bf16_tile"] > tile_tol
    assert worst["ratio"] <= 1.0, f"{what}: element error exceeds its bound: {worst}"
    assert worst["tile"] <= tile_tol, f"{what}: tile relative error exceeds {tile_tol}: {worst}"
    return worst


def check_bound(got, ref, bound, what="values"):
    """Every element of got finite and |got - ref| <= bound (ref, bound fp64).  Written as a negated `<=` so that a NaN
    counts as bad.  Returns the worst error/bound ratio and, for an fp32 got, the worst ratio of got rounded to bf16."""
    g = got.double()
    ratio = (g - ref).abs() / (bound + 1e-300)
    bad = ~(ratio <= 1.0)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond their bound, first at {i}: got {g[tuple(i)].item():.9e} "
                             f"ref {ref[tuple(i)].item():.9e} bound {bound[tuple(i)].item():.3e}; worst ratio "
                             f"{ratio.nan_to_num(math.inf).max().item():.3g}")
    out = dict(ratio=ratio.max().item(), bf16_ratio=None, bf16_rejected=None)
    if got.dtype == F32:
        out["bf16_ratio"] = ((bf16_twin(got).double() - ref).abs() / (bound + 1e-300)).max().item()
        out["bf16_rejected"] = out["bf16_ratio"] > 1
    return out


def sum_bound(ref, mag, depth, bf16_out):
    """Bound of an fp32 sum with terms meeting at most `depth` roundings; a bf16 output rounds that sum once more."""
    b = gamma(depth) * mag
    return BF16_REL * ref.abs() + (1 + BF16_REL) * b if bf16_out else b


def assert_colsum_close(out, a, prior=None, *, parts, what="colsum"):
    """out[n] = prior + sum over rows of a[rows, n], per column within sum_bound (mag = |prior| + sum |a|); parts = number of
    fp32 partials the kernel forms (64 for colsum, 2 * SMs for the RMSNorm dw)."""
    ad = a.double()
    ref, mag = ad.sum(0), ad.abs().sum(0)
    del ad
    if prior is not None:
        ref, mag = ref + prior.double(), mag + prior.double().abs()
    depth = reduce_depth(a.shape[0], parts, prior is not None)
    return check_bound(out, ref, sum_bound(ref, mag, depth, out.dtype == BF16), what)


def scatter_reference(ids, dout, vocab):
    """(rows, sums, abs_sums, counts) of dtable[ids[t]] += dout[t] in fp64 over the ids in [0, vocab); rows = the distinct ids
    that occur."""
    valid = (ids >= 0) & (ids < vocab)
    rows, inv, counts = torch.unique(ids[valid], return_inverse=True, return_counts=True)
    d = dout[valid].double()
    s = torch.zeros(rows.numel(), d.shape[1], dtype=F64, device=d.device).index_add_(0, inv, d)
    m = torch.zeros_like(s).index_add_(0, inv, d.abs())
    return rows, s, m, counts


def assert_scatter_close(table, prior, ids, dout, what="embedding_bwd"):
    """table = prior with dout[t] added to row ids[t] for every id in [0, V).  Rows no valid id touches keep every bit.
    A touched row hit `count` times: fp32 table, within gamma_count * (|prior| + sum |dout|), and a row hit once bit-equal
    to the one fp32 add prior + dout; bf16 table, within count * 2^-8 * (|prior| + sum |dout|), one bf16 rounding per atomic
    add in any order.  Returns the check_bound stats plus the most repeated row's id, count and relative error."""
    V = table.shape[0]
    rows, s, m, counts = scatter_reference(ids, dout, V)
    ival = torch.int32 if table.dtype == F32 else torch.int16
    changed = (table.view(ival) != prior.view(ival)).any(1)
    changed[rows] = False
    assert not bool(changed.any()), f"{what}: rows no id touches were written: {changed.nonzero()[:8, 0].tolist()}"
    p = prior[rows].double()
    ref, mag = p + s, p.abs() + m
    cnt = counts.double()[:, None]
    if table.dtype == F32:
        bound = gamma(cnt) * mag
        one = counts == 1
        want = prior[rows[one]] + s[one].float()            # dout is bf16: exact in fp32, so this is the one fp32 add
        got1 = table[rows[one]]
        normal = want.abs() >= 2.0 ** -126
        assert torch.equal(got1[normal], want[normal]), f"{what}: a row hit once is not prior + dout in fp32"
    else:
        bound = cnt * BF16_REL * mag
    st = check_bound(table[rows], ref, bound, what)
    k = int(counts.argmax())
    got_k = table[rows[k]].double()
    st.update(top_id=int(rows[k]), top_count=int(counts[k]),
              top_rel=((got_k - ref[k]).norm() / ref[k].norm()).item(),
              top_err=((got_k - ref[k]).abs() / (BF16_REL * mag[k])).max().item())
    return st


# AdamW bounds of test_kernels_at_scale_gpu.test_grad_sqnorm_and_adamw_beyond_one_wave: fp32 arithmetic with (1 - beta2) and
# the bias corrections formed from fp32 betas; bounds scale with the magnitudes of the terms, not of their sum.
def adamw_ratios(P, MA, M_, V_, master0, m0, v0, ref, hp):
    """Worst error/bound ratio of exp_avg, exp_avg_sq, master and the bf16 parameters against optim_ref's fp64 step `ref`."""
    pr, mr, vr, _ = ref
    b1, b2, step = hp["beta1"], hp["beta2"], hp["step"]
    m0, v0, master0 = m0.double(), v0.double(), master0.double()
    geff = (mr - b1 * m0) / (1 - b1)
    m_mag = b1 * m0.abs() + (1 - b1) * geff.abs()
    mb = 2.0 ** -18 * m_mag
    vb = 2.0 ** -18 * b2 * v0 + 2.0 ** -15 * (1 - b2) * geff.pow(2)
    denom = vr.sqrt() / math.sqrt(1 - b2 ** step) + hp["eps"]
    upd_mag = hp["lr"] / (1 - b1 ** step) * m_mag / denom
    pb = 2.0 ** -22 * master0.abs() + 2.0 ** -14 * upd_mag
    out = {}
    for name, got, want, bound in (("exp_avg", M_, mr, mb), ("exp_avg_sq", V_, vr, vb), ("master", MA, pr, pb),
                                   ("params", P, pr, BF16_REL * pr.abs() + pb)):
        r = (got.double() - want).abs() / (bound + 1e-300)
        out[name] = r.nan_to_num(math.inf).max().item()
    return out


# ----------------------------------------------------------------------------------------------------------
# 0. The checkers accept an fp32 result and reject its bf16 rounding and the faults they exist for (CPU)
# ----------------------------------------------------------------------------------------------------------
def _cpu_gemm(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(BF16)
    B = torch.randn(K, N, generator=g).to(BF16)
    return g, A, B


def test_gemm_f32_checker_rejects_bf16_rounding():
    _, A, B = _cpu_gemm(256, 512, 4096, 11)
    exact = A.double() @ B.double()
    good = exact.float()
    st = assert_gemm_f32_close(good, A, B)
    assert st["bf16_ratio"] > 1 and st["bf16_tile"] > TILE32
    with pytest.raises(AssertionError):
        assert_gemm_f32_close(bf16_twin(good), A, B)


def test_gemm_f32_checker_rejects_tile_added_twice():
    """Accumulate onto an fp32 C0: tile (1, 1) reduce-added twice."""
    g, A, B = _cpu_gemm(384, 768, 1024, 12)
    c0 = torch.randn(384, 768, generator=g) * 32
    prod = A.double() @ B.double()
    good = (c0.double() + prod).float()
    bad = good.clone()
    bad[128:256, 256:512] += prod[128:256, 256:512].float()
    assert_gemm_f32_close(good, A, B, c_old=c0)
    with pytest.raises(AssertionError):
        assert_gemm_f32_close(bad, A, B, c_old=c0)
    with pytest.raises(AssertionError):
        assert_gemm_f32_close(bf16_twin(good), A, B, c_old=c0)
    # four micro-batches summed into one output: the list form
    A2 = [A] + [torch.randn(384, 1024, generator=g).to(BF16) for _ in range(3)]
    acc = c0.double() + sum(a.double() @ B.double() for a in A2)
    assert_gemm_f32_close(acc.float(), A2, [B] * 4, c_old=c0, adds=4)
    acc[0:128, 0:256] -= (A2[2].double() @ B.double())[0:128, 0:256]
    with pytest.raises(AssertionError):
        assert_gemm_f32_close(acc.float(), A2, [B] * 4, c_old=c0, adds=4)


def test_gemm_f32_checker_rejects_dropped_k_block():
    """One 64-wide k-block missing from one tile at K = 8192.  That block's A values are scaled by 2^-6, so the missing block
    is ~1.4e-3 of the tile's norm: less than one bf16 rounding, far more than the fp32 accumulation."""
    g = torch.Generator().manual_seed(13)
    M, N, K, kb = 256, 512, 8192, 77
    A = torch.randn(M, K, generator=g)
    A[:, kb * 64:(kb + 1) * 64] *= 2.0 ** -6
    A = A.to(BF16)
    B = torch.randn(K, N, generator=g).to(BF16)
    exact = A.double() @ B.double()
    bad = exact.clone()
    bad[128:256, 0:256] -= A[128:256, kb * 64:(kb + 1) * 64].double() @ B[kb * 64:(kb + 1) * 64, 0:256].double()
    assert_gemm_f32_close(exact.float(), A, B)
    with pytest.raises(AssertionError):
        assert_gemm_f32_close(bad.float(), A, B)
    d = (bad - exact)[128:256, 0:256]
    assert (d.norm() / exact[128:256, 0:256].norm()).item() < 2.0 ** -9


def test_scatter_checker_rejects_missing_token_row():
    """fp32 scatter of 4096 tokens onto an fp32 table, a quarter of them one pad id: accepted; with one pad token's row
    missing, or rounded to bf16, rejected.  Untouched rows written: rejected."""
    g = torch.Generator().manual_seed(14)
    V, h, T, pad = 1000, 256, 4096, 321
    ids = torch.randint(0, V, (T,), generator=g)
    ids[torch.randperm(T, generator=g)[:T // 4]] = pad
    ids[[5, 77]] = torch.tensor([-1, V])                   # skipped
    dout = torch.randn(T, h, generator=g).to(BF16)
    prior = torch.randn(V, h, generator=g) * 4
    valid = (ids >= 0) & (ids < V)
    good = prior.clone().index_add_(0, ids[valid], dout[valid].float())
    st = assert_scatter_close(good, prior, ids, dout)
    assert st["bf16_ratio"] > 1 and st["top_id"] == pad
    drop = int((ids == pad).nonzero()[100])
    keep = valid.clone()
    keep[drop] = False
    bad = prior.clone().index_add_(0, ids[keep], dout[keep].float())
    with pytest.raises(AssertionError):
        assert_scatter_close(bad, prior, ids, dout)
    with pytest.raises(AssertionError):
        assert_scatter_close(bf16_twin(good), prior, ids, dout)
    untouched = [r for r in range(V) if not bool((ids == r).any())][0]
    stray = good.clone()
    stray[untouched, 7] += 2.0 ** -20
    with pytest.raises(AssertionError, match="rows no id touches"):
        assert_scatter_close(stray, prior, ids, dout)


def test_colsum_checker_rejects_missing_partial():
    """colsum of [8192, 256] in the kernel's order (64 fp32 partials of rows p, p + 64, ...): accepted; column 37 missing the
    rows of partial 9, or the result rounded to bf16, rejected."""
    g = torch.Generator().manual_seed(15)
    rows, n = 8192, 256
    a = torch.randn(rows, n, generator=g).to(BF16)
    prior = torch.randn(n, generator=g) * 16
    partials = a.float().view(rows // 64, 64, n).sum(0)   # partials[p] = rows p, p + 64, ...
    lanes = partials.view(8, 8, n).sum(0)                 # lane l = partials l, l + 8, ...
    total = lanes[0].clone()
    for k in range(1, 8):
        total += lanes[k]
    good = total + prior
    st = assert_colsum_close(good, a, prior, parts=64)
    assert st["bf16_ratio"] > 1
    col = int(partials[9].abs().argmax())
    bad = good.clone()
    bad[col] -= partials[9, col]
    with pytest.raises(AssertionError):
        assert_colsum_close(bad, a, prior, parts=64)
    with pytest.raises(AssertionError):
        assert_colsum_close(bf16_twin(good), a, prior, parts=64)
    # the bf16 form: one rounding of the fp32 sum is accepted, a missing partial is not
    assert_colsum_close((total + prior.to(BF16).float()).to(BF16), a, prior.to(BF16), parts=64)
    with pytest.raises(AssertionError):
        assert_colsum_close(bad.to(BF16), a, prior, parts=64)


def test_reduce_depth_counts_the_kernels_roundings():
    # 8192 rows in 64 partials: 127 + 7 + 7 (+ 1); 63 rows: one row per partial, 7 + 7
    assert reduce_depth(8192, 64, False) == 141 and reduce_depth(8192, 64, True) == 142
    assert reduce_depth(63, 63, False) == 14
    # RMSNorm dw at 8192 rows on 132 SMs: 264 partials of <= 32 rows
    assert reduce_depth(8192, 264, True) == 31 + 32 + 7 + 1


# ----------------------------------------------------------------------------------------------------------
# 1. fp32 weight-gradient GEMMs at every dW shape of DecoderEngine.backward / _layer_bwd
# ----------------------------------------------------------------------------------------------------------
def _dw_cases():
    """(id, M, N, K): out [M, N] fp32 = a^T b with a stored [K, M] and b [K, N], K = tokens per micro-batch."""
    cases = []
    for name, s in MODELS.items():
        T, h, I, V = s["M"], s["h"], s["I"], s["V"]
        qn, n_qkv = s["nh"] * HEAD_DIM, (s["nh"] + 2 * s["kvh"]) * HEAD_DIM
        cases += [(f"{name}-qkv_dW", h, n_qkv, T), (f"{name}-o_dW", qn, h, T), (f"{name}-gate_up_dW", h, 2 * I, T),
                  (f"{name}-down_dW", I, h, T), (f"{name}-lm_head_dW", h, V, T),
                  (f"{name}-tied_embed_dW", V, h, T)]               # dE = dlogits^T @ hf
    return cases


DW_CASES = _dw_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
def test_gemm_f32_weight_grad_shapes(case, fp64_reference):
    """(a) fresh: the output is a view at an offset into a NaN-filled flat buffer, as the gradient views are; it must equal
    the kernel's own fp32 accumulators, round to the bf16 GEMM's output, pass the fp64 check, and leave the rest of the
    buffer alone.  (b) accumulate four micro-batches onto a random fp32 C0 (each with a new copy of the smaller operand; the
    larger one, 2.5 GB for dlogits at V 151 936, is shared): after every call the output is the previous content + the fresh
    product in fp32, bit for bit; at the end it passes the fp64 check against C0 + the sum of the four products."""
    o = ops()
    name, M, N, K = case
    seed = 1100 + DW_CASES.index(case)
    g = gen(seed)
    a_st, b_st = randn((K, M), g), randn((K, N), g)
    pad = 8                                                # 32 bytes: the flat views' alignment
    buf = torch.full((M * N + 2 * pad,), NAN, dtype=F32, device=DEV)
    out = buf[pad:pad + M * N].view(M, N)
    o.gemm(a_st, b_st, out=out, trans_a=True)
    torch.cuda.synchronize()
    assert torch.equal(out, _acc(a_st, b_st, True, False)), f"{name}: fp32 output != the kernel's accumulators"
    assert torch.equal(out.to(BF16), o.gemm(a_st, b_st, trans_a=True)), f"{name}: rounded fp32 output != bf16 GEMM"
    st = assert_gemm_f32_close(out, a_st.t(), b_st, what=f"{name} fresh")
    print(f"[gemm fp32 {name} M={M} N={N} K={K} fresh] worst err/bound {st['ratio']:.3f} c_need {st['c_need']:.3e} "
          f"worst tile {st['tile']:.3e} | bf16-rounded: err/bound {st['bf16_ratio']:.1f} tile {st['bf16_tile']:.2e}")
    assert st["bf16_ratio"] > 1 and st["bf16_tile"] > TILE32          # both checks reject the bf16-rounded output
    assert bool(buf[:pad].isnan().all()) and bool(buf[-pad:].isnan().all()), f"{name}: wrote outside the output view"

    def c0():                                              # regenerated for the final check instead of kept (1.5 GB)
        return torch.randn(M, N, generator=gen(seed + 50), device=DEV) * math.sqrt(K)

    out.copy_(c0())
    assert bool((bf16_twin(out[:64]) != out[:64]).float().mean() > 0.99)     # C0 is not bf16-representable
    want = torch.empty(M, N, dtype=F32, device=DEV)
    As, Bs = [a_st], [b_st]
    for i in range(1, 4):
        As.append(randn((K, M), g) if M <= N else a_st)
        Bs.append(b_st if M <= N else randn((K, N), g))
    for i in range(4):
        o.gemm(As[i], Bs[i], out=want, trans_a=True)      # the fresh product, checked above
        want.add_(out)
        o.gemm(As[i], Bs[i], out=out, trans_a=True, accumulate=True)
        normal = want.abs() >= 2.0 ** -126                  # subnormal sums flush to zero
        wrong = (out != want) & normal
        assert not bool(wrong.any()), f"{name}: micro-batch {i}: {int(wrong.sum())} elements != previous + fresh, " \
                                      f"first at {wrong.nonzero()[0].tolist()}"
        assert bool((out[~normal] == 0).all())
        del normal, wrong
    del want
    assert bool(buf[:pad].isnan().all()) and bool(buf[-pad:].isnan().all()), f"{name}: wrote outside the output view"
    st = assert_gemm_f32_close(out, [a.t() for a in As], Bs, c_old=c0(), adds=4, what=f"{name} 4 micro-batches")
    print(f"[gemm fp32 {name} M={M} N={N} K={K} 4 micro-batches onto C0] worst err/bound {st['ratio']:.3f} "
          f"c_need {st['c_need']:.3e} worst tile {st['tile']:.3e} | bf16-rounded: err/bound {st['bf16_ratio']:.1f}")
    assert st["bf16_ratio"] > 1 and st["bf16_tile"] > TILE32


# ----------------------------------------------------------------------------------------------------------
# 2. Reducers at the benchmark shapes and past one persistent-grid trip
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h", [1536, 3072])
@pytest.mark.parametrize("rows", ["W-1", "W", "W+1", 4096, 8192])
def test_rmsnorm_bwd_fp32_dw(rows, h):
    """RMSNorm backward with an fp32 dw (W = 2 * SMs CTAs, each carrying its dw partial over its rows), fresh into NaN and
    accumulated onto a dw0 bf16 cannot represent.  dx is bit-equal to the bf16-dw form's; dw per column against the fp64
    sum of dy * bf16(x * rstd) (the forward's rounded x-hat) with the fp32 bound of the kernel's summation depth."""
    o = ops()
    n = units(rows, 2 * sm_count())
    parts = min(n, 2 * sm_count())
    g = gen(1200 + h + n)
    x = _rows_with_spread(n, h, g)
    w = (1 + 0.1 * torch.randn(h, generator=g, device=DEV)).to(BF16)
    dy, dres = randn((n, h), g), randn((n, h), g)
    rstd = torch.rsqrt(x.double().pow(2).mean(-1) + EPS).float()
    dw0 = torch.randn(h, generator=g, device=DEV) * 4
    assert bool((bf16_twin(dw0) != dw0).all())
    terms = dy.double() * (x.double() * rstd.double()[:, None]).float().to(BF16).double()
    for accumulate in (False, True):
        dw = dw0.clone() if accumulate else torch.full((h,), NAN, dtype=F32, device=DEV)
        dx = torch.full((n, h), NAN, dtype=BF16, device=DEV)
        o.rmsnorm_bwd(dy, x, w, rstd, dw, dres=dres, accumulate_dw=accumulate, dx=dx)
        dw16 = dw0.to(BF16) if accumulate else torch.full((h,), NAN, dtype=BF16, device=DEV)     # bf16-dw form
        dx16 = o.rmsnorm_bwd(dy, x, w, rstd, dw16, dres=dres, accumulate_dw=accumulate)
        assert torch.equal(dx, dx16), "dx differs between the fp32-dw and the bf16-dw forms"
        depth = reduce_depth(n, parts, accumulate)
        st = assert_colsum_close(dw, terms, dw0 if accumulate else None, parts=parts,
                                 what=f"rmsnorm dw fp32 [{n}, {h}] acc={accumulate}")
        st16 = assert_colsum_close(dw16, terms, dw0.to(BF16) if accumulate else None, parts=parts,
                                   what=f"rmsnorm dw bf16 [{n}, {h}] acc={accumulate}")
        print(f"[rmsnorm_bwd dw rows={n} h={h} accumulate={accumulate} depth {depth}] fp32 err/bound {st['ratio']:.3f} "
              f"(bf16-rounded {st['bf16_ratio']:.1f}); bf16 form err/bound {st16['ratio']:.3f}")
        assert st["bf16_ratio"] > 1


QWEN_QKV = (12 + 2 * 2) * HEAD_DIM       # 2048


@pytest.mark.gpu
@pytest.mark.parametrize("view", ["dqkv", "column_slice"])
@pytest.mark.parametrize("rows", [63, 64, 65, 8192])
def test_colsum_both_forms(rows, view):
    """The Qwen2 q/k/v bias gradient: column sums of dqkv [rows, 2048], or of the column slice [:, 520:1800] (ld 2048 > n),
    over 63 / 64 / 65 rows (around the 64 partials) and 8192 (the benchmark's tokens).  Fresh into NaN and accumulated onto
    a prior; the fp32 output is a view between NaN sentinels.  fp32: fp32 bound, and its bf16 rounding fails it; bf16: one
    rounding of the fp32 sum on top."""
    o = ops()
    g = gen(1300 + rows + len(view))
    full = randn((rows, QWEN_QKV), g)
    a = full if view == "dqkv" else full[:, 520:1800]
    n = a.shape[1]
    parts = min(rows, 64)
    prior32 = torch.randn(n, generator=g, device=DEV) * math.sqrt(rows)
    for accumulate in (False, True):
        buf = torch.full((n + 16,), NAN, dtype=F32, device=DEV)
        out = buf[8:8 + n]
        if accumulate:
            out.copy_(prior32)
        o.colsum(a, out, accumulate=accumulate)
        assert bool(buf[:8].isnan().all()) and bool(buf[-8:].isnan().all()), "colsum fp32 wrote outside its output"
        st = assert_colsum_close(out, a, prior32 if accumulate else None, parts=parts,
                                 what=f"colsum fp32 [{rows}, {n}] acc={accumulate}")
        assert st["bf16_ratio"] > 1
        out16 = prior32.to(BF16) if accumulate else torch.full((n,), NAN, dtype=BF16, device=DEV)
        prior16 = out16.clone() if accumulate else None
        o.colsum(a, out16, accumulate=accumulate)
        st16 = assert_colsum_close(out16, a, prior16, parts=parts, what=f"colsum bf16 [{rows}, {n}] acc={accumulate}")
        print(f"[colsum rows={rows} n={n} ld={a.stride(0)} accumulate={accumulate}] fp32 err/bound {st['ratio']:.3f} "
              f"(bf16-rounded {st['bf16_ratio']:.1f}); bf16 form err/bound {st16['ratio']:.3f}")


EMB = {"qwen2-1.5b": (8192, 151936, 1536), "llama3.2-3b": (4096, 128256, 3072)}      # T, V, h


def _ids(dist, T, V, g):
    if dist == "uniform":
        ids = torch.randint(0, V, (T,), generator=g, device=DEV)
    elif dist == "zipf":                                   # p(rank r) ~ 1 / (r + 1), ranks shuffled over the vocabulary
        w = 1.0 / torch.arange(1, V + 1, device=DEV, dtype=torch.float64)
        ids = torch.randperm(V, generator=g, device=DEV)[torch.multinomial(w, T, replacement=True, generator=g)]
    elif dist == "pad":                                    # one id (a pad or BOS token) takes 25 % of the tokens
        ids = torch.randint(0, V, (T,), generator=g, device=DEV)
        ids[torch.randperm(T, generator=g, device=DEV)[:T // 4]] = V // 3 + 7
    else:                                                  # "edges": an eighth of the tokens each at id 0 and id V - 1
        ids = torch.randint(0, V, (T,), generator=g, device=DEV)
        perm = torch.randperm(T, generator=g, device=DEV)
        ids[perm[:T // 8]] = 0
        ids[perm[T // 8:T // 4]] = V - 1
    ids[[3, 100, T // 2 + 1, T - 1]] = torch.tensor([-1, V, -100, V + 12345], device=DEV)     # out of range
    return ids


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["uniform", "zipf", "pad", "edges"])
@pytest.mark.parametrize("model", list(EMB))
def test_embedding_at_real_vocab(model, dist):
    """embedding_fwd and both embedding_bwd forms at a real vocabulary and the benchmark's tokens per micro-batch.

    Out-of-range ids (< 0 or >= V) are handled differently by the two directions: the forward reads row 0 for them, the
    backward skips them (no row receives their gradient).  Both behaviours are pinned down here.

    Forward: bit-equal to table[ids].  Backward: onto a prior table (fp32: content bf16 cannot represent, as in the tied
    model where the head's GEMM term is already there), untouched rows keep every bit, touched rows within the bound of
    assert_scatter_close.  The bf16 form's error on the most repeated row is printed: the cost of bf16 atomics on a pad
    token."""
    o = ops()
    T, V, h = EMB[model]
    g = gen(1400 + len(model) + 17 * len(dist))
    ids = _ids(dist, T, V, g)
    dout = randn((T, h), g)
    table16 = randn((V, h), g)
    emb = o.embedding_fwd(ids, table16)
    valid = (ids >= 0) & (ids < V)
    assert torch.equal(emb, table16[torch.where(valid, ids, 0)]), "embedding_fwd != table[ids] (out-of-range ids -> row 0)"
    del emb

    t16 = table16.clone()
    o.embedding_bwd(ids, dout, t16)
    st16 = assert_scatter_close(t16, table16, ids, dout, what=f"embedding_bwd bf16 {model} {dist}")
    del t16, table16
    prior = torch.randn(V, h, generator=g, device=DEV)
    assert bool((bf16_twin(prior[:1024]) != prior[:1024]).float().mean() > 0.99)
    t32 = prior.clone()
    o.embedding_bwd(ids, dout, t32)
    st = assert_scatter_close(t32, prior, ids, dout, what=f"embedding_bwd fp32 {model} {dist}")
    print(f"[embedding {model} T={T} V={V} h={h} {dist}] most repeated id {st['top_id']} x{st['top_count']}: "
          f"bf16 atomics relative error {st16['top_rel']:.2e} (max err {st16['top_err']:.3f} x 2^-8 sum|terms|), "
          f"fp32 {st['top_rel']:.2e}; fp32 err/bound {st['ratio']:.3f} (bf16-rounded {st['bf16_ratio']:.1f}), "
          f"bf16 form err/bound {st16['ratio']:.3f}")
    assert st["bf16_ratio"] > 1
    if dist == "pad":
        assert st["top_count"] >= T // 4 - 4            # four positions hold out-of-range ids


def _fill_normal(t, g, std, chunk=1 << 28):
    for s in range(0, t.numel(), chunk):
        t[s:s + chunk].normal_(0, std, generator=g)
    return t


def adamw_run(G, decay_end, hp, scale, mgn, seed, positions=None, G_ref=None):
    """One AdamW step over the gradients G from a random state drawn from `seed` (14 bytes of state per element).  Returns
    the worst error/bound ratios (adamw_ratios) against optim_ref in fp64 on the CPU, at `positions` (every element when
    None), for the gradients G_ref (default G).  The clip coefficient comes from the kernel's own norm of G, which the
    callers check against fp64; the reference applies it as part of grad_scale."""
    o = ops()
    n = G.numel()
    g = gen(seed)
    master = _fill_normal(torch.empty(n, device=DEV), g, 0.02)
    m = _fill_normal(torch.empty(n, device=DEV), g, 1e-3)
    v = _fill_normal(torch.empty(n, device=DEV), g, 3e-3).square_()
    idx = torch.arange(n, device=DEV) if positions is None else positions
    s0 = [t[idx].double().cpu() for t in (master, m, v)]
    P = torch.empty(n, dtype=BF16, device=DEV)
    sq = o.grad_sqnorm(G, scale=scale)
    coef = mgn / max(math.sqrt(sq.item()), mgn)
    o.adamw_step(P, G, master, m, v, sq, decay_end=decay_end, grad_scale=scale, max_grad_norm=mgn, **hp)
    got = [t[idx].cpu() for t in (P, master, m, v)]
    del master, m, v, P
    gr = (G if G_ref is None else G_ref)[idx].double().cpu()
    ref = optim_ref.adamw_step(*s0, gr, decay_mask=idx.cpu() < decay_end, grad_scale=scale * coef, max_grad_norm=0, **hp)
    return adamw_ratios(*got, *s0, ref, hp)


HP = dict(lr=3e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01)


@pytest.mark.gpu
@pytest.mark.parametrize("clip", [True, False])
@pytest.mark.parametrize("step", [1, 1000])
def test_sqnorm_and_adamw_fp32_grads_beyond_one_wave(step, clip):
    """grad_sqnorm and AdamW on fp32 gradients bf16 cannot represent, over three grid-stride trips (W = 8 * SMs * 256 * 8
    elements) plus 13 chunks, the weight-decay boundary inside the second trip.  Per element against optim_ref in fp64 with
    the bounds of the bf16-gradient test; the same step fed the gradients rounded to bf16 must violate them."""
    o = ops()
    W = 8 * sm_count() * 256 * 8
    n, decay_end = 3 * W + 8 * 13, W + 8 * 5
    g = gen(1500 + step + clip)
    G = torch.randn(n + 8, generator=g, device=DEV) * 0.01
    assert bool((bf16_twin(G) != G).float().mean() > 0.99)
    scale = 0.5
    for m_ in (n, n + 5):                                  # n + 5: the block-0 tail loop
        sq_ref = (G[:m_].double() * scale).pow(2).sum().item()
        assert abs(o.grad_sqnorm(G[:m_], scale=scale).item() - sq_ref) <= 1e-5 * sq_ref
    G = G[:n]
    mgn = 1.0 if clip else 1e3
    assert (math.sqrt((G.double() * scale).pow(2).sum().item()) > mgn) == clip
    hp = dict(HP, step=step)
    r32 = adamw_run(G, decay_end, hp, scale, mgn, seed=1550 + step)
    r16 = adamw_run(bf16_twin(G), decay_end, hp, scale, mgn, seed=1550 + step, G_ref=G)
    print(f"[adamw fp32 grads n={n} step={step} clip={clip}] worst err/bound {r32} | fed bf16(g): {r16}")
    assert max(r32.values()) <= 1.0, r32
    assert max(r16["exp_avg"], r16["exp_avg_sq"], r16["master"]) > 1.0, "the checks cannot tell fp32 from bf16 gradients"


# ----------------------------------------------------------------------------------------------------------
# 3. Past 2^31 elements (the Llama-3.2-3B flat buffers hold 3.6e9)
# ----------------------------------------------------------------------------------------------------------
N31 = 1 << 31


def _chunked_sqnorm64(G, scale):
    return sum((G[s:s + (1 << 28)].double() * scale).pow(2).sum().item() for s in range(0, G.numel(), 1 << 28))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "fp32"])
def test_grad_sqnorm_past_2_31(dtype):
    """n = 2^31 + 8 * 13 + 5 gradients (4.3 GB bf16, 8.6 GB fp32).  Large values just past index 2^31 and in the 5-element
    tail: an index that wrapped at 2^31 would read other elements and change the sum.  Against a chunked fp64 sum."""
    o = ops()
    n = N31 + 8 * 13 + 5
    G = _fill_normal(torch.empty(n, dtype=dtype, device=DEV), gen(1600), 1.0)
    G[N31:N31 + 4096] = 300.0
    G[N31 - 8:N31] = -50.0
    G[-5:] = 1000.0
    scale = 0.5
    sq = o.grad_sqnorm(G, scale=scale).item()
    ref = _chunked_sqnorm64(G, scale)
    print(f"[grad_sqnorm {dtype} n={n}] relative error {abs(sq - ref) / ref:.2e}")
    assert abs(sq - ref) <= 1e-5 * ref


@pytest.mark.gpu
def test_adamw_past_2_31():
    """AdamW over n = 2^31 + 8 * 13 elements with decay_end = 2^31 + 40, fp32 gradients and then bf16 ones (about 39 GB of
    state and gradients: run only with 45 GB free).  Against optim_ref in fp64 on the 64 K elements from 2^31 - 64 K to the
    end (around 2^31, around decay_end and the end) and on 1 M random positions; the update is elementwise, so sampled
    positions are a complete check of each."""
    free = torch.cuda.mem_get_info()[0]
    print(f"[adamw past 2^31] free device memory {free / 1e9:.1f} GB")
    if free < 45e9:
        pytest.skip(f"needs 45 GB of free device memory, {free / 1e9:.1f} GB free")
    n, decay_end = N31 + 8 * 13, N31 + 8 * 5
    positions = torch.cat([torch.arange(N31 - (1 << 16), n),
                           torch.randint(0, n, (1 << 20,), generator=torch.Generator().manual_seed(5))]).to(DEV)
    hp = dict(HP, step=3)
    scale, mgn = 0.5, 1.0
    for dtype in (F32, BF16):
        G = _fill_normal(torch.empty(n, dtype=dtype, device=DEV), gen(1700), 0.01)
        sq, ref = ops().grad_sqnorm(G, scale=scale).item(), _chunked_sqnorm64(G, scale)
        assert abs(sq - ref) <= 1e-5 * ref and math.sqrt(ref) > mgn          # clipping is active
        r = adamw_run(G, decay_end, hp, scale, mgn, seed=1701, positions=positions)
        print(f"[adamw past 2^31 {dtype} n={n} decay_end={decay_end}] worst err/bound {r}")
        assert max(r.values()) <= 1.0, r
        del G
