"""The kernels at the shapes the two training benchmarks issue, and past the first trip of their persistent loops.

Almost every kernel here walks its work in a persistent or grid-stride loop whose trip size scales with the SM count
(8 * SMs rows for the RMSNorm forward, 2 * SMs rows for its backward, 16 * SMs * 256 8-element chunks for SwiGLU,
8 * SMs * 256 * 8 elements for the optimizer, one 128x256 tile per CTA for the GEMM).  Each test below runs a kernel at,
just below and just above one trip and at the benchmark sizes (Llama-3.2-3B: h 3072, I 8192, 24/8 heads, V 128 256,
M = 4096 tokens; Qwen2-1.5B: h 1536, I 8960, 12/2 heads with qkv bias, V 151 936, M = 8192 tokens), against an fp64
reference, with checks that localise an error: per element and per 128x256 output tile for the GEMM, per row for the
row kernels.  A relative error over a whole tensor cannot see one wrong row among 4096 or one wrong tile among 16 000.

The checkers are plain torch and have CPU tests of their own (no gpu mark): each feeds them a correct bf16 result and a
sabotaged one and asserts that only the correct one is accepted.
"""
import math

import pytest
import torch

from oracle import llama_ref as R
from oracle import optim_ref

DEV = "cuda:0"
BF16 = torch.bfloat16

TILE_M, TILE_N = 128, 256      # GEMM output tile (two 64-row consumer warpgroups x wgmma N)
BF16_REL = 2.0 ** -8           # one bf16 rounding (8 significant bits): at most half an ulp, <= 2^-8 of the value rounded
# Per-element allowance for the fp32 accumulation of the tensor cores, times (|A| |B|)_ij.  Measured on an H100 80GB HBM3
# (700 W power limit): every training shape needs c_need <= 6.6e-7 except the lm-head dX GEMMs, 2.06e-6 at K = 128 256 and
# 2.21e-6 at K = 151 936.  c is ~4x the worst of those.
GEMM_C = 9e-6
# Relative Frobenius error of one output tile.  A bf16 rounding error is uniform within half an ulp, 2^-8 .. 2^-9 of the value:
# ~1.6e-3 rms for one rounding, ~2.3e-3 for the residual epilogue's two.
TILE_TOL = 4e-3
# Relative error of one row of a row kernel (one rounding per element, ~1.6e-3 rms; a row of 8 elements can reach 2^-8).
ROW_TOL = 4e-3
_CHUNK = 1 << 28               # fp64 elements per operand chunk of the GEMM reference (2 GB)


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


def relerr(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


# ----------------------------------------------------------------------------------------------------------
# Checkers
# ----------------------------------------------------------------------------------------------------------
def _tile_sums(x, tm, tn):
    """Sums of x [r, c] over tm x tn tiles (the last tile row / column may be partial)."""
    r, c = x.shape
    pr, pc = (-r) % tm, (-c) % tn
    if pr or pc:
        x = torch.nn.functional.pad(x, (0, pc, 0, pr))
    return x.view((r + pr) // tm, tm, (c + pc) // tn, tn).sum((1, 3))


def assert_gemm_close(out, A, B, *, bias=None, c_old=None, residual=None, c=GEMM_C, tile_tol=TILE_TOL, what="gemm"):
    """Check out [M, N] against A [M, K] @ B [K, N] (+ bias [N]) (+ c_old or residual [M, N]) evaluated in fp64.

    A and B are the logical operands (pass a.t() for a stored-transposed operand); any device.  Three checks:
      per element   |out - ref| <= 2^-8 * ref_pre + c * (|A| @ |B|)
                    ref_pre = |ref| for one rounding (plain, bias, accumulate into c_old: C = bf16(c_old + acc + bias));
                    |A @ B + bias| + |ref| for the residual epilogue, which rounds the product and then the sum;
                    c * (|A| @ |B|) bounds the fp32 accumulation
      per tile      relative Frobenius error of every 128x256 output tile <= tile_tol
      finite        every element (callers pre-fill outputs that are not accumulated into with NaN, so an element that is
                    never written fails here)
    The reference is formed in row x column chunks of at most _CHUNK fp64 elements per operand.  Returns the worst
    error/bound ratio, the smallest c the output needs (c_need) and the worst tile error."""
    M, K = A.shape
    N = B.shape[1]
    assert B.shape[0] == K and tuple(out.shape) == (M, N), (tuple(out.shape), tuple(A.shape), tuple(B.shape))
    rows = min(M, max(TILE_M, _CHUNK // K // TILE_M * TILE_M))
    cols = min(N, max(TILE_N, min(_CHUNK // K, (_CHUNK // 2) // rows) // TILE_N * TILE_N))
    worst = dict(ratio=0.0, at=None, c_need=0.0, tile=0.0, tile_at=None)
    for r0 in range(0, M, rows):
        a = A[r0:r0 + rows].double()
        aa = a.abs()
        for c0 in range(0, N, cols):
            b = B[:, c0:c0 + cols].double()
            ref = a @ b
            mag = aa @ b.abs()
            del b
            if bias is not None:
                ref += bias[c0:c0 + cols].double()
            pre = ref.abs() if residual is not None else None
            for extra in (c_old, residual):
                if extra is not None:
                    ref += extra[r0:r0 + rows, c0:c0 + cols].double()
            pre = ref.abs() if pre is None else pre + ref.abs()
            got = out[r0:r0 + rows, c0:c0 + cols].double()
            fin = torch.isfinite(got)
            if not bool(fin.all()):
                i, j = (~fin).nonzero()[0].tolist()
                raise AssertionError(f"{what}: {int((~fin).sum())} non-finite (unwritten?) outputs in rows {r0}.. cols {c0}..,"
                                     f" first at ({r0 + i}, {c0 + j})")
            d = got - ref
            del got
            err = d.abs()
            ratio = err / (BF16_REL * pre + c * mag + 1e-300)
            k = int(ratio.argmax())
            if ratio.view(-1)[k].item() > worst["ratio"]:
                worst["ratio"] = ratio.view(-1)[k].item()
                worst["at"] = (r0 + k // ratio.shape[1], c0 + k % ratio.shape[1])
            del ratio
            worst["c_need"] = max(worst["c_need"], ((err - BF16_REL * pre).clamp_min(0) / (mag + 1e-300)).max().item())
            del err, pre, mag
            trel = (_tile_sums(d * d, TILE_M, TILE_N) / _tile_sums(ref * ref, TILE_M, TILE_N).clamp_min(1e-300)).sqrt()
            del d, ref
            k = int(trel.argmax())
            if trel.view(-1)[k].item() > worst["tile"]:
                worst["tile"] = trel.view(-1)[k].item()
                worst["tile_at"] = (r0 // TILE_M + k // trel.shape[1], c0 // TILE_N + k % trel.shape[1])
    assert worst["ratio"] <= 1.0, f"{what}: element error exceeds its bound: {worst}"
    assert worst["tile"] <= tile_tol, f"{what}: tile relative error exceeds {tile_tol}: {worst}"
    return worst


def assert_rows_close(got, ref, tol, what="rows"):
    """relerr of every row (first dimension; the rest is flattened) <= tol.  A row whose reference is all zero must be
    exactly zero.  For attention, pass tensors reshaped to one (head, q-tile) block per row."""
    n = got.shape[0]
    assert ref.shape[0] == n
    per = max(1, got[0].numel())
    step = max(1, (1 << 26) // per)
    worst, worst_row = 0.0, -1
    for i0 in range(0, n, step):
        g = got[i0:i0 + step].reshape(-1, per).double()
        r = ref[i0:i0 + step].reshape(-1, per).double()
        en, rn = (g - r).norm(dim=1), r.norm(dim=1)
        rel = torch.where(rn > 0, en / rn.clamp_min(1e-300), torch.where(en > 0, torch.full_like(en, math.inf), en))
        rel = torch.where(torch.isnan(rel), torch.full_like(rel, math.inf), rel)
        k = int(rel.argmax())
        if rel[k].item() > worst:
            worst, worst_row = rel[k].item(), i0 + k
    assert worst <= tol, f"{what}: row {worst_row} has relative error {worst:.3e} > {tol}"
    return worst


def bf16_ulp(t):
    """Spacing of bf16 numbers at |t| (8 significant bits); the smallest normal spacing for |t| below 2^-126."""
    _, e = torch.frexp(t.abs().float().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(t, dtype=torch.float32), e - 8)


def assert_within_ulps(got, ref, ulps=2, max_frac=0.01, what="values"):
    """Every element finite and within `ulps` bf16 ulps of ref, and at most max_frac of the elements different at all.
    Written as a negated `<=` so that a NaN (an output pre-filled with NaN and never written) counts as bad."""
    g, r = got.float(), ref.float()
    bad = ~((g - r).abs() <= ulps * bf16_ulp(r))
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond {ulps} ulps, first at {i}: "
                             f"{g[tuple(i)].item()} vs {r[tuple(i)].item()}")
    frac = (g != r).double().mean().item()
    assert frac <= max_frac, f"{what}: {frac:.4f} of the elements differ from the reference (> {max_frac})"


# ----------------------------------------------------------------------------------------------------------
# 0. The checkers reject the failures they are meant to find (CPU)
# ----------------------------------------------------------------------------------------------------------
def test_checker_rejects_dropped_k_block():
    """One 64-wide k-block missing from one tile at the lm-head dX depth K = 128 256.  That k-block's A values are scaled by
    0.45, so the missing block is ~1 % of the tile's norm: 2.5x the per-tile limit, yet only ~0.25 % over the 16 tiles, which
    a single relative error over the tensor accepts."""
    g = torch.Generator().manual_seed(1)
    M, N, K, kb = 512, 1024, 128256, 1000
    A = torch.randn(M, K, generator=g)
    A[:, kb * 64:(kb + 1) * 64] *= 0.45
    A = A.to(BF16)
    B = torch.randn(K, N, generator=g).to(BF16)
    exact = A.double() @ B.double()
    bad = exact.clone()
    bad[128:256, 256:512] -= A[128:256, kb * 64:(kb + 1) * 64].double() @ B[kb * 64:(kb + 1) * 64, 256:512].double()
    assert_gemm_close(exact.to(BF16), A, B)
    with pytest.raises(AssertionError):
        assert_gemm_close(bad.to(BF16), A, B)
    assert relerr(bad.to(BF16), exact) < 4e-3


def test_checker_rejects_tile_copied_from_neighbour():
    """Output tile (3, 2) holds tile (2, 2).  The rows of A repeat every 128 rows up to a 2^-6 perturbation, so neighbouring
    tiles differ by ~2 % and the copy is ~0.2 % of the 128-tile output: below a global 4e-3, far above the per-tile limit."""
    g = torch.Generator().manual_seed(2)
    M, N, K = 2048, 2048, 256
    A = (torch.randn(TILE_M, K, generator=g).repeat(M // TILE_M, 1) + 2 ** -6 * torch.randn(M, K, generator=g)).to(BF16)
    B = torch.randn(K, N, generator=g).to(BF16)
    exact = A.double() @ B.double()
    bad = exact.clone()
    bad[384:512, 512:768] = exact[256:384, 512:768]
    assert_gemm_close(exact.to(BF16), A, B)
    with pytest.raises(AssertionError):
        assert_gemm_close(bad.to(BF16), A, B)
    assert relerr(bad.to(BF16), exact) < 4e-3


def test_checker_rejects_bias_added_twice():
    g = torch.Generator().manual_seed(3)
    A = torch.randn(256, 64, generator=g).to(BF16)
    B = torch.randn(64, 512, generator=g).to(BF16)
    bias = torch.randn(512, generator=g)
    exact = A.double() @ B.double() + bias.double()
    assert_gemm_close(exact.to(BF16), A, B, bias=bias)
    with pytest.raises(AssertionError):
        assert_gemm_close((exact + bias.double()).to(BF16), A, B, bias=bias)
    # the epilogues with a second operand: accepted when right, rejected when the bias is doubled
    C = torch.randn(256, 512, generator=g).to(BF16)
    assert_gemm_close((exact + C.double()).to(BF16), A, B, bias=bias, c_old=C)
    assert_gemm_close((exact.to(BF16).double() + C.double()).to(BF16), A, B, bias=bias, residual=C)
    with pytest.raises(AssertionError):
        assert_gemm_close((exact + bias.double() + C.double()).to(BF16), A, B, bias=bias, residual=C)


def test_checker_rejects_one_scaled_rmsnorm_row():
    """One row of a 4096-row RMSNorm output scaled by (1 + 2^-5): 0.05 % of the tensor's norm, 3 % of the row's."""
    g = torch.Generator().manual_seed(4)
    x = torch.randn(4096, 256, generator=g).to(BF16)
    w = (1 + 0.1 * torch.randn(256, generator=g)).to(BF16)
    ref = R.rms_norm(x.double(), w.double(), 1e-5, "bf16")
    good = ref.to(BF16)
    bad = good.clone()
    bad[1234] = (bad[1234].double() * (1 + 2 ** -5)).to(BF16)
    assert_rows_close(good, ref, ROW_TOL)
    assert_within_ulps(good, ref)
    with pytest.raises(AssertionError):
        assert_rows_close(bad, ref, ROW_TOL)
    with pytest.raises(AssertionError):
        assert_within_ulps(bad, ref)
    assert relerr(bad, ref) < 4e-3
    # never-written output, pre-filled with NaN: the last row and one 8-element chunk of another row (0.03 % of the elements,
    # far below the 1 % of elements allowed to differ by an ulp) must be rejected on their own
    unwritten = good.clone()
    unwritten[-1] = float("nan")
    unwritten[7, 248:256] = float("nan")
    with pytest.raises(AssertionError, match="beyond"):
        assert_within_ulps(unwritten, ref)
    with pytest.raises(AssertionError):
        assert_rows_close(unwritten, ref, ROW_TOL)


def test_checker_rejects_unwritten_output():
    A = torch.randn(200, 64).to(BF16)
    B = torch.randn(64, 300).to(BF16)
    out = (A.double() @ B.double()).to(BF16)
    out[150:, 256:] = float("nan")
    with pytest.raises(AssertionError, match="non-finite"):
        assert_gemm_close(out, A, B)


# ----------------------------------------------------------------------------------------------------------
# GPU helpers
# ----------------------------------------------------------------------------------------------------------
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def randn(shape, g, scale=1.0, dtype=BF16):
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def nan_bf16(*shape):
    return torch.full(shape, float("nan"), dtype=BF16, device=DEV)


def units(spec, W):
    """'W-1' / 'W' / 'W+1' -> one persistent-loop trip of W units and its neighbours; an int is taken as is."""
    return spec if isinstance(spec, int) else {"W-1": W - 1, "W": W, "W+1": W + 1}[spec]


@pytest.fixture
def fp64_reference():
    """fp64 references on the device with no reduced-precision matmul; settings restored, cache released afterwards."""
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old[0], old[1]
    torch.set_float32_matmul_precision(old[2])
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------
# 1. GEMM at the shapes of the two training steps (decoder_engine.py: _layer_fwd, backward, _layer_bwd)
# ----------------------------------------------------------------------------------------------------------
HEAD_DIM = 128
MODELS = {
    "llama3.2-3b": dict(M=4096, h=3072, I=8192, nh=24, kvh=8, V=128256, bias=False),
    "qwen2-1.5b": dict(M=8192, h=1536, I=8960, nh=12, kvh=2, V=151936, bias=True),
}


def _gemm_cases():
    """(id, M, N, K, trans_a, trans_b, epilogue) of every distinct plain GEMM of one training step.  The gate|up forward and
    the down-projection dX run through gemm_swiglu / gemm_swiglu_bwd (tested below)."""
    cases = []
    for name, s in MODELS.items():
        M, h, I, V = s["M"], s["h"], s["I"], s["V"]
        qn = s["nh"] * HEAD_DIM                               # attention output width (o_proj input)
        n_qkv = (s["nh"] + 2 * s["kvh"]) * HEAD_DIM           # fused q|k|v projection width
        cases += [
            (f"{name}-qkv", M, n_qkv, h, False, False, "bias" if s["bias"] else "none"),
            (f"{name}-o", M, h, qn, False, False, "residual"),
            (f"{name}-down", M, h, I, False, False, "residual"),               # K = I > 4608: raster group of 8
            (f"{name}-lm_head", M, V, h, False, False, "none"),
            (f"{name}-lm_head_dX", M, h, V, False, True, "none"),
            (f"{name}-gate_up_dX", M, h, 2 * I, False, True, "none"),
            (f"{name}-o_dX", M, qn, h, False, True, "none"),
            (f"{name}-qkv_dX", M, h, n_qkv, False, True, "none"),
            (f"{name}-lm_head_dW", h, V, M, True, False, "accumulate"),
            (f"{name}-down_dW", I, h, M, True, False, "accumulate"),
            (f"{name}-gate_up_dW", h, 2 * I, M, True, False, "accumulate"),
            (f"{name}-o_dW", qn, h, M, True, False, "accumulate"),
            (f"{name}-qkv_dW", h, n_qkv, M, True, False, "accumulate"),
        ]
    return cases


GEMM_CASES = _gemm_cases()


def _run_gemm(a_st, b_st, M, N, K, ta, tb, epi, max_ctas=0, c_old=None, bias=None, res=None):
    o = ops()
    if epi == "accumulate":
        out = c_old.clone()
    else:
        out = nan_bf16(M, N)
    o.gemm(a_st, b_st, out=out, trans_a=ta, trans_b=tb, accumulate=epi == "accumulate", bias=bias, residual=res,
           max_ctas=max_ctas)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_training_shapes(case, fp64_reference):
    name, M, N, K, ta, tb, epi = case
    g = gen(100 + GEMM_CASES.index(case))
    a_st = randn((K, M) if ta else (M, K), g)
    b_st = randn((N, K) if tb else (K, N), g)
    A = a_st.t() if ta else a_st
    B = b_st.t() if tb else b_st
    bias = torch.randn(N, generator=g, device=DEV) if epi == "bias" else None
    res = randn((M, N), g, math.sqrt(K)) if epi == "residual" else None
    c_old = randn((M, N), g, math.sqrt(K)) if epi == "accumulate" else None
    out = _run_gemm(a_st, b_st, M, N, K, ta, tb, epi, c_old=c_old, bias=bias, res=res)
    st = assert_gemm_close(out, A, B, bias=bias, c_old=c_old, residual=res, what=name)
    print(f"[gemm {name} M={M} N={N} K={K} ta={int(ta)} tb={int(tb)} {epi}] worst err/bound {st['ratio']:.3f} "
          f"c_need {st['c_need']:.2e} worst tile {st['tile']:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_gemm_swiglu_training_shapes(model, fp64_reference):
    """gate|up projection + SwiGLU epilogue (forward), and the down-projection dX GEMM + SwiGLU backward epilogue."""
    o = ops()
    s = MODELS[model]
    M, h, I = s["M"], s["h"], s["I"]
    g = gen(200 + len(model))
    x = randn((M, h), g)
    w = randn((h, 2 * I), g, 1 / math.sqrt(h))
    gu, m = nan_bf16(M, 2 * I), nan_bf16(M, I)
    o.gemm_swiglu(x, w, gate_up=gu, out=m)
    st = assert_gemm_close(gu, x, w, what=f"{model} gate|up")
    print(f"[gemm {model} gate|up M={M} N={2 * I} K={h}] worst err/bound {st['ratio']:.3f} c_need {st['c_need']:.2e} "
          f"worst tile {st['tile']:.2e}")
    gd, ud = gu[:, :I].double(), gu[:, I:].double()
    ref = gd * torch.sigmoid(gd) * ud                      # SwiGLU of the kernel's own (checked) gate|up, fp64
    assert torch.isfinite(m.float()).all()
    assert ((m.double() - ref).abs() <= (BF16_REL + 2.0 ** -20) * ref.abs()).all()     # one rounding + fp32 SFU sigmoid
    del gd, ud, ref
    # backward: d(m) = dY @ W_down^T (K-major B) with the SwiGLU backward in the epilogue == plain dX GEMM + swiglu_bwd kernel
    dy = randn((M, h), g)
    wd = randn((I, h), g, 1 / math.sqrt(h))
    dm = nan_bf16(M, I)
    o.gemm(dy, wd, out=dm, trans_b=True)
    st = assert_gemm_close(dm, dy, wd.t(), what=f"{model} down dX")
    print(f"[gemm {model} down_dX M={M} N={I} K={h} tb=1] worst err/bound {st['ratio']:.3f} c_need {st['c_need']:.2e} "
          f"worst tile {st['tile']:.2e}")
    dgu = nan_bf16(M, 2 * I)
    o.gemm_swiglu_bwd(dy, wd, gu, dgate_up=dgu)
    assert torch.equal(dgu, o.swiglu_bwd(gu, dm))


LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("epi", ["bias", "accumulate", "residual"])
@pytest.mark.parametrize("nwg", [1, 2])
@pytest.mark.parametrize("ta,tb", LAYOUTS)
def test_gemm_tile_to_cta_independence(ta, tb, nwg, epi, fp64_reference):
    """Each output tile is accumulated by one CTA in k order, so the tile -> CTA assignment (max_ctas) changes no bit.
    More tiles than SMs; 23 k-blocks (not a multiple of the 4- or 5-stage ring, so ring phases wrap inside a tile), the last
    one 24 wide; a partial raster group (8 m-tiles of 128 rows, or one of 64, against a group of 16)."""
    sms = sm_count()
    K = 22 * 64 + 24
    if nwg == 2:
        M = 1000
        N = 256 * -(-(sms + 12) // 8) - 8
    else:
        M = 48
        N = 256 * (sms + 12) - 8
    g = gen(300 + 10 * nwg + 2 * ta + tb)
    a_st = randn((K, M) if ta else (M, K), g)
    b_st = randn((N, K) if tb else (K, N), g)
    bias = torch.randn(N, generator=g, device=DEV)
    res = randn((M, N), g, math.sqrt(K)) if epi == "residual" else None
    c_old = randn((M, N), g, math.sqrt(K)) if epi == "accumulate" else None
    ref = _run_gemm(a_st, b_st, M, N, K, ta, tb, epi, 0, c_old, bias, res)
    assert_gemm_close(ref, a_st.t() if ta else a_st, b_st.t() if tb else b_st, bias=bias, c_old=c_old, residual=res,
                      what=f"gemm M={M} N={N} K={K}")
    for k in (1, 2, 7, sms - 1):
        got = _run_gemm(a_st, b_st, M, N, K, ta, tb, epi, k, c_old, bias, res)
        assert torch.equal(got, ref), f"max_ctas={k} changed the result"


@pytest.mark.gpu
@pytest.mark.parametrize("tb", [False, True])
def test_gemm_skinny_split_k(tb, fp64_reference):
    """Split-K decode GEMM with 11 k-blocks (the last 24 wide) cut into 1, 2, 3 and 11 ranges: correct against fp64, and the
    fp32 reduction workspace handed back zeroed so that the next call (different inputs) is correct too."""
    o = ops()
    M, N, K = 48, 776, 10 * 64 + 24
    for split in (1, 2, 3, 11):
        for seed in (0, 1):
            g = gen(400 + 10 * split + seed)
            a = randn((M, K), g)
            b_st = randn((N, K) if tb else (K, N), g)
            bias = torch.randn(N, generator=g, device=DEV)
            out = nan_bf16(M, N)
            o.gemm_skinny(a, b_st, out=out, trans_b=tb, bias=bias, split_k=split)
            assert_gemm_close(out, a, b_st.t() if tb else b_st, bias=bias, what=f"split_k={split} call {seed}")
            ws = o._workspaces[(a.device, "splitk")]
            assert not bool(ws.any()), f"split_k={split}: workspace not zero after the call"


# ----------------------------------------------------------------------------------------------------------
# 2. Row kernels beyond one wave
# ----------------------------------------------------------------------------------------------------------
EPS = 1e-5


def _rows_with_spread(n, h, g):
    """[n, h] bf16 rows whose scales spread over 1/4 .. 4, so every row has its own rstd."""
    scale = torch.exp2(torch.rand(n, 1, generator=g, device=DEV) * 4 - 2)
    return (torch.randn(n, h, generator=g, device=DEV) * scale).to(BF16)


@pytest.mark.gpu
@pytest.mark.parametrize("h", [1536, 3072, 4096, 8192])
@pytest.mark.parametrize("rows", ["W-1", "W", "W+1", 4096, 8192])
def test_rmsnorm_fwd_beyond_one_wave(rows, h):
    """Persistent CTA-per-row forward (h >= 1024): W = 8 * SMs rows per trip; the next-row prefetch and the double-buffered
    warp partials run from the second trip on."""
    o = ops()
    n = units(rows, 8 * sm_count())
    g = gen(500 + h)
    x = _rows_with_spread(n, h, g)
    w = (1 + 0.1 * torch.randn(h, generator=g, device=DEV)).to(BF16)
    y = nan_bf16(n, h)
    rstd = torch.full((n,), float("nan"), device=DEV)
    o.rmsnorm_fwd(x, w, EPS, out=y, rstd=rstd)
    xd = x.double()
    rstd_ref = torch.rsqrt(xd.pow(2).mean(-1) + EPS)
    rel = ((rstd.double() - rstd_ref).abs() / rstd_ref)
    assert rel.max().item() <= 1e-5, f"rstd row {int(rel.argmax())}: relative error {rel.max().item():.2e}"
    # rstd differing in its last fp32 bit can flip the intermediate bf16 rounding and then the final one: two ulps
    ref = R.rms_norm(xd, w.double(), EPS, "bf16")
    assert_within_ulps(y, ref, ulps=2, max_frac=0.01, what=f"rmsnorm y [{n}, {h}]")


@pytest.mark.gpu
@pytest.mark.parametrize("h", [1536, 3072])
@pytest.mark.parametrize("rows", ["W-1", "W", "W+1", 4096])
def test_rmsnorm_bwd_beyond_one_wave(rows, h):
    """RMSNorm backward with the residual gradient and dw accumulation: W = 2 * SMs CTAs, each carrying its dw partial across
    its rows through the software pipeline.  dx per row; dw per column against the fp64 sum over all rows."""
    o = ops()
    n = units(rows, 2 * sm_count())
    g = gen(600 + h)
    x = _rows_with_spread(n, h, g)
    w = (1 + 0.1 * torch.randn(h, generator=g, device=DEV)).to(BF16)
    dy, dres = randn((n, h), g), randn((n, h), g)
    dw0 = randn((h,), g, 4.0)
    rstd = torch.rsqrt(x.double().pow(2).mean(-1) + EPS).float()
    dw = dw0.clone()
    dx = nan_bf16(n, h)
    o.rmsnorm_bwd(dy, x, w, rstd, dw, dres=dres, accumulate_dw=True, dx=dx)
    rs = rstd.double()[:, None]
    xh = x.double() * rs
    gg = dy.double() * w.double()
    dx_ref = rs * (gg - xh * (gg * xh).mean(-1, keepdim=True)) + dres.double()
    assert_rows_close(dx, dx_ref, ROW_TOL, what=f"rmsnorm dx [{n}, {h}]")
    terms = dy.double() * xh.float().to(BF16).double()      # dw sums dy * bf16(x * rstd), the forward's rounded x-hat
    dw_ref = dw0.double() + terms.sum(0)
    mag = dw0.double().abs() + terms.abs().sum(0)
    # one bf16 rounding of the sum, plus the fp32 summation (a few dozen sequential adds per column: << 2^-16 of mag)
    err = (dw.double() - dw_ref).abs()
    bound = BF16_REL * dw_ref.abs() + 2.0 ** -16 * mag
    assert (err <= bound).all(), f"dw column {int((err / bound).argmax())}: error/bound {(err / bound).max().item():.2f}"


@pytest.mark.gpu
@pytest.mark.parametrize("rows,inter", [("W-1", 8), ("W", 8), ("W+1", 8), (4096, 8192), (8192, 8960)])
def test_swiglu_beyond_one_wave(rows, inter):
    """Grid-stride SwiGLU forward and backward: W = 16 * SMs * 256 chunks of 8 channels per trip (one chunk per row in the
    first three cases), and the two benchmark MLP widths."""
    o = ops()
    n = units(rows, 16 * sm_count() * 256)
    g = gen(700 + inter)
    gu = randn((n, 2 * inter), g, 2.0)
    dm = randn((n, inter), g)
    m = nan_bf16(n, inter)
    o.swiglu_fwd(gu, out=m)
    gd, ud = gu[:, :inter].double(), gu[:, inter:].double()
    sg = torch.sigmoid(gd)
    assert_rows_close(m, gd * sg * ud, ROW_TOL, what=f"swiglu fwd [{n}, {inter}]")
    dgu = nan_bf16(n, 2 * inter)
    o.swiglu_bwd(gu, dm, dgate_up=dgu)
    dmd = dm.double()
    assert_rows_close(dgu[:, :inter], dmd * ud * sg * (1 + gd * (1 - sg)), ROW_TOL, what=f"swiglu d(gate) [{n}, {inter}]")
    assert_rows_close(dgu[:, inter:], dmd * gd * sg, ROW_TOL, what=f"swiglu d(up) [{n}, {inter}]")


@pytest.mark.gpu
@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("positions", ["sequence", "position_ids", "wrapped"])
@pytest.mark.parametrize("nh,kvh", [(24, 8), (12, 2)])
def test_rope_at_bench_heads(nh, kvh, positions, backward):
    """RoPE over the q and k heads of the packed projection: 24 + 8 heads (256 threads per token) and 12 + 2 (112 threads,
    not a multiple of 32).  Positions up to the end of an 8192-row table, explicit position_ids, and tokens > seq_len
    (4 sequences of 2048: position = token % seq_len)."""
    o = ops()
    d, T, table = 128, 8192, 8192
    H = nh + kvh
    ld = (nh + 2 * kvh) * d
    cos, sin = o.rope_tables(d, table, 500000.0, DEV)
    g = gen(800 + nh)
    qkv = randn((T, ld), g)
    pid = None
    if positions == "sequence":
        seq_len, pos = T, torch.arange(T, device=DEV)
    elif positions == "wrapped":
        seq_len = 2048
        pos = torch.arange(T, device=DEV) % seq_len
    else:
        seq_len = T
        pos = torch.randint(0, table, (T,), generator=g, device=DEV)
        pos[0], pos[-1] = table - 1, 0
        pid = pos.int()
    x = qkv.clone()
    o.rope_inplace(x, cos, sin, seq_len, H, d, position_ids=pid, backward=backward)
    c, s = cos.double()[pos][:, None, :], sin.double()[pos][:, None, :]
    if backward:
        s = -s
    qk = qkv[:, :H * d].double().view(T, H, d)
    x1, x2 = qk[..., :d // 2], qk[..., d // 2:]
    ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
    assert_rows_close(x[:, :H * d].view(T, H, d), ref, ROW_TOL, what=f"rope {nh}+{kvh} {positions}")
    assert torch.equal(x[:, H * d:], qkv[:, H * d:])                  # v untouched


def _ce_reference(L, labels, ignore_index=-100):
    """fp64 (lse, per-token loss) of logits L [T, V] (any float dtype)."""
    Ld = L.double()
    lse = torch.logsumexp(Ld, -1)
    valid = labels != ignore_index
    lab = labels.clamp_min(0)
    lt = torch.where(valid, lse - Ld.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse))
    return lse, lt


@pytest.mark.gpu
@pytest.mark.parametrize("V,ld", [(128256, 128256), (151936, 151936), (50257, 50264)])
def test_cross_entropy_and_argmax_real_vocab(V, ld):
    """Cross-entropy forward / backward and argmax over 4096 rows of real vocabularies (V = 50 257 takes the scalar tail
    loops; its rows are padded to a multiple of 8).  Labels at column 0 and V - 1, ignored rows, rows at logit scale 30;
    tied maxima in different threads' chunks and in the tail; padding columns never touched."""
    o = ops()
    T = 4096
    g = gen(900 + V % 1000)
    buf = randn((T, ld), g, 2.0)
    buf[::16] = randn((T // 16, ld), g, 30.0)
    buf[:, V:] = 2048.0                                            # above every logit: any read of the padding shows
    big = 1000.0
    ties = {5: [8 * 1030, 8 * 2000 + 3, 8 * 3000], 6: [8 * 900 + 7, 8 * 5], 7: [8 * 6000 + 1, V - 1], 8: [V - 1],
            9: [V - 2, V - 1], 10: [0, V - 1]}
    for r, cols in ties.items():
        buf[r, cols] = big
    logits = buf[:, :V]
    labels = torch.randint(0, V, (T,), generator=g, device=DEV)
    labels[1::10], labels[2::10], labels[3::10] = 0, V - 1, -100
    orig = buf.clone()

    am = o.argmax(logits)
    want = torch.argmax(logits.float(), -1)
    for r, cols in ties.items():
        assert want[r].item() == min(cols)
    assert torch.equal(am, want), f"argmax differs in rows {(am != want).nonzero()[:8, 0].tolist()}"

    loss_out, loss_tok, lse = o.ce_fwd(logits, labels)
    lse_ref, lt_ref = _ce_reference(logits, labels)
    tol = 2e-5 * (1 + lse_ref.abs())
    assert ((lse.double() - lse_ref).abs() <= tol).all(), f"lse row {int(((lse.double() - lse_ref).abs() / tol).argmax())}"
    assert ((loss_tok.double() - lt_ref).abs() <= tol).all(), \
        f"loss row {int(((loss_tok.double() - lt_ref).abs() / tol).argmax())}"
    # the rows that count come from the labels alone; every one of them must have a positive loss (fp64 and kernel), so the
    # criterion's "loss > 0" rule cannot silently drop a labelled row
    keep = labels != -100
    cnt = int(keep.sum())
    assert bool((lt_ref[keep] > 0).all()) and bool((loss_tok[keep] > 0).all())
    mean_ref = lt_ref[keep].sum().item() / cnt
    assert loss_out[1].item() == cnt
    assert abs(loss_out[0].item() - mean_ref) <= 1e-5 * mean_ref

    gs = 0.5
    o.ce_bwd_(logits, labels, loss_tok, lse, loss_out, grad_scale=gs)
    for r0 in range(0, T, 1024):
        Ld = orig[r0:r0 + 1024, :V].double()
        lab = labels[r0:r0 + 1024]
        p = torch.exp(Ld - lse_ref[r0:r0 + 1024, None])
        p[lab >= 0, lab[lab >= 0]] -= 1.0
        p *= torch.where(keep[r0:r0 + 1024], gs / cnt, 0.0)[:, None]
        assert_rows_close(buf[r0:r0 + 1024, :V], p, ROW_TOL, what=f"dlogits rows {r0}.. (V {V})")
        del Ld, p
    assert torch.equal(buf[:, V:], orig[:, V:]), "padding columns between V and ld were written"

    # a batch whose labels are all ignored: loss 0, count 0, all-zero dlogits
    lg = orig[:64].clone()[:, :V]                                   # keeps the padded row stride
    ign = torch.full((64,), -100, dtype=torch.int64, device=DEV)
    lo, lt, ls = o.ce_fwd(lg, ign)
    assert lo[0].item() == 0.0 and lo[1].item() == 0.0
    o.ce_bwd_(lg, ign, lt, ls, lo)
    assert not bool(lg.any())


@pytest.mark.gpu
@pytest.mark.parametrize("clip", [True, False])
@pytest.mark.parametrize("step", [1, 1000])
def test_grad_sqnorm_and_adamw_beyond_one_wave(step, clip):
    """Flat-buffer global norm and AdamW over three grid-stride trips (W = 8 * SMs * 256 * 8 elements) plus 13 chunks, the
    weight-decay boundary at a multiple of 8 inside the second trip.  Per element against optim_ref in fp64."""
    o = ops()
    W = 8 * sm_count() * 256 * 8
    n, decay_end = 3 * W + 8 * 13, W + 8 * 5
    g = gen(1000 + step + clip)
    grads = randn((n + 5,), g, 0.01)
    G = grads[:n]
    master = torch.randn(n, generator=g, device=DEV) * 0.02
    m0 = torch.randn(n, generator=g, device=DEV) * 1e-3
    v0 = torch.rand(n, generator=g, device=DEV) * 1e-5
    scale = 0.5
    g64 = G.double() * scale
    sq_ref = g64.pow(2).sum().item()
    sq = o.grad_sqnorm(G, scale=scale)
    assert abs(sq.item() - sq_ref) <= 1e-5 * sq_ref
    g5 = grads[:n + 5]                                              # n % 8 == 5: the block-0 tail loop
    sq5_ref = (g5.double() * scale).pow(2).sum().item()
    assert abs(o.grad_sqnorm(g5, scale=scale).item() - sq5_ref) <= 1e-5 * sq5_ref

    mgn = 1.0 if clip else 1e3
    assert (math.sqrt(sq_ref) > mgn) == clip
    hp = dict(lr=3e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=step)
    P, MA, M_, V_ = master.to(BF16), master.clone(), m0.clone(), v0.clone()
    o.adamw_step(P, G, MA, M_, V_, sq, decay_end=decay_end, grad_scale=scale, max_grad_norm=mgn, **hp)
    mask = torch.arange(n) < decay_end
    pr, mr, vr, _ = optim_ref.adamw_step(master.double().cpu(), m0.double().cpu(), v0.double().cpu(), G.double().cpu(),
                                         decay_mask=mask, grad_scale=scale, max_grad_norm=mgn, **hp)
    pr, mr, vr = pr.to(DEV), mr.to(DEV), vr.to(DEV)
    geff = (mr - hp["beta1"] * m0.double()) / (1 - hp["beta1"])
    # fp32 arithmetic; (1 - beta2) and the bias corrections are formed from fp32 betas (1 - 0.999f is 1.3e-5 off).  Bounds
    # scale with the magnitudes of the terms, not of their sum: beta1 m0 and (1 - beta1) g can cancel.
    m_mag = hp["beta1"] * m0.double().abs() + (1 - hp["beta1"]) * geff.abs()
    mb = 2.0 ** -18 * m_mag
    vb = 2.0 ** -18 * hp["beta2"] * v0.double() + 2.0 ** -15 * (1 - hp["beta2"]) * geff.pow(2)
    denom = vr.sqrt() / math.sqrt(1 - hp["beta2"] ** step) + hp["eps"]
    upd_mag = hp["lr"] / (1 - hp["beta1"] ** step) * m_mag / denom
    pb = 2.0 ** -22 * master.double().abs() + 2.0 ** -14 * upd_mag
    for name, got, ref, bound in (("exp_avg", M_, mr, mb), ("exp_avg_sq", V_, vr, vb), ("master", MA, pr, pb)):
        err = (got.double() - ref).abs()
        ok = err <= bound
        if not bool(ok.all()):
            i = int((err / bound).argmax())
            raise AssertionError(f"{name}: {int((~ok).sum())} elements beyond their bound; worst at {i}: got {got[i].item():.9e} "
                                 f"ref {ref[i].item():.9e} bound {bound[i].item():.3e} | master {master[i].item():.6e} "
                                 f"m0 {m0[i].item():.6e} v0 {v0[i].item():.6e} g {geff[i].item():.6e} "
                                 f"m {M_[i].item():.9e}/{mr[i].item():.9e} v {V_[i].item():.9e}/{vr[i].item():.9e}")
    assert ((P.double() - pr).abs() <= BF16_REL * pr.abs() + pb).all()        # bf16(master)
