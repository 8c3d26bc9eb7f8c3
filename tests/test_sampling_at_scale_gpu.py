"""Token choice at real vocabularies and serving widths: the ops after the head (token_penalty_multi_scores, softmax_f32_,
top_p_sampling_reject), the composed GenerationInferenceModel._choose path, and penalised or sampled generation end to end.

Every op runs at V = 128 256 (Llama 3) and 151 936 (Qwen2) with up to 1 024 rows, against fp64 restatements written here in
plain torch.  The checkers have CPU tests of their own (no gpu mark), each rejecting a planted fault:
  penalty   a history with entry 0 dropped, a frequency term applied once instead of `times` times, the temperature
            applied before the penalty, an EOS ban that is off by one at cur_len == min_len;
  sampling  a token of probability 0, a token whose fp64 mass strictly above it exceeds top_p by more than the allowance.

Penalty checks, per element: an element no rule touches is the correctly rounded fp32 v / temp, bit for bit; an EOS-banned
element outside the history is the correctly rounded -1e10f / temp; a bad token is -1e10f exactly.  A penalised element
passes four fp32 roundings (v*alpha or v/alpha, times*beta, two subtractions; nvcc may fuse one into an fma) and one
division: within 2 ulps of the largest intermediate term, scaled by 1/temp, plus one ulp of the result.  Near a
cancellation that is many ulps of the result itself, which is why the allowance is taken from the terms.

Generation runs on the dense-cache generate(), the paged-cache generate() (graph and eager) and continuous_generate on a
pool that pre-empts, on a tiny model (vocab 512) and at the Llama-3.2-1B width (2 layers, V = 128 256): a presence penalty
far above the logit range bans every token of the history (the last prompt token and the earlier outputs); every penalised
greedy token passes the teacher-forced check after the fp64 penalty for its own history; no EOS appears before min_length,
greedy or sampled; greedy with a temperature alone passes the plain teacher-forced check.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the tests print these):
  token_penalty_multi_scores  worst penalised error 1.18 ulps of the largest term (bound PEN_ULPS = 2); every other element
                              bit-exact.  A first call at 1 024 rows with a 4 097-wide history: 2 to 24 ms (host clock,
                              workspace allocation included; the steady state was not measured).
  softmax_f32_                worst relative error 3.96e-6 where p >= 2^-126, worst |sum(p) - 1| 3.6e-7, every -1e10 logit
                              exactly 0, padding untouched.
  top_p_sampling_reject       the sampled token's fp64 mass above it stayed below top_p on every row (closest 7.2e-6
                              below); chi-square p-values 0.45 (top_p 1, 300 tokens) and 0.44 (top_p 0.6, 59 tokens).
  _choose                     greedy rows all took the fp64 arg-max of the penalised row.
  generation                  teacher-forced worst gap / TAU (TAU as in the continuous-batching file) 0.80 with
                              penalties (decisive fraction 0.68 at the Llama-3.2-1B width, 0.81 tiny) and 0.64 with a
                              temperature alone; continuous_generate pre-empted 7 (Llama-3.2-1B width) and 9 (tiny) times.
The whole file takes 76 s there.
"""
import functools
import time

import numpy as np
import pytest
import torch

from oracle import generation_ref as G
from oracle import llama_ref as R
from test_continuous_batching_at_scale_gpu import teacher_forced_check

DEV = "cuda:0"
BF16 = torch.bfloat16
VOCABS = (128256, 151936)
HIST = 4097                                  # history width of the penalty tests
NEG = float(np.float32(-1e10))               # the ban value, -1e10f
# penalised elements: rounding error in ulps of the largest intermediate term.  2 is the bound of the four roundings
# (measured worst 1.18)
PEN_ULPS = 2.0
# softmax: relative error per element against fp64 (where p >= 2^-126), and |sum(p) - 1|; about 4x the measured worst
SOFTMAX_REL = 1.6e-5
SOFTMAX_SUM = 1.5e-6
# nucleus: the sampled token's fp64 mass strictly above it may exceed top_p by this much.  The kernel compares an fp32 sum
# of up to 151 936 terms, at most ~50 roundings deep (38 per thread, then the warp and block trees): |error| <= 3e-6, and
# this is 4x that.  Measured, the mass above never exceeded top_p (closest: 7.2e-6 below it).
NUC_ALLOW = 1.2e-5


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


# ----------------------------------------------------------------------------------------------------------
# fp64 restatements and checkers (plain torch: they run on the CPU in their own tests and on the GPU beside the kernels)
# ----------------------------------------------------------------------------------------------------------
def ulp32(x):
    """fp32 ulp at |x| (fp64 tensor), as fp64."""
    f = x.abs().float()
    return (torch.nextafter(f, torch.full_like(f, float("inf"))) - f).double()


def history_counts(pre_ids, V, cur_len):
    """[rows, V] int64 occurrences of each id in the prefix of pre_ids before its first negative entry; rows whose
    cur_len < 0 count nothing (the op skips them)."""
    valid = torch.cumprod((pre_ids >= 0).to(torch.int64), 1).bool() & (cur_len >= 0)[:, None]
    times = torch.zeros(pre_ids.shape[0], V, dtype=torch.int64, device=pre_ids.device)
    times.scatter_add_(1, pre_ids.clamp(min=0), valid.to(torch.int64))
    return times


def penalty_fp64(c):
    """The op's formula in fp64 on the fp32 inputs of case `c`.  Returns (value, class, largest intermediate term); class is
    0 untouched, 1 EOS-banned outside the history, 2 bad token, 3 penalised."""
    v = c["logits"].double()
    rows, V = v.shape
    col = torch.arange(V, device=v.device)
    ban = ((c["cur_len"] >= 0) & (c["cur_len"] < c["min_len"]))[:, None] & torch.isin(col, c["eos"])[None]
    v = torch.where(ban, torch.full_like(v, NEG), v)
    a, b, g, t = (c[k].double()[:, None] for k in ("penalty", "frequency", "presence", "temperature"))
    times = history_counts(c["pre_ids"], V, c["cur_len"])
    hit = times != 0
    vp = torch.where(v < 0, v * a, v / a)
    tb = times.double() * b
    s1 = vp - tb
    s = s1 - g
    term = torch.stack([vp.abs(), tb.abs(), s1.abs(), s.abs()]).amax(0)
    del tb, s1
    val = torch.where(hit, s, v) / t
    bad = torch.isin(col, c["bad"])[None].expand(rows, V)
    val = torch.where(bad, torch.full_like(val, NEG), val)
    cls = torch.zeros(rows, V, dtype=torch.int8, device=v.device)
    cls[ban & ~hit] = 1
    cls[hit] = 3
    cls[bad] = 2
    return val, cls, torch.where(hit, term, torch.zeros_like(term))


def check_penalty(got, c):
    """Assert the op's output `got` [rows, V] fp32 against penalty_fp64 of case `c`; returns the worst penalised error in
    ulps of the largest term (the bound is PEN_ULPS)."""
    val, cls, term = penalty_fp64(c)
    t = c["temperature"].double()[:, None].expand_as(val)

    def exact(mask, want, what):
        bad = mask & (got.view(torch.int32) != want.view(torch.int32))
        if bool(bad.any()):
            r, i = (int(x) for x in bad.nonzero()[0])
            raise AssertionError(f"{what} element (row {r}, token {i}): {got[r, i].item()!r}, expected {want[r, i].item()!r}")

    # v / temp and -1e10f / temp, correctly rounded: the fp64 quotient of fp32 operands rounds to the fp32 quotient
    exact(cls == 0, (c["logits"].double() / t).float(), "untouched")
    exact(cls == 1, (torch.full_like(val, NEG) / t).float(), "EOS-banned")
    exact(cls == 2, torch.full_like(got, NEG), "bad-token")
    pen = cls == 3
    err = (got.double() - val).abs() - ulp32(val)
    ratio = torch.where(pen, err / (ulp32(term) / t), torch.zeros_like(err))
    worst = ratio.max().item() if bool(pen.any()) else 0.0
    if not worst <= PEN_ULPS:                                        # NaN fails
        r, i = (int(x) for x in (ratio == ratio.max()).nonzero()[0]) if worst == worst else (0, 0)
        raise AssertionError(f"penalised element (row {r}, token {i}): {got[r, i].item()!r}, fp64 {val[r, i].item()!r}, "
                             f"{worst:.2f} ulps of the largest term (allowed {PEN_ULPS})")
    return worst


def penalty_case(rows, V, seed, device, width=HIST):
    """Histories (by row): empty (entry 0 is -1, junk after it), full, ragged, one id ~4000 times, ids 0 and V-1 with an
    EOS id inside, a single entry.  cur_len at min_len - 1, min_len, -1 or past it; three EOS ids; bad tokens with V-1;
    penalty below and above 1; frequency, presence and temperature in [0.3, 2]; logits of both signs and zeros."""
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape):
        return torch.rand(*shape, generator=g, dtype=torch.float64)

    eos = torch.tensor([2, V // 2 + 1, V - 2])
    pre = torch.randint(0, V, (rows, width), generator=g)
    kind = (torch.arange(rows) + 3) % 6                              # a single row gets the repeated id
    for r in range(rows):
        k = int(kind[r])
        if k == 0:
            pre[r, 0] = -1
        elif k == 2:
            pre[r, int(torch.randint(1, width, (1,), generator=g)):] = -1
        elif k == 3:
            pre[r, :width - 97] = int(torch.randint(0, V, (1,), generator=g))
        elif k == 4:
            n = int(torch.randint(8, width, (1,), generator=g))
            pre[r, [0, 1, n - 1, n // 2]] = torch.tensor([0, V - 1, V - 1, int(eos[r % 3])])
            pre[r, n:] = -1
        elif k == 5:
            pre[r, 1:] = -1
    min_len = torch.randint(1, 50, (rows,), generator=g)
    sel = (torch.arange(rows) // 6) % 4
    cur_len = torch.where(sel == 0, min_len - 1, torch.where(sel == 1, min_len, torch.where(
        sel == 2, torch.full_like(min_len, -1), min_len + torch.randint(0, 100, (rows,), generator=g))))
    logits = (torch.randn(rows, V, generator=g) * 5).float()
    logits[rnd(rows, V) < 0.05] = 0.0
    pen = torch.where(torch.arange(rows) % 2 == 0, 0.5 + 0.45 * rnd(rows), 1.05 + 0.95 * rnd(rows)).float()
    c = dict(pre_ids=pre, logits=logits, penalty=pen, frequency=(0.3 + 1.7 * rnd(rows)).float(),
             presence=(0.3 + 1.7 * rnd(rows)).float(), temperature=(0.3 + 1.7 * rnd(rows)).float(), cur_len=cur_len,
             min_len=min_len, eos=eos, bad=torch.tensor([5, 1000 % V, V - 1]))
    return {k: v.to(device) for k, v in c.items()}


def penalty_restated(c, fault=None):
    """The op in fp32 torch arithmetic (each operation correctly rounded, no fma), with an optional planted fault."""
    logits = c["logits"].clone()
    rows, V = logits.shape
    col = torch.arange(V, device=logits.device)
    pre = c["pre_ids"].clone()
    if fault == "history_entry_0_dropped":
        pre[:, 0] = -1
    lim = c["cur_len"] <= c["min_len"] if fault == "eos_ban_off_by_one" else c["cur_len"] < c["min_len"]
    ban = ((c["cur_len"] >= 0) & lim)[:, None] & torch.isin(col, c["eos"])[None]
    v = torch.where(ban, torch.full_like(logits, NEG), logits)
    a, b, g, t = (c[k][:, None] for k in ("penalty", "frequency", "presence", "temperature"))
    if fault == "temperature_first":
        v = v / t
    times = history_counts(pre, V, c["cur_len"])
    if fault == "frequency_once":
        times = (times > 0).to(torch.int64)
    vp = torch.where(v < 0, v * a, v / a)
    v = torch.where(times != 0, (vp - times.float() * b) - g, v)
    if fault != "temperature_first":
        v = v / t
    return torch.where(torch.isin(col, c["bad"])[None], torch.full_like(v, NEG), v)


def mass_above(p64, tok):
    """fp64 mass strictly above each row's sampled token: p64 [rows, V], tok [rows]."""
    pt = p64.gather(1, tok[:, None])
    return torch.where(p64 > pt, p64, torch.zeros_like(p64)).sum(-1)


def check_sample(tok, p, top_p, what=""):
    """Every sampled token lies in its row's support (p > 0, a real column) and in its fp64 nucleus: the mass strictly above
    it is below top_p + NUC_ALLOW.  p [rows, V] fp32 (the probabilities the sampler read), tok [rows].  Returns the worst
    (mass above - top_p)."""
    rows, V = p.shape
    assert bool(((tok >= 0) & (tok < V)).all()), f"{what}: token outside [0, {V})"
    pt = p.gather(1, tok[:, None])[:, 0]
    if not bool((pt > 0).all()):
        r = int((pt <= 0).nonzero()[0])
        raise AssertionError(f"{what}: row {r} sampled token {int(tok[r])} of probability {pt[r].item()!r}")
    over = mass_above(p.double(), tok) - top_p.double()
    worst = over.max().item()
    if not worst < NUC_ALLOW:
        r = int(over.argmax())
        raise AssertionError(f"{what}: row {r} token {int(tok[r])}: fp64 mass above it exceeds top_p {top_p[r].item():.3f} "
                             f"by {worst:.3g}")
    return worst


# ----------------------------------------------------------------------------------------------------------
# the checkers reject planted faults (CPU)
# ----------------------------------------------------------------------------------------------------------
def _small_case():
    return penalty_case(24, 1000, seed=1, device="cpu", width=80)


def test_penalty_checker_accepts_the_restatements():
    c = _small_case()
    got = penalty_restated(c)
    check_penalty(got, c)
    ref = G.token_penalty_multi_scores_v2(c["pre_ids"].numpy(), c["logits"].numpy(), c["penalty"].numpy(),
                                          c["frequency"].numpy(), c["presence"].numpy(), c["temperature"].numpy(),
                                          c["bad"].numpy(), c["cur_len"].numpy(), c["min_len"].numpy(), c["eos"].numpy())
    check_penalty(torch.from_numpy(ref), c)
    val, cls, _ = penalty_fp64(c)
    assert {int(x) for x in cls.unique()} == {0, 1, 2, 3}           # every class occurs


@pytest.mark.parametrize("fault,match", [("history_entry_0_dropped", "penalised"), ("frequency_once", "penalised"),
                                         ("temperature_first", "penalised"), ("eos_ban_off_by_one", "untouched")])
def test_penalty_checker_rejects(fault, match):
    c = _small_case()
    with pytest.raises(AssertionError, match=match):
        check_penalty(penalty_restated(c, fault), c)


def _nucleus_row():
    p = torch.tensor([[0.5, 0.25, 0.125, 0.0625, 0.0625, 0.0]])
    return p, torch.tensor([0.6])


def test_sample_checker_accepts_the_nucleus():
    p, tp = _nucleus_row()
    assert check_sample(torch.tensor([1]), p, tp) < 0 and check_sample(torch.tensor([0]), p, tp) < 0


def test_sample_checker_rejects_a_zero_probability_token():
    p, tp = _nucleus_row()
    with pytest.raises(AssertionError, match="probability 0.0"):
        check_sample(torch.tensor([5]), p, torch.ones(1))


def test_sample_checker_rejects_a_token_outside_the_nucleus():
    p, tp = _nucleus_row()
    with pytest.raises(AssertionError, match="exceeds top_p"):
        check_sample(torch.tensor([2]), p, tp)                        # mass above 0.75 >= 0.6
    q = torch.tensor([[0.5, 0.5 - 2 * NUC_ALLOW, 2 * NUC_ALLOW]])      # mass above token 2 is top_p + 2 allowances
    with pytest.raises(AssertionError, match="exceeds top_p"):
        check_sample(torch.tensor([2]), q, torch.tensor([1.0 - 4 * NUC_ALLOW]))


def test_restatement_top_p_falls_back_inside_the_support():
    """The row of 1 023 tokens of 2^-10 at V = 128 256 sums to 1 - 2^-10 < u: no CDF value exceeds u, and the sampler must
    return the last token with mass, not V - 1 (p = 0)."""
    V = 128256
    p = np.zeros((2, V), np.float32)
    p[:, :1023] = 2.0 ** -10
    u = np.full((32, 2), 1 - 2.0 ** -12, np.float32)
    assert G.top_p_sampling_reject(p, np.array([1.0, 0.95], np.float32), u).tolist() == [1022, 1022]


# ----------------------------------------------------------------------------------------------------------
# token_penalty_multi_scores
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("rows", [1, 64, 1024])
def test_token_penalty_at_real_vocab(V, rows):
    c = penalty_case(rows, V, seed=rows + V, device=DEV)
    got = c["logits"].clone()
    t0 = time.perf_counter()
    ops().token_penalty_multi_scores(c["pre_ids"], got, c["penalty"], c["frequency"], c["presence"], c["temperature"],
                                     c["bad"], c["cur_len"], c["min_len"], c["eos"])
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    worst = check_penalty(got, c)
    print(f"[penalty V {V} rows {rows}] worst penalised error {worst:.3f} ulps of the largest term; one call {ms:.2f} ms "
          f"(host clock, first call)")


# ----------------------------------------------------------------------------------------------------------
# softmax_f32_
# ----------------------------------------------------------------------------------------------------------
def softmax_rows(rows, V, ld, seed):
    """[rows, ld] fp32 with NaN padding.  Rows cycle through: random logits scaled by 1/temperature (0.3 .. 2), the same
    with a third of the entries at -1e10, one dominant logit, all-equal logits."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.full((rows, ld), float("nan"), dtype=torch.float32, device=DEV)
    temp = 0.3 + 1.7 * torch.rand(rows, 1, generator=g, device=DEV)
    x[:, :V] = torch.randn(rows, V, generator=g, device=DEV) * 2 / temp
    kind = torch.arange(rows, device=DEV) % 4
    banned = (kind == 1)[:, None] & (torch.rand(rows, V, generator=g, device=DEV) < 1 / 3)
    x[:, :V] = torch.where(banned, torch.full_like(x[:, :V], NEG), x[:, :V])
    top = torch.randint(0, V, (rows,), generator=g, device=DEV)
    dom = (kind == 2).nonzero()[:, 0]
    x[dom, top[dom]] += 40.0
    eq = (kind == 3).nonzero()[:, 0]
    x[eq, :V] = torch.randn(eq.numel(), 1, generator=g, device=DEV)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("pad", [0, 4, 64])
def test_softmax_f32_at_real_vocab(V, pad):
    rows = 1024
    x = softmax_rows(rows, V, V + pad, seed=V + pad)
    ref = torch.softmax(x[:, :V].double(), -1)
    p = x.clone()
    ops().softmax_f32_(p[:, :V] if pad else p)
    torch.cuda.synchronize()
    assert bool(torch.isnan(p[:, V:]).all()), "padding written"
    q = p[:, :V]
    assert bool((q[x[:, :V] == NEG] == 0).all()), "a -1e10 logit has nonzero probability"
    err = (q.double() - ref).abs()
    normal = ref >= 2.0 ** -126                                      # fp32 keeps full precision down to 2^-126
    rel = torch.where(normal, err / ref, torch.zeros_like(err)).max().item()
    small = torch.where(normal, torch.zeros_like(err), err).max().item()
    dsum = (q.double().sum(-1) - 1).abs().max().item()
    print(f"[softmax V {V} ld V+{pad}] worst relative error {rel:.3g}, worst absolute error below 2^-126 {small:.3g}, "
          f"worst |sum - 1| {dsum:.3g}")
    assert rel <= SOFTMAX_REL and small <= 2.0 ** -126 and dsum <= SOFTMAX_SUM, (rel, small, dsum)
    # the pitched call writes the same bits as the dense one
    dense = x[:, :V].contiguous()
    ops().softmax_f32_(dense)
    assert torch.equal(dense, q)


# ----------------------------------------------------------------------------------------------------------
# top_p_sampling_reject
# ----------------------------------------------------------------------------------------------------------
TOP_PS = (0.0, 0.25, 0.6, 0.95, 1.0)


def _padded(p, pad, fill=1.0):
    """p [rows, V] in a [rows, V + pad] buffer whose padding holds `fill` (a sampler reading it would return a pad column)."""
    rows, V = p.shape
    buf = torch.full((rows, V + pad), fill, dtype=torch.float32, device=DEV)
    buf[:, :V] = p
    return buf[:, :V]


def dyadic_rows(rows, V, seed):
    """Probabilities that are multiples of 2^-23 summing to exactly 1: every partial sum is exact in fp32 whatever the
    summation order.  A third of the entries are 0, the first 7 always; some rows hold a dominant token or mass at V - 1."""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 32, size=(rows, V), dtype=np.int32)
    w[rng.random((rows, V), dtype=np.float32) < 1 / 3] = 0
    w[:, :7] = 0
    r = np.arange(rows)
    w[r[r % 7 == 0], rng.integers(7, V, size=int((r % 7 == 0).sum()))] = 2 ** 21
    w[r % 5 == 1, V - 1] = 2 ** 20
    w[:, 500] += (2 ** 23 - w.sum(-1, dtype=np.int64)).astype(np.int32)
    assert (w >= 0).all() and (w.sum(-1, dtype=np.int64) == 2 ** 23).all()
    return w.astype(np.float32) * np.float32(2.0 ** -23)


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_top_p_bit_exact_against_restatement_at_real_vocab(V):
    rows = 1024
    p = dyadic_rows(rows, V, seed=V)
    tp = np.array([TOP_PS[i % len(TOP_PS)] for i in range(rows)], np.float32)
    rng = np.random.default_rng(V + 1)
    u = ((rng.integers(0, 2 ** 16, size=(32, rows)) + 0.5) / 2 ** 16).astype(np.float32)
    got = ops().top_p_sampling_reject(_padded(torch.from_numpy(p).to(DEV), 4), torch.from_numpy(tp).to(DEV),
                                      uniform=torch.from_numpy(u).to(DEV)).cpu().numpy()
    want = G.top_p_sampling_reject(p, tp, u)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} rows differ, first row {bad[:1]}: {got[bad[:1]]} vs {want[bad[:1]]}"
    check_sample(torch.from_numpy(got), torch.from_numpy(p), torch.from_numpy(tp), "dyadic rows")


def support_rows(V, seed):
    """Rows whose fp32 total is below u = 1 - 2^-12, so that no CDF value exceeds u, with p[V - 1] = 0: 1 023 tokens of
    2^-10 at the start, scattered, and just before V - 1; and a softmax row scaled by 1 - 2^-10."""
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(4, V)
    p[0, :1023] = 2.0 ** -10
    p[1, torch.randperm(V - 1, generator=g)[:1023]] = 2.0 ** -10
    p[2, V - 1024:V - 1] = 2.0 ** -10
    p[3, :V - 1] = torch.softmax(torch.randn(V - 1, generator=g, dtype=torch.float64), -1) * (1 - 2.0 ** -10)
    return p.float()


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_top_p_samples_inside_the_support(V):
    """The sampler must not return a token of probability 0 when the row's fp32 total is at most u (fails with the
    reference's fall-back to V - 1)."""
    p = support_rows(V, seed=V).repeat(2, 1)
    tp = torch.tensor([1.0] * 4 + [0.95] * 4)
    u = torch.full((32, 8), 1 - 2.0 ** -12)
    got = ops().top_p_sampling_reject(_padded(p.to(DEV), 64), tp.to(DEV), uniform=u.to(DEV)).cpu()
    check_sample(got, p, tp, "rows summing below u")
    dy = [0, 1, 2, 4, 5, 6]                                          # the dyadic rows: bit-exact against the restatement
    assert got[dy].tolist() == G.top_p_sampling_reject(p[dy].numpy(), tp[dy].numpy(), u[:, dy].numpy()).tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_top_p_on_softmax_rows_at_real_vocab(V):
    """Real softmax rows from softmax_f32_ in a pitched buffer (padding 1.0), per-row top_p: the token is in the fp64
    nucleus, has p > 0 (rows with banned tokens among them) and is never a padding column."""
    rows = 1024
    x = softmax_rows(rows, V, V + 64, seed=V + 7)
    x[:, V:] = 1.0
    ops().softmax_f32_(x[:, :V])
    p = x[:, :V]
    tp = torch.tensor([TOP_PS[1 + i % 4] for i in range(rows)], device=DEV)
    worst = -1.0
    for seed in range(4):
        g = torch.Generator(device=DEV).manual_seed(seed)
        tok = ops().top_p_sampling_reject(p, tp, generator=g)
        worst = max(worst, check_sample(tok, p, tp, f"softmax rows seed {seed}"))
    print(f"[top-p softmax rows V {V}] worst (fp64 mass above the token - top_p) {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("top_p", [1.0, 0.6])
def test_top_p_frequencies_follow_the_nucleus(top_p):
    """300 tokens with mass, at scattered places of a V = 128 256 row; 60 000 seeded draws (explicit uniforms).  The counts
    must follow p renormalised over the nucleus {mass strictly above < top_p} (chi-square, p-value > 1e-3); no other token
    may occur."""
    from scipy.stats import chisquare

    V, K, N = 128256, 300, 60000
    g = torch.Generator().manual_seed(11)
    where = torch.randperm(V, generator=g)[:K]
    w = (torch.arange(K, dtype=torch.float64) + 1) ** -0.8 * (0.5 + torch.rand(K, generator=g, dtype=torch.float64))
    p = torch.zeros(V, dtype=torch.float64)
    p[where] = w / w.sum()
    p32 = p.float()
    above = torch.stack([p32[p32 > p32[i]].double().sum() for i in where])
    nucleus = above < top_p
    if top_p < 1:
        assert (above - top_p).abs().min() > 1e-3                   # no token near the nucleus edge
    u = torch.rand(32, N, generator=torch.Generator().manual_seed(12)).to(DEV)
    tok = ops().top_p_sampling_reject(p32.to(DEV)[None].expand(N, V), torch.full((N,), top_p, device=DEV), uniform=u).cpu()
    counts = torch.bincount(tok, minlength=V)
    assert int(counts.sum()) == N and int(counts[where[nucleus]].sum()) == N, "a token outside the nucleus was drawn"
    exp = p32[where[nucleus]].double()
    exp = exp / exp.sum() * N
    obs = counts[where[nucleus]].double()
    order = torch.argsort(exp, descending=True)
    exp, obs = exp[order], obs[order]
    keep = exp >= 5                                                  # pool the bins expected below 5 counts
    e = torch.cat([exp[keep], exp[~keep].sum()[None]]) if bool((~keep).any()) else exp
    o = torch.cat([obs[keep], obs[~keep].sum()[None]]) if bool((~keep).any()) else obs
    pv = chisquare(o.numpy(), e.numpy()).pvalue
    print(f"[top-p frequencies top_p {top_p}] {int(nucleus.sum())} tokens in the nucleus, chi-square p-value {pv:.3g}")
    assert pv > 1e-3, pv


# ----------------------------------------------------------------------------------------------------------
# the composed _choose path
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_choose_at_real_vocab(V):
    """bf16 logits through GenerationInferenceModel._choose at 1 024 rows: with penalties the greedy token is the fp64
    arg-max up to the penalty allowance of the top two; sampled tokens lie in the fp64 nucleus with p > 0."""
    from paddlenlp_b200.experimental.transformers.generation_utils import GenerationInferenceModel

    rows = 1024
    c = penalty_case(rows, V, seed=V + 3, device=DEV)
    lg = (c["logits"] * 0.6).to(BF16)
    c["logits"] = lg.float()
    c["bad"] = torch.empty(0, dtype=torch.int64, device=DEV)        # _choose passes no bad tokens
    st = dict(pre_ids=c["pre_ids"], penalty=c["penalty"], frequency=c["frequency"], presence=c["presence"],
              temperature=c["temperature"], step_idx=c["cur_len"], min_dec_len=c["min_len"], eos=c["eos"], plain=False,
              top_p=None, generator=None)
    tok = GenerationInferenceModel._choose(None, lg, st)
    val, _, term = penalty_fp64(c)
    allow = PEN_ULPS * ulp32(term) / c["temperature"].double()[:, None] + ulp32(val)
    best = val.argmax(-1)
    chosen = val.gather(1, tok[:, None])[:, 0]
    slack = allow.gather(1, best[:, None])[:, 0] + allow.gather(1, tok[:, None])[:, 0]
    short = val.max(-1).values - chosen
    assert bool((short <= slack).all()), f"greedy rows off the fp64 arg-max: {(short > slack).nonzero()[:4, 0].tolist()}"
    print(f"[_choose greedy V {V}] {int((tok != best).sum())} rows take another token within the allowance")
    p64 = torch.softmax(val, -1)
    tp = torch.tensor([TOP_PS[1 + i % 4] for i in range(rows)], device=DEV)
    worst = -1.0
    for seed in (1, 2):
        st.update(top_p=tp, generator=torch.Generator(device=DEV).manual_seed(seed))
        tok = GenerationInferenceModel._choose(None, lg, st)
        worst = max(worst, check_sample(tok, p64, tp, f"_choose sampled, seed {seed}"))
    print(f"[_choose sampled V {V}] worst (fp64 mass above the token - top_p) {worst:.3g}")


# ----------------------------------------------------------------------------------------------------------
# end to end: generate() (dense and paged cache) and continuous_generate
# ----------------------------------------------------------------------------------------------------------
E2E = {
    "tiny": dict(model_type="llama", tied=False, scale=4.0, vocab_size=512, hidden_size=128, intermediate_size=344,
                 num_attention_heads=2, num_key_value_heads=1, rms_norm_eps=1e-5, rope_theta=10000.0, requests=24,
                 max_prompt=40, new=64, block_size=32, max_batch_size=8, num_blocks=6),
    "llama3_2_1b": dict(model_type="llama", tied=True, scale=1.0, vocab_size=128256, hidden_size=2048, intermediate_size=8192,
                        num_attention_heads=32, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, requests=16,
                        max_prompt=40, new=64, block_size=32, max_batch_size=8, num_blocks=6),
}
PATHS = ("dense", "paged_graph", "paged_eager", "continuous")
PRESENCE = 1e4                     # far above the logit range: a history token can never win
PENALTIES = dict(penalty_score=1.3, frequency_score=0.4, presence_score=0.6, temperature=0.7)
MIN_LEN = 6


@functools.lru_cache(maxsize=None)
def _e2e(width):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    spec = dict(E2E[width])
    model_type, tied, scale = spec.pop("model_type"), spec.pop("tied"), spec.pop("scale")
    run = {k: spec.pop(k) for k in ("requests", "max_prompt", "new", "block_size", "max_batch_size", "num_blocks")}
    kw = dict(num_hidden_layers=2, max_position_embeddings=128, **spec)
    cfg = R.RefConfig(model_type=model_type, **kw)
    w = R.init_weights(cfg, seed=9)
    w = {k: (v * scale).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    if tied:
        w.pop("lm_head.weight")
    train = T.LlamaForCausalLM(T.LlamaConfig(tie_word_embeddings=tied, **kw))
    train.set_state_dict(w)
    models = {}
    for name, extra in (("dense", {}), ("paged", dict(block_attn=True, block_size=run["block_size"])),
                        ("append", dict(block_attn=True, append_attn=True, block_size=run["block_size"]))):
        models[name] = LlamaForCausalLMInferenceModel(T.LlamaConfig(tie_word_embeddings=tied, **kw), **extra)
        models[name].set_state_dict(w)
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, cfg.vocab_size, (int(torch.randint(1, run["max_prompt"] + 1, (1,), generator=g)),),
                             generator=g) for _ in range(run["requests"])]

    def fwd(ids):
        return train.engine.forward_logits(ids.to(DEV)[None])[0].float()
    return models, prompts, run, fwd


def _run(width, path, min_length=0, **kw):
    """Generate run["new"] tokens for every prompt on one path; returns (one 1-D tensor per request, stats or None)."""
    models, prompts, run, _ = _e2e(width)
    new = run["new"]
    if path == "continuous":
        reqs = [(p, new, min_length) for p in prompts]
        return models["append"].continuous_generate(reqs, max_batch_size=run["max_batch_size"],
                                                    num_blocks=run["num_blocks"], **kw)
    B, S = len(prompts), max(p.numel() for p in prompts)
    ids = torch.zeros(B, S, dtype=torch.int64)
    for b, p in enumerate(prompts):
        ids[b, :p.numel()] = p
    enc = torch.tensor([p.numel() for p in prompts], dtype=torch.int32)
    m = models["dense" if path == "dense" else "paged"]
    out, _, _ = m.generate(ids.to(DEV), seq_len_encoder=enc.to(DEV), max_length=new, min_length=min_length,
                           use_cuda_graph=path != "paged_eager", **kw)
    out = out.cpu()
    return [out[b] for b in range(B)], None


def penalised_rows(rows, prompt, out, penalty_score=1.0, frequency_score=0.0, presence_score=0.0, temperature=1.0,
                   min_length=0, eos=()):
    """fp64 penalties on the rows that predict out[t] (row t): history = the last prompt token + out[:t], cur_len = t;
    EOS-banned entries become -inf."""
    T, V = rows.shape
    hist = torch.cat([prompt[-1:], out[:T - 1]])
    times = torch.zeros(T, V, dtype=torch.float64)
    times[torch.arange(T), hist] = 1.0
    times = times.cumsum(0)
    v = rows
    hit = times > 0
    vp = torch.where(v < 0, v * penalty_score, v / penalty_score)
    v = torch.where(hit, vp - times * frequency_score - presence_score, v) / temperature
    if len(eos) and min_length > 0:
        v[:min(min_length, T), list(eos)] = -float("inf")
    return v


def _history_hits(prompts, outs):
    """(request, position) pairs whose token is already in its history (last prompt token + earlier outputs)."""
    hits = []
    for r, (p, o) in enumerate(zip(prompts, outs)):
        seen = {int(p[-1])}
        for t, x in enumerate(o.tolist()):
            if x in seen:
                hits.append((r, t))
            seen.add(x)
    return hits


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("width", list(E2E))
def test_presence_penalty_bans_the_history(width, path):
    """presence_score far above the logit range: no generated token repeats its history (fails where generate() leaves
    the history without the last prompt token); the same greedy run without penalties does repeat one."""
    _, prompts, _, _ = _e2e(width)
    plain, _ = _run(width, path)
    assert _history_hits(prompts, plain), "the unpenalised run never repeats its history: the test would be vacuous"
    outs, stats = _run(width, path, presence_score=PRESENCE)
    hits = _history_hits(prompts, outs)
    assert not hits, f"{len(hits)} tokens repeat their history, first (request, position) {hits[0]}"
    assert all(o.numel() == len(plain[0]) for o in outs)
    if stats is not None:
        assert stats["preemptions"] > 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("width", list(E2E))
def test_penalised_greedy_matches_training_forward(width, path):
    """Repetition, frequency and presence penalties with a temperature: every token is checked teacher-forced against the
    training-path forward after the fp64 penalty for its own history (in continuous_generate this also catches a recycled
    slot that keeps the previous request's history)."""
    _, prompts, run, fwd = _e2e(width)
    outs, stats = _run(width, path, **PENALTIES)
    reqs = [(p, run["new"]) for p in prompts]
    worst, frac, copy, n = teacher_forced_check(fwd, reqs, outs,
                                                transform=lambda r, lg, p, o: penalised_rows(lg, p, o, **PENALTIES))
    print(f"[{width} {path} penalised] teacher-forced over {n} positions: worst gap / tau {worst:.3f}, decisive fraction "
          f"{frac:.3f}, copy {copy:.3f}; stats {stats}")
    if stats is not None:
        assert stats["preemptions"] > 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("width", list(E2E))
def test_min_length_holds_back_eos(width, path):
    """EOS is a token the unconstrained run emits before min_length: with min_length no EOS appears before it, greedy or
    sampled at top_p = 1."""
    _, prompts, _, _ = _e2e(width)
    plain, _ = _run(width, path)
    early = torch.cat([o[:MIN_LEN] for o in plain])
    eos = int(torch.bincount(early).argmax())
    for kw in (dict(), dict(top_p=1.0, seed=5)):
        outs, _ = _run(width, path, min_length=MIN_LEN, eos_token_id=eos, **kw)
        for r, o in enumerate(outs):
            assert eos not in o[:MIN_LEN].tolist(), (kw, r, o[:MIN_LEN].tolist(), eos)
            assert o.numel() >= MIN_LEN, (kw, r, o.numel())


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("width", list(E2E))
def test_temperature_alone_keeps_greedy_tokens(width, path):
    """Dividing distinct bf16 logits by a positive temperature keeps them distinct and ordered in fp32: greedy decoding
    with temperature 0.7 (the fp32 penalty path) passes the plain teacher-forced check."""
    _, prompts, run, fwd = _e2e(width)
    outs, _ = _run(width, path, temperature=0.7)
    worst, frac, _, n = teacher_forced_check(fwd, [(p, run["new"]) for p in prompts], outs)
    print(f"[{width} {path} temperature 0.7] teacher-forced over {n} positions: worst gap / tau {worst:.3f}")
