"""Continuous batching at serving scale: the step kernels across warps up to 1 024 slots, append_attention over one
serving-shaped mixed step, and continuous_generate at preset widths against the training-path forward.

The step kernels (step_paddle, retire_admit, update_inputs in generation.cu) are single 1 024-thread CTAs whose list
positions, victim arg-max and stop count cross warps through shared memory; at a handful of slots only warp 0 ever works.
Here whole request queues run at 33, 256, 1 000 and 1 024 slots with the device state kept on the device across steps, and
again with the state copied from the host before every step (which points to the first call that diverges); every field
must equal the numpy restatements after every step, and the run must have taken the cross-warp paths it is meant to test.

append_attention is checked per (row, head) against fp64 on a 256-slot step: prompts at every q-tile and page edge admitted
beside 234 decode rows, a prompt chunk on an unaligned cached prefix, idle slots in the middle and at the end, pages
recycled from retired slots and filled with NaN, and rows past every sequence's length NaN.

continuous_generate runs several hundred requests at the Llama-3.2-1B and Qwen2-1.5B widths (two layers) on a pool tight
enough to pre-empt, with every cache row the step must not read poisoned with NaN before every append_attention call (in the
captured graphs too).  Each generated token is checked teacher-forced against the training-path forward of the request's
prompt + output: the chosen token's logit must lie within TAU * max|logits| of the row's maximum at every position, so a
decode that goes wrong after a near-tie still fails where it goes wrong.  The checker's own CPU tests (no gpu mark) show it
rejects a shifted, a corrupted, a swapped and a truncated output, and a reference model that only copies its input token.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, over every case below (the tests print these):
  append_attention, d = 64 and 128, block sizes 32 / 64 / 128, auto and 7 splits:
    decode rows   worst element error / bound 0.995 (the half-ulp term), c_need <= 4.6e-8, worst (row, head) rel. error
                  2.5e-3
    prompt rows   worst element error / bound 0.49, c_need <= 2.9e-3, worst (row, head) rel. error 3.7e-3
  continuous_generate, teacher-forced: worst gap / TAU 0.76 at the Llama-3.2-1B width (decisive fraction 0.81; the
  reference predicts a prompt row's own token at 1.6 % of the prompt rows; 33 of 400 requests part from the eager run at a
  near-tie) and 0.87 at the Qwen2-1.5B width (decisive fraction 0.77; 0.0 %; 85 of 240 requests part at a near-tie).
The whole file takes 107 s there.
"""
import math
import time

import numpy as np
import pytest
import torch

import continuous_sim as sim
import step_sim
from oracle import generation_ref as G
from oracle import llama_ref as R
from oracle import retire_admit_ref as RA
from test_decode_attention_at_scale_gpu import assert_attention_close

DEV = "cuda:0"
BF16 = torch.bfloat16
# append_attention allowances, about 4x / 1.5x the measured worst (see the header): decode rows run the fp32 decode kernel,
# prompt rows the flash-attention kernel, which rounds P to bf16 before P V
DECODE_C, DECODE_HEAD_TOL = 2e-7, 4e-3
PREFILL_C, PREFILL_HEAD_TOL = 1e-2, 6e-3
# teacher-forced bound: the bound the benchmark-width decode test asserts between cached decode and the uncached forward
TAU = 2e-2
# largest fraction of random prompt rows at which the reference may predict the token it was just fed (~0 for a model
# that uses its context)
MAX_COPY = 0.1


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


# ----------------------------------------------------------------------------------------------------------
# Teacher-forced checker
# ----------------------------------------------------------------------------------------------------------
def teacher_forced_check(forward, requests, outs, tau=TAU, max_copy=MAX_COPY, transform=None):
    """Check every generated token against `forward(ids 1-D) -> logits [len(ids), V]` of its request's prompt + output.

    For request (prompt, max_length) with output o: len(o) == max_length, and at every position t the logit of o[t] in the
    row that predicts it is within tau * max|row| of that row's maximum.  `transform(r, rows, prompt, out) -> rows`, if given,
    maps request r's fp64 rows [max_length, V] (row t predicts o[t]) before the check, e.g. to apply the penalties of each
    position's history; it may set banned entries to -inf, and max|row| is taken over the finite entries.  The reference must depend on the context, not only
    on the row's own input token: over the (random) prompt rows its arg-max may be that input token at no more than max_copy
    of the rows.  A model that copies its input predicts the same output from any context, so no attention or cache error
    could move its tokens.  (Generated rows are not counted: a model's own output may repeat itself legitimately.)
    Returns (worst gap / (tau * max|row|), fraction of generated positions whose top-1 / top-2 margin exceeds
    tau * max|row|, fraction of prompt rows whose arg-max is their input token, number of generated positions)."""
    worst, decisive, copies, prompt_rows, total = 0.0, 0, 0, 0, 0
    for r, ((prompt, max_len), out) in enumerate(zip(requests, outs)):
        prompt = torch.as_tensor(prompt).reshape(-1).to(torch.int64).cpu()
        out = torch.as_tensor(out).reshape(-1).to(torch.int64).cpu()
        assert out.numel() == max_len, f"request {r}: {out.numel()} tokens, max_length {max_len}"
        p = prompt.numel()
        full = forward(torch.cat([prompt, out])).double().cpu()
        copies += int((full[:p].argmax(-1) == prompt).sum())
        prompt_rows += p
        lg = full[p - 1:p - 1 + max_len]
        if transform is not None:
            lg = transform(r, lg, prompt, out)
        scale = lg.masked_fill(~torch.isfinite(lg), 0.0).abs().amax(-1)
        top2 = lg.topk(2, dim=-1).values
        gap = (top2[:, 0] - lg.gather(1, out[:, None])[:, 0]) / (tau * scale)
        bad = ~(gap <= 1.0)                                   # NaN fails
        if bool(bad.any()):
            t = int(bad.nonzero()[0])
            raise AssertionError(f"request {r}: token {int(out[t])} at position {t} is {gap[t].item():.2f} x tau below the "
                                 f"reference maximum (reference arg-max {int(lg[t].argmax())})")
        worst = max(worst, gap.max().item())
        decisive += int(((top2[:, 0] - top2[:, 1]) > tau * scale).sum())
        total += max_len
    copy = copies / max(prompt_rows, 1)
    assert copy <= max_copy, f"the reference arg-max is the row's own input token at {copy:.0%} of the prompt rows"
    return worst, decisive / max(total, 1), copy, total


def _tiny_oracle():
    cfg = R.RefConfig(vocab_size=512, hidden_size=128, intermediate_size=344, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=1, rope_theta=10000.0, model_type="llama", max_position_embeddings=128,
                      rms_norm_eps=1e-5)
    w = R.init_weights(cfg, seed=9)
    w = {k: (v * 4).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    g = torch.Generator().manual_seed(5)
    reqs = [(torch.randint(1, cfg.vocab_size, (p,), generator=g), m) for p, m in [(7, 12), (3, 12), (11, 9), (1, 10)]]
    outs = [G.greedy_generate(ids[None], w, cfg, max_new=m)[0][0] for ids, m in reqs]
    return reqs, outs, lambda ids: R.model_forward(ids[None], w, cfg)[0]


def test_checker_accepts_the_oracle_greedy_output():
    reqs, outs, fwd = _tiny_oracle()
    worst, frac, copy, n = teacher_forced_check(fwd, reqs, outs)
    assert worst == 0.0 and n == sum(m for _, m in reqs)
    assert frac >= 0.5 and copy <= MAX_COPY, (frac, copy)


def test_checker_rejects_a_model_that_copies_its_input():
    """A reference whose arg-max is the row's own input token accepts the same output from any context (the greedy output
    repeats the last prompt token), so it cannot check attention or the cache."""
    reqs, _, _ = _tiny_oracle()

    def copy_forward(ids):
        return 8.0 * torch.nn.functional.one_hot(ids, 512).double() + 0.01 * torch.randn(ids.numel(), 512, dtype=torch.float64)
    outs = [ids[-1:].repeat(m) for ids, m in reqs]
    with pytest.raises(AssertionError, match="own input token at 100%"):
        teacher_forced_check(copy_forward, reqs, outs)


def test_checker_rejects_a_shifted_output():
    reqs, outs, fwd = _tiny_oracle()
    bad = list(outs)
    bad[0] = torch.cat([outs[0][1:], outs[0][-1:]])           # every token one position early
    with pytest.raises(AssertionError, match="request 0: .* below"):
        teacher_forced_check(fwd, reqs, bad)


def test_checker_rejects_one_replaced_token():
    reqs, outs, fwd = _tiny_oracle()
    r = 2
    lg = fwd(torch.cat([reqs[r][0], outs[r]]))[reqs[r][0].numel() - 1:].double()
    top2 = lg.topk(2, dim=-1)
    margin = (top2.values[:, 0] - top2.values[:, 1]) / lg.abs().amax(-1)
    t = int(margin[:-1].argmax())                              # the most decisive position; the runner-up replaces the top-1
    assert margin[t] > TAU
    bad = list(outs)
    bad[r] = outs[r].clone()
    bad[r][t] = int(top2.indices[t, 1])
    with pytest.raises(AssertionError, match=f"request {r}: .* position {t} "):
        teacher_forced_check(fwd, reqs, bad)


def test_checker_rejects_swapped_outputs():
    reqs, outs, fwd = _tiny_oracle()
    assert reqs[0][1] == reqs[1][1]                            # same length: only the content tells them apart
    with pytest.raises(AssertionError, match="request 0: .* below"):
        teacher_forced_check(fwd, reqs, [outs[1], outs[0]] + outs[2:])


def test_checker_rejects_a_truncated_output():
    reqs, outs, fwd = _tiny_oracle()
    with pytest.raises(AssertionError, match="request 3: 9 tokens, max_length 10"):
        teacher_forced_check(fwd, reqs, outs[:3] + [outs[3][:-1]])


# ----------------------------------------------------------------------------------------------------------
# 1. step bookkeeping, bit-exact, across warps
# ----------------------------------------------------------------------------------------------------------
DIM = 64          # width of the rebuild_padding operand
P_EOS = 0.005


def _upload(st):
    return {k: torch.from_numpy(v.copy()).to(DEV) for k, v in st.items()}


def _device_step(d, header, T, topk, tmp, width, bs, max_prompt, max_seq):
    """One continuous_generate step on the device state `d` (header: pinned; T: its token_num): get_padding_offset and
    rebuild_padding, the bookkeeping after the model, step_paddle and retire_admit.  Returns the op outputs to compare."""
    o = ops()
    res = {}
    if T > 0:
        this, enc, dec = d["seq_lens_this_time"], d["seq_lens_encoder"], d["seq_lens_decoder"]
        cum = torch.cumsum(width - this, 0, dtype=torch.int32)
        res["padding"] = o.get_padding_offset(d["input_ids"], cum, T, this)
        res["rebuild"] = o.rebuild_padding(tmp, res["padding"][1], dec, enc, width)
        o.set_value_by_flags_and_idx_v2(d["pre_ids"], d["input_ids"], this, enc, dec, d["step_idx"], d["stop_flags"])
        tk = torch.from_numpy(topk).to(DEV)
        d["step_idx"].add_((~d["stop_flags"]).to(torch.int64))
        o.set_stop_value_multi_ends(tk, d["stop_flags"], torch.tensor([sim.EOS], device=DEV), seq_lens=this,
                                    next_tokens=d["next_tokens"])
        torch.logical_or(d["stop_flags"], d["step_idx"] >= d["max_dec_len"], out=d["stop_flags"])
        res["not_need_stop"] = torch.zeros(1, dtype=torch.bool, device=DEV)
        stop_nums = torch.full((1,), this.numel(), dtype=torch.int64, device=DEV)
        o.update_inputs(d["stop_flags"], res["not_need_stop"], this, enc, dec, d["input_ids"], stop_nums, d["next_tokens"],
                        d["is_block_step"])
    o.step_paddle(*[d[k] for k in sim.STEP_ORDER], block_size=bs)
    o.retire_admit(d, header, bs, max_prompt, max_seq)
    return res


def _compare(what, d, header, res, st, hdr, want):
    for k in st:
        got = d[k].cpu().numpy()
        if not np.array_equal(got, st[k]):
            bad = np.argwhere(got != st[k])[:4].tolist()
            raise AssertionError(f"{what}: field {k} differs at {bad}")
    assert np.array_equal(header.numpy()[:RA.HEADER_INTS], hdr), (what, header.numpy(), hdr)
    for k, v in want.items():
        got = res[k]
        if k == "padding":
            for name, a, b in zip(("x_remove_padding", "cum_offsets_out", "padding_offset", "cu_seqlens_q", "cu_seqlens_k"),
                                  got, v):
                assert np.array_equal(a.cpu().numpy(), b), f"{what}: get_padding_offset {name} differs"
        elif k == "rebuild":
            assert np.array_equal(got.view(torch.int16).cpu().numpy(), v), f"{what}: rebuild_padding differs"
        else:
            assert bool(got.cpu()[0]) == bool(v[0]), f"{what}: not_need_stop {bool(got.cpu()[0])}, restatement {bool(v[0])}"


def run_queue(bsz, bs, num_blocks, seed, one_token_wave=False, max_steps=2000):
    """Drain a queue of 3 * bsz + 5 requests (prompts of up to 2.5 pages, half of them ending 0 .. 3 rows before a page
    boundary so that their first tokens grow into a decoder block; outputs of 1 .. 2.5 pages, EOS with p = P_EOS; with
    one_token_wave the first bsz requests ask for one token, so that they all retire in one call)
    through the restatements and through the CUDA ops twice: on a device-resident state and on a copy of
    the host state taken before every step; after every step every field, the header, the op outputs and the block
    ownership must agree.  Returns the events the run went through."""
    def prompt_lens(rng, n):
        free = rng.randint(1, 5 * bs // 2 + 1, size=n)
        page_end = rng.randint(1, 3, size=n) * bs - rng.randint(0, 4, size=n)
        return np.where(rng.rand(n) < 0.5, free, page_end)

    st, rng, nb, _ = sim.make_queue_state(seed, bsz=bsz, block_size=bs, num_requests=3 * bsz + 5, max_dec=5 * bs // 2,
                                          num_blocks=num_blocks, prompt_lens=prompt_lens)
    if one_token_wave:
        st["req_max_dec_len"][:bsz] = 1
    plens = np.diff(st["prompt_offsets"])
    max_prompt, max_seq = int(plens.max()), int((plens + st["req_max_dec_len"]).max())
    width = st["input_ids"].shape[1]
    header = sim.new_header()
    ev = dict(admitted=0, retired=0, parked_hi=-1, recovered_hi=-1, last_slot=False, preemptions=0, steps=0)
    dev = _upload(st)
    hdev = torch.zeros(RA.HEADER_INTS, dtype=torch.int32).pin_memory()
    ops().retire_admit(dev, hdev, bs, max_prompt, max_seq)
    RA.retire_admit(st, header, bs)
    torch.cuda.synchronize()
    _compare(f"bsz {bsz} block {bs} pool {nb} first admission", dev, hdev, {}, st, header, {})
    emitted = {}
    while True:
        sim.check_blocks(st, nb)
        ev["admitted"] = max(ev["admitted"], int(header[RA.ADMITTED]))
        ev["retired"] = max(ev["retired"], int(header[RA.RETIRED]))
        ev["last_slot"] |= bool(st["slot_request"][-1] >= 0)
        if header[RA.DONE]:
            break
        ev["steps"] += 1
        assert ev["steps"] < max_steps
        T = int(header[RA.TOKEN_NUM])
        topk = tmp_bits = None
        want = {}
        if T > 0:
            topk = sim.draw_tokens(rng, bsz, p_eos=P_EOS)
            tmp_bits = rng.randint(-2 ** 15, 2 ** 15, size=(T, DIM)).astype(np.int16)
            tmp_bits[(tmp_bits & 0x7F80) == 0x7F80] = 0               # no NaN / inf bit patterns
            cum = np.cumsum(width - st["seq_lens_this_time"]).astype(np.int32)
            want["padding"] = G.get_padding_offset_v2(st["input_ids"], cum, T, st["seq_lens_this_time"])
            want["rebuild"] = G.rebuild_padding_v2(tmp_bits, want["padding"][1], st["seq_lens_decoder"],
                                                   st["seq_lens_encoder"], width)
        fresh, hfresh = _upload(st), torch.from_numpy(header.copy()).pin_memory()
        tmp = torch.from_numpy(tmp_bits).to(DEV).view(BF16) if T > 0 else None
        outs = [_device_step(x, h, T, topk, tmp, width, bs, max_prompt, max_seq) for x, h in ((dev, hdev), (fresh, hfresh))]
        parked_before = st["is_block_step"].copy()
        if T > 0:
            want["not_need_stop"] = sim.apply_tokens(st, topk, emitted)
        G.step_paddle(st, bs)
        newly = np.nonzero(st["is_block_step"] & ~parked_before)[0]
        back = np.nonzero(~st["is_block_step"] & parked_before)[0]
        ev["parked_hi"] = max([ev["parked_hi"]] + newly.tolist())
        ev["recovered_hi"] = max([ev["recovered_hi"]] + back.tolist())
        RA.retire_admit(st, header, bs)
        torch.cuda.synchronize()
        for (x, h), res, mode in zip(((dev, hdev), (fresh, hfresh)), outs, ("resident", "per-call")):
            _compare(f"bsz {bsz} block {bs} pool {nb} step {ev['steps']} ({mode})", x, h, res, st, header, want)
    ev["preemptions"] = int(header[RA.PREEMPTIONS])
    assert (st["out_lens"] > 0).all() and (st["out_lens"] <= st["req_max_dec_len"]).all()
    return ev


# (slots, block size) -> (tight pool, roomy pool) in pages.  The tight pools pre-empt; at 128-row pages the outputs are too
# short to outgrow a page twice within the reserve retire_admit keeps, so that case runs the roomy pool only.
STEP_CASES = {(33, 32): (45, 400), (256, 64): (500, 3000), (1000, 64): (2000, 6000), (1024, 32): (1400, 8000),
              (1024, 128): (None, 8000)}


@pytest.mark.gpu
@pytest.mark.parametrize("bsz,bs", list(STEP_CASES))
def test_step_kernels_match_restatement_across_warps(bsz, bs):
    """Whole queues through the step kernels, bit-exact after every step; the roomy run admits bsz requests at once and
    retires them together one step later, the tight run pre-empts and recovers."""
    tight, roomy = STEP_CASES[bsz, bs]
    evs = [run_queue(bsz, bs, roomy, seed=bsz + bs, one_token_wave=True)]
    if tight is not None:
        evs.append(run_queue(bsz, bs, tight, seed=bsz + bs + 1))
    print(f"[step bookkeeping bsz {bsz} block {bs}] " + "; ".join(str(e) for e in evs))
    assert evs[0]["admitted"] > 32 and evs[0]["retired"] > 32 and evs[0]["last_slot"], evs[0]
    if tight is not None:
        assert evs[1]["preemptions"] > 0, evs[1]
        if bsz >= 256:
            assert evs[1]["parked_hi"] >= 32 and evs[1]["recovered_hi"] >= 32, evs[1]


def _dry_pool(used):
    """bsz = len(used) running slots, each with one encoder block and used[b] decoder blocks, the pool dry, and slot 5
    asking for one more block (its next token starts a page)."""
    bsz, bs, bnps = len(used), 16, 8
    st, _ = step_sim.make_state(bsz=bsz, block_size=bs, block_num_per_seq=bnps, length=bnps * bs,
                                               num_blocks=int(sum(used)) + bsz, max_dec=4)
    nxt = 0
    st["block_tables"][:] = -1
    for b in range(bsz):
        n = 1 + int(used[b])
        st["block_tables"][b, :n] = np.arange(nxt, nxt + n)
        nxt += n
        st["seq_lens_decoder"][b] = n * bs - 1
    st["seq_lens_decoder"][5] = (1 + int(used[5])) * bs
    st["encoder_block_lens"][:] = 1
    st["used_list_len"][:] = used
    st["seq_lens_encoder"][:] = 0
    st["seq_lens_this_time"][:] = 1
    st["step_idx"][:] = 2
    st["free_list"][:] = -1
    st["free_list_len"][0] = 0
    return st, bs


@pytest.mark.gpu
@pytest.mark.parametrize("holders,victim", [((40, 700), 40), ((1000,), 1000)])
def test_step_paddle_preempts_the_largest_holder_at_1024_slots(holders, victim):
    """A dry pool at 1 024 slots: the largest decoder-block holder is parked, the lowest index among equals (slots in
    different warps meet only in the second stage of the arg-max)."""
    used = np.ones(1024, np.int32)
    used[list(holders)] = 3
    st, bs = _dry_pool(used)
    d = _upload(st)
    ops().step_paddle(*[d[k] for k in sim.STEP_ORDER], block_size=bs)
    G.step_paddle(st, bs)
    torch.cuda.synchronize()
    for k in sim.STEP_ORDER:
        assert np.array_equal(d[k].cpu().numpy(), st[k]), k
    assert np.nonzero(st["is_block_step"])[0].tolist() == [victim]
    assert st["block_tables"][5, 2] >= 0


# ----------------------------------------------------------------------------------------------------------
# 2. append_attention over one serving-shaped step
# ----------------------------------------------------------------------------------------------------------
PROMPTS = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 512]
CHUNK = (150, 100)          # a prompt chunk of 100 rows on a 150-row cached prefix
IDLE_MID = (17, 18, 100, 201)


def _serving_layout(bs, seed=0):
    """Per slot of a 256-slot step: (kind, cached rows, new rows, rows the slot held in the step before)."""
    B = 256
    rng = np.random.RandomState(seed)
    idle = set(IDLE_MID) | {B - 2, B - 1}
    free = [b for b in range(B) if b not in idle]
    special = rng.choice(free, size=len(PROMPTS) + 1, replace=False).tolist()
    rest = [b for b in free if b not in special]
    # decode: cached lengths spread over 1 .. 2047 (attended rows 2 .. 2048), with page multiples and page multiples - 1
    dec = np.linspace(1, 2047, len(rest)).round().astype(int)
    edges = [bs, 2 * bs, 4 * bs - 1, 8 * bs, 2048 - bs, 2047, 128, 511, 1024]
    dec[rng.choice(len(rest), size=len(edges), replace=False)] = edges
    lay = {}
    for b, n in zip(rest, dec):
        lay[b] = ("decode", int(n), 1, int(n))                     # the step before appended row n - 1
    for b, p in zip(special[:-1], PROMPTS):
        lay[b] = ("prompt", 0, p, int(rng.randint(1, 600)))         # admitted into a slot whose request retired
    lay[special[-1]] = ("chunk", CHUNK[0], CHUNK[1], CHUNK[0])
    for b in idle:
        lay[b] = ("idle", int(rng.randint(1, 900)), 0, int(rng.randint(1, 900)))   # stale decode length, retired
    return [lay[b] for b in range(B)]


def _serving_case(nh, kvh, d, bs, seed):
    """Build the pool, run the step before (which the retiring slots still decode in), retire: NaN into their pages and
    hand those to the admitted prompts.  Returns everything the checked call needs."""
    o = ops()
    lay = _serving_layout(bs, seed)
    B = len(lay)
    mb = 2048 // bs + 1
    g = torch.Generator(device=DEV).manual_seed(seed)
    # pages each slot holds in the step before: what its checked row(s) need, or (a retiring slot) its old request's
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
    kc = torch.full((nb, kvh, bs, d), float("nan"), dtype=BF16, device=DEV)
    vc = torch.full((nb, kvh, bs, d), float("nan"), dtype=BF16, device=DEV)
    cos, sin = o.rope_tables(d, 4096, 10000.0, DEV)
    ld = (nh + 2 * kvh) * d

    def fill(b, rows):                     # random history rows 0 .. rows-1 of slot b
        for j in range(math.ceil(rows / bs)):
            n = min(bs, rows - j * bs)
            p = int(tables[b, j])
            kc[p, :, :n] = torch.randn(kvh, n, d, generator=g, device=DEV).to(BF16)
            vc[p, :, :n] = torch.randn(kvh, n, d, generator=g, device=DEV).to(BF16)

    def call(chunks, tbl, splits, qkv=None):
        """chunks: per slot (kind, cached, new): decode rows have enc 0, prompt rows enc = new; idle slots keep cached."""
        n = [c[2] for c in chunks]
        enc = torch.tensor([x if k in ("prompt", "chunk") else 0 for k, _, x in chunks], dtype=torch.int32, device=DEV)
        dec = torch.tensor([c[1] for c in chunks], dtype=torch.int32, device=DEV)
        this = torch.tensor(n, dtype=torch.int32, device=DEV)
        cu = torch.tensor([0] + np.cumsum(n).tolist(), dtype=torch.int32, device=DEV)
        if qkv is None:
            qkv = torch.randn(sum(n), ld, generator=g, device=DEV).to(BF16)
        out = torch.full((sum(n), nh * d), float("nan"), dtype=BF16, device=DEV)
        o.append_attention(qkv, kc, vc, enc, dec, this, cu, tbl.to(DEV), cos, sin, nh, max_q_len=max(n), out=out,
                           num_splits=splits)
        return qkv, out, cu.tolist()

    # the step before: decode slots append row (cached - 1), the chunk slot runs its prefix as a prompt, the slots whose
    # request retires after it (prompt slots of the checked step, idle slots) decode their last row
    prev = []
    for k, c, n, h in lay:
        if k == "chunk":
            prev.append(("prompt", 0, h))
        else:
            fill(len(prev), h - 1)
            prev.append(("decode", h - 1, 1))
    call(prev, tables, splits=7)
    # retire: NaN into the retired slots' pages, which the admitted prompts take first
    recycled = []
    for b, (k, c, n, h) in enumerate(lay):
        if k in ("prompt", "idle"):
            pages = [int(x) for x in tables[b] if x >= 0]
            kc[pages] = float("nan")
            vc[pages] = float("nan")
            recycled += pages
            tables[b] = -1
    pool = recycled + unused
    for b, (k, c, n, h) in enumerate(lay):
        if k == "prompt":
            tables[b, :new_pages[b]] = torch.tensor(pool[:new_pages[b]], dtype=torch.int32)
            pool = pool[new_pages[b]:]
    assert len(recycled) > sum(new_pages) // 2
    chunks = [(k, c, n) for k, c, n, _ in lay]
    qkv = torch.randn(sum(n for _, _, n in chunks), ld, generator=g, device=DEV).to(BF16)
    return chunks, tables, kc, vc, call, qkv


APPEND_CASES = [(64, 32, 8, 32), (64, 32, 8, 64), (64, 32, 8, 128), (64, 14, 2, 32), (64, 14, 2, 64), (64, 14, 2, 128),
                (128, 24, 8, 64), (128, 12, 2, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("d,nh,kvh,bs", APPEND_CASES)
def test_append_attention_serving_step(d, nh, kvh, bs):
    """One 256-slot step per (row, head) against fp64, auto and 7 splits; no row past a sequence's length, no page outside
    its table and no idle slot is read or written."""
    chunks, tables, kc, vc, call, qkv0 = _serving_case(nh, kvh, d, bs, seed=d + nh + bs)
    tdev = tables.to(DEV).long()
    # what the step may touch: rows below every sequence's length in its own pages
    live = torch.zeros(kc.shape[0], bs, dtype=torch.bool)
    for b, (k, cached, n) in enumerate(chunks):
        T = cached + n if k != "idle" else 0
        for j in range(math.ceil(T / bs)):
            live[int(tables[b, j]), :min(bs, T - j * bs)] = True
    live = live.to(DEV)[:, None, :, None]
    for splits in (0, 7):
        qkv, out, cu = call(chunks, tables, splits, qkv0.clone())     # RoPE rotates qkv in place
        torch.cuda.synchronize()
        seq = {}

        def seq_rows(b):
            if b not in seq:
                T = chunks[b][1] + chunks[b][2]
                pages = tdev[b, :math.ceil(T / bs)]
                seq[b] = (kc[pages].transpose(0, 1).reshape(kvh, -1, d), vc[pages].transpose(0, 1).reshape(kvh, -1, d))
            return seq[b]

        checked = 0
        for kind, c, tol in (("decode", DECODE_C, DECODE_HEAD_TOL), ("prompt", PREFILL_C, PREFILL_HEAD_TOL)):
            idx, where = [], []
            for b, (k, cached, n) in enumerate(chunks):
                if k != "idle" and (k == "decode") == (kind == "decode"):
                    for i in range(n):
                        idx.append(cu[b] + i)
                        where.append((b, cached + i))

            def rows(m):
                b, pos = where[m]
                K, V = seq_rows(b)
                return K[:, :pos + 1], V[:, :pos + 1]
            sel = torch.tensor(idx, device=DEV)
            assert_attention_close(out[sel], qkv[sel, :nh * d].reshape(len(idx), nh, d), rows, c=c, head_tol=tol,
                                   what=f"serving step {kind} rows d={d} nh={nh} kvh={kvh} block_size={bs} splits={splits}")
            checked += len(idx)
        assert checked == out.shape[0]
        # nothing was written outside the sequences: rows past every length and every page outside the tables (the
        # retired slots' recycled pages among them) still hold NaN, and no row the step attends to does
        for cache in (kc, vc):
            assert bool((torch.isnan(cache) == ~live).all())


# ----------------------------------------------------------------------------------------------------------
# 3. continuous_generate at preset widths against the training-path forward
# ----------------------------------------------------------------------------------------------------------
GEN_WIDTHS = {
    "llama3_2_1b": dict(model_type="llama", tied=True, hidden_size=2048, intermediate_size=8192, num_attention_heads=32,
                        num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, block_size=64, max_batch_size=192,
                        num_requests=400, num_blocks=600),
    "qwen2_1_5b": dict(model_type="qwen2", tied=False, hidden_size=1536, intermediate_size=8960, num_attention_heads=12,
                       num_key_value_heads=2, rms_norm_eps=1e-6, rope_theta=1000000.0, block_size=32, max_batch_size=64,
                       num_requests=240, num_blocks=420),
}


def _gen_requests(n, vocab, seed=7):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, vocab, (int(torch.randint(1, 301, (1,), generator=g)),), generator=g),
             int(torch.randint(1, 161, (1,), generator=g))) for _ in range(n)]


def _poisoned(real):
    """append_attention that first fills NaN into every page of the layer's cache no block table references and every
    referenced row at or past its slot's seq_lens_decoder + seq_lens_this_time (no host sync, no boolean indexing: the
    wrapper is captured into the decode graphs with the call)."""

    def wrapper(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q,
                block_tables, cos, sin, nh, max_q_len, **kw):
        nb, _, bs, _ = key_cache.shape
        B, mb = block_tables.shape
        held = block_tables >= 0
        page = torch.where(held, block_tables, nb).long()                            # -1 -> a dummy page nb
        limit = (seq_lens_decoder + seq_lens_this_time).long()
        pos = torch.arange(mb * bs, device=qkv.device).view(1, mb, bs)
        stale = (pos >= limit.view(B, 1, 1)).view(B * mb, bs)
        rows = torch.ones(nb + 1, bs, dtype=torch.bool, device=qkv.device)
        rows.scatter_(0, page.view(-1, 1).expand(-1, bs), stale)                     # referenced pages: their stale rows
        ref = torch.zeros(nb + 1, dtype=torch.int32, device=qkv.device)
        ref.index_add_(0, page.view(-1), held.view(-1).to(torch.int32))
        rows.masked_fill_((ref == 0).view(-1, 1), True)                              # unreferenced pages: every row
        mask = rows[:nb].view(nb, 1, bs, 1)
        key_cache.masked_fill_(mask, float("nan"))
        value_cache.masked_fill_(mask, float("nan"))
        return real(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q,
                    block_tables, cos, sin, nh, max_q_len, **kw)
    return wrapper


@pytest.mark.gpu
@pytest.mark.parametrize("width", list(GEN_WIDTHS))
def test_continuous_generate_matches_training_forward(width, monkeypatch):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200 import ops as O
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    spec = dict(GEN_WIDTHS[width])
    model_type, tied = spec.pop("model_type"), spec.pop("tied")
    bs, B, n_req, nb = (spec.pop(k) for k in ("block_size", "max_batch_size", "num_requests", "num_blocks"))
    kw = dict(vocab_size=4096, num_hidden_layers=2, max_position_embeddings=512, **spec)
    cfg = R.RefConfig(qkv_bias=model_type == "qwen2", model_type=model_type, **kw)
    w = R.init_weights(cfg, seed=41)
    # the tied embedding stays as initialised: scaled up it would dominate the residual stream too, and the model would
    # predict its own input token whatever the context (teacher_forced_check refuses such a reference)
    if tied:
        w.pop("lm_head.weight")
    else:
        w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(BF16).float()
    C = T.Qwen2Config if model_type == "qwen2" else T.LlamaConfig
    M = T.Qwen2ForCausalLM if model_type == "qwen2" else T.LlamaForCausalLM
    train = M(C(tie_word_embeddings=tied, **kw))
    train.set_state_dict(w)
    inf = LlamaForCausalLMInferenceModel(C(tie_word_embeddings=tied, **kw), block_attn=True, append_attn=True, block_size=bs)
    inf.set_state_dict(w)
    del w
    reqs = _gen_requests(n_req, cfg.vocab_size)
    monkeypatch.setattr(O, "append_attention", _poisoned(O.append_attention))

    steps = []
    real_fp = inf._forward_packed

    def recording(ids, caches, block_tables, enc, dec, this_time, cu, cum, max_q_len, max_len):
        n_dec = int(((this_time == 1) & (enc == 0)).sum())
        steps.append((int(ids.numel()), int(max_q_len), n_dec))
        return real_fp(ids, caches, block_tables, enc, dec, this_time, cu, cum, max_q_len, max_len)

    t0 = time.perf_counter()
    monkeypatch.setattr(inf, "_forward_packed", recording)
    eager, st_e = inf.continuous_generate(reqs, max_batch_size=B, num_blocks=nb, use_cuda_graph=False)
    monkeypatch.setattr(inf, "_forward_packed", real_fp)
    outs, st_g = inf.continuous_generate(reqs, max_batch_size=B, num_blocks=nb)
    t1 = time.perf_counter()
    print(f"[{width}] stats {st_g}; two runs {t1 - t0:.1f} s")
    assert {k: v for k, v in st_e.items() if k != "decode_step_ms"} == {k: v for k, v in st_g.items() if k != "decode_step_ms"}
    assert st_g["free_blocks_at_exit"] == nb and bool((inf.last_block_tables == -1).all())
    assert st_g["preemptions"] > 0 and st_g["recoveries"] > 0, st_g
    decode_rows = [t for t, q, _ in steps if q == 1]
    assert min(decode_rows) <= 128
    if B > 128:
        assert max(decode_rows) > 128, max(decode_rows)
    assert any(q > 1 and n_dec > 0 and t > n_dec for t, q, n_dec in steps)

    def fwd(ids):
        return train.engine.forward_logits(ids.to(DEV)[None])[0].float()
    # the split-K GEMMs reduce their K-range partials in arrival order, so two runs may round a logit differently and part
    # at a near-tie; up to there the graph run equals the eager run token for token, and both pass the check in full
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
          f"{frac:.3f}, reference arg-max = input token at {copy:.3f}; {parted} requests part from the eager run at a near-tie; {len(steps)} steps, decode-only rows "
          f"{min(decode_rows)} .. {max(decode_rows)}; check {time.perf_counter() - t1:.1f} s")
    assert frac >= 0.5, frac
