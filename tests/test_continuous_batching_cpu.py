"""The retire_admit restatement (oracle/retire_admit_ref.py) driven with step_paddle's restatement over a request queue and a
tight block pool, and the argument errors of b200_retire_admit, which come back through the library without a device."""
import numpy as np
import pytest
import torch

import continuous_sim as sim
from oracle import generation_ref as G
from oracle import retire_admit_ref as RA


def _drain(seed, bs=4, **kw):
    st, rng, nb, prompts = sim.make_queue_state(seed, block_size=bs, **kw)
    header, emitted, admitted_order = sim.new_header(), {}, []
    RA.retire_admit(st, header, bs)
    admitted_order += [int(r) for r in st["slot_request"] if r >= 0]
    steps = 0
    while not header[RA.DONE]:
        steps += 1
        assert steps < 5000, "the queue must drain"
        sim.model_step(st, rng, emitted)
        G.step_paddle(st, bs, first_token_id=0)
        sim.check_blocks(st, nb)
        empty_before = st["slot_request"] < 0
        # an empty slot holds no block, so admission never overwrites a live table row
        assert (st["block_tables"][empty_before] == -1).all() and (st["encoder_block_lens"][empty_before] == 0).all()
        before = st["slot_request"]
        RA.retire_admit(st, header, bs)
        sim.check_blocks(st, nb)
        # admitted this call (a recovered slot has step_idx > 0), in slot order
        new = [int(st["slot_request"][b]) for b in range(len(before)) if st["step_idx"][b] == 0 and st["seq_lens_encoder"][b] > 0]
        assert len(new) == header[RA.ADMITTED]
        admitted_order += new
        for b in np.nonzero(st["is_block_step"])[0]:                       # a parked slot holds no block
            assert (st["block_tables"][b] == -1).all() and st["encoder_block_lens"][b] == 0
        for b in np.nonzero((st["seq_lens_encoder"] > 0) & (st["step_idx"] > 0))[0]:
            # recovered this step: the row is the prompt + every token generated so far, re-prefilled from position 0
            r = int(st["slot_request"][b])
            want = np.concatenate([prompts[r], emitted[r]])
            assert st["seq_lens_encoder"][b] == want.size and np.array_equal(st["input_ids"][b, :want.size], want), (r, b)
    return st, header, emitted, admitted_order, nb


@pytest.mark.parametrize("seed", range(24))
def test_queue_drains_fifo_with_every_block_owned_once(seed):
    st, header, emitted, order, nb = _drain(seed)
    R = st["req_max_dec_len"].shape[0]
    assert order == list(range(R)), "requests are admitted in queue order"
    for r in range(R):                                                     # every request completed, with its own tokens
        n = int(st["out_lens"][r])
        assert 1 <= n <= st["req_max_dec_len"][r]
        assert st["out_ids"][r, :n].tolist() == emitted[r], r
        assert n == st["req_max_dec_len"][r] or emitted[r][-1] == sim.EOS
    assert int(st["free_list_len"][0]) == nb and header[RA.FREE_BLOCKS] == nb
    assert (st["block_tables"] == -1).all()
    assert header[RA.PREEMPTIONS] == header[RA.RECOVERIES]                 # every parked sequence came back


def test_tight_pools_preempt_and_recover():
    totals = np.zeros(2, int)
    for seed in range(24):
        _, header, _, _, _ = _drain(seed)
        totals += (header[RA.PREEMPTIONS], header[RA.RECOVERIES])
    assert totals[0] > 0 and totals[1] > 0, totals


# ---- argument errors through the C-ABI, with integer stand-ins for device addresses that are never dereferenced ----
pytest_nodev = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a machine without a CUDA device")
ADDR = [(i + 1) << 20 for i in range(27)]


def _args(bsz=8, block_size=64, bnps=4, length=512, max_prompt=100, max_seq=300):
    # bsz, block_size, block_num_per_seq, length, pre_id_length, num_requests, out_stride, max_prompt_len, max_seq_len, stream
    return ADDR + [bsz, block_size, bnps, length, 257, 5, 256, max_prompt, max_seq, None]


@pytest_nodev
@pytest.mark.parametrize("bad,needle", [
    (dict(bsz=1025), "need 0 < bsz <= 1024"),
    (dict(max_prompt=257), "does not fit block_num_per_seq"),
    (dict(length=299), "too narrow for prompt + max length"),
])
def test_retire_admit_argument_errors(bad, needle):
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    rc = lib.b200_retire_admit(*_args(**bad))
    msg = lib.b200_last_error().decode()
    assert rc < 0, (rc, msg)
    assert msg.startswith("retire_admit:") and needle in msg, msg
