"""A continuous-batching simulation: a request queue drained through step_paddle + retire_admit (oracle or CUDA ops), with a
random-token stand-in for the model and the reference's bookkeeping between two calls (set_value_by_flags_and_idx_v2,
step_idx / length stop, set_stop_value_multi_ends v2, update_inputs).  Shared by the CPU invariant test of the restatement
and the GPU bit-exactness test of the kernel."""
import numpy as np

from oracle import generation_ref as G
from oracle import retire_admit_ref as RA

EOS = 2
# argument order of ops.step_paddle (tests/step_sim.py ORDER)
STEP_ORDER = ("stop_flags", "seq_lens_this_time", "ori_seq_lens_encoder", "seq_lens_encoder", "seq_lens_decoder", "block_tables",
              "encoder_block_lens", "is_block_step", "step_block_list", "step_lens", "recover_block_list", "recover_lens",
              "need_block_list", "need_block_len", "used_list_len", "free_list", "free_list_len", "input_ids", "pre_ids",
              "step_idx", "next_tokens")


def make_queue_state(seed, bsz=6, block_size=4, num_requests=24, max_prompt=12, max_dec=24, spare_blocks=3, num_blocks=None,
                     prompt_lens=None):
    """Empty slots, a free list of every block, and a queue of `num_requests` requests (prompt lengths U{1..max_prompt}, or
    `prompt_lens(rng, num_requests)`); the pool is `spare_blocks` above the largest single request's pages (or `num_blocks`,
    if given and larger), so that pre-emption and recovery happen."""
    rng = np.random.RandomState(seed)
    plens = rng.randint(1, max_prompt + 1, size=num_requests) if prompt_lens is None else prompt_lens(rng, num_requests)
    decs = rng.randint(1, max_dec + 1, size=num_requests)
    need = int(max((p + d + block_size - 1) // block_size for p, d in zip(plens, decs)))
    num_blocks = max(need + spare_blocks, num_blocks or 0)
    bnps = need + 1                                   # one spare column: step_paddle recovers with used + 1 blocks
    length = bnps * block_size
    prompts = [rng.randint(5, 1000, size=int(p)).astype(np.int64) for p in plens]
    st = {
        "stop_flags": np.ones(bsz, bool), "is_block_step": np.zeros(bsz, bool),
        "seq_lens_this_time": np.zeros(bsz, np.int32), "ori_seq_lens_encoder": np.zeros(bsz, np.int32),
        "seq_lens_encoder": np.zeros(bsz, np.int32), "seq_lens_decoder": np.zeros(bsz, np.int32),
        "block_tables": np.full((bsz, bnps), -1, np.int32), "encoder_block_lens": np.zeros(bsz, np.int32),
        "step_block_list": np.full(bsz, -1, np.int32), "step_lens": np.zeros(1, np.int32),
        "recover_block_list": np.full(bsz, -1, np.int32), "recover_lens": np.zeros(1, np.int32),
        "need_block_list": np.full(bsz, -1, np.int32), "need_block_len": np.zeros(1, np.int32),
        "used_list_len": np.zeros(bsz, np.int32), "free_list": np.arange(num_blocks, dtype=np.int32),
        "free_list_len": np.array([num_blocks], np.int32), "input_ids": np.zeros((bsz, length), np.int64),
        "pre_ids": np.full((bsz, max_dec + 1), -1, np.int64), "step_idx": np.zeros(bsz, np.int64),
        "next_tokens": np.full(bsz, -1, np.int64), "max_dec_len": np.zeros(bsz, np.int64), "min_dec_len": np.zeros(bsz, np.int64),
        "slot_request": np.full(bsz, -1, np.int32),
        "prompt_ids": np.concatenate(prompts), "prompt_offsets": np.concatenate([[0], np.cumsum(plens)]).astype(np.int32),
        "req_max_dec_len": decs.astype(np.int64), "req_min_dec_len": np.zeros(num_requests, np.int64),
        "cursor": np.zeros(1, np.int32), "out_ids": np.full((num_requests, max_dec), -1, np.int64),
        "out_lens": np.zeros(num_requests, np.int32),
    }
    return st, rng, num_blocks, prompts


def draw_tokens(rng, bsz, p_eos=0.04):
    """The token each slot 'generates': random, EOS with probability p_eos."""
    topk = rng.randint(5, 1000, size=bsz).astype(np.int64)
    topk[rng.rand(bsz) < p_eos] = EOS
    return topk


def apply_tokens(st, topk, emitted):
    """The reference's bookkeeping of one model step over the running slots, given the tokens they chose (logged in
    emitted[request]), up to update_inputs.  Returns update_inputs' not_need_stop (stop_nums = the slot count)."""
    running = ~st["stop_flags"]
    st["pre_ids"][:] = G.set_value_by_flags_and_idx_v2(st["pre_ids"], st["input_ids"], st["seq_lens_encoder"],
                                                       st["seq_lens_decoder"], st["step_idx"], st["stop_flags"])
    st["step_idx"] += running
    topk, sf, nxt = G.set_stop_value_multi_ends_v2(topk, st["stop_flags"], st["seq_lens_this_time"], np.array([EOS]),
                                                   st["next_tokens"])
    sf |= running & (st["step_idx"] >= st["max_dec_len"])
    st["stop_flags"][:], st["next_tokens"][:] = sf, nxt
    for b in np.nonzero(running)[0]:
        emitted.setdefault(int(st["slot_request"][b]), []).append(int(topk[b]))
    nns, stt, enc, dec, ids = G.update_inputs(st["stop_flags"], st["seq_lens_this_time"], st["seq_lens_encoder"],
                                              st["seq_lens_decoder"], st["input_ids"], np.array([running.shape[0]]),
                                              st["next_tokens"], st["is_block_step"])
    st["seq_lens_this_time"][:], st["seq_lens_encoder"][:], st["seq_lens_decoder"][:], st["input_ids"][:] = stt, enc, dec, ids
    return nns


def model_step(st, rng, emitted, p_eos=0.04):
    """One model step over the running slots: draw_tokens, then apply_tokens."""
    apply_tokens(st, draw_tokens(rng, st["stop_flags"].shape[0], p_eos), emitted)


def check_blocks(st, num_blocks):
    fl = st["free_list"][: int(st["free_list_len"][0])].tolist()
    held = [int(x) for x in st["block_tables"].reshape(-1) if x >= 0]
    assert sorted(fl + held) == list(range(num_blocks)), "every cache block is owned exactly once"


def new_header():
    return np.zeros(RA.HEADER_INTS, np.int32)
