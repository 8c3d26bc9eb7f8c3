"""CPU oracle of the generation path (TEST INFRASTRUCTURE ONLY — see oracle/llama_ref.py header).

  * bookkeeping ops restated in numpy from the reference's CUDA kernels (file:line beside each function); pinned
    against the known-answer vectors of the reference's own op tests (csrc/xpu/test/python/test_*.py), committed as
    tests/golden/bookkeeping.json by oracle/make_bookkeeping_golden.py.
  * greedy generation restated as "run the (uncached) oracle forward on the growing sequence and take the argmax" —
    the definition KV-cache decoding must agree with (tests/transformers/llama/test_modeling.py:171-219 cache
    consistency, atol 1e-3).  The fused-inference numerics themselves are unpinned in the reference (every
    dygraph-vs-fused comparison in tests/llm/test_predictor.py is @skip).
"""
import numpy as np
import torch

from . import llama_ref as R


# csrc/gpu/get_padding_offset_v2.cu:17-53
def get_padding_offset_v2(input_ids, cum_offsets, token_num, seq_lens):
    bsz, max_len = input_ids.shape
    seq_lens = seq_lens.reshape(-1)
    x_remove = np.zeros(int(token_num), np.int64)
    padding_offset = np.zeros(int(token_num), np.int32)
    cum_out = np.zeros(bsz, np.int32)
    cu_q = np.zeros(bsz + 1, np.int32)
    for bi in range(bsz):
        cum_offset = 0 if bi == 0 else int(cum_offsets[bi - 1])
        for i in range(int(seq_lens[bi])):
            padding_offset[bi * max_len - cum_offset + i] = cum_offset
            x_remove[bi * max_len - cum_offset + i] = input_ids[bi, i]   # RemovePaddingV2 gets cum_offsets_out (:80-85)
        cum_out[bi] = cum_offset
        cu_q[bi + 1] = (bi + 1) * max_len - int(cum_offsets[bi])
    return x_remove, cum_out, padding_offset, cu_q, cu_q.copy()


# csrc/gpu/rebuild_padding_v2.cu:18-69
def rebuild_padding_v2(tmp_out, cum_offsets, seq_lens_decoder, seq_lens_encoder, max_len):
    bsz = seq_lens_encoder.reshape(-1).shape[0]
    out = np.zeros((bsz, tmp_out.shape[1]), tmp_out.dtype)
    for bi in range(bsz):
        dec, enc = int(seq_lens_decoder.reshape(-1)[bi]), int(seq_lens_encoder.reshape(-1)[bi])
        if dec == 0 and enc == 0:
            continue
        seq_id = enc - 1 if dec == 0 else 0
        out[bi] = tmp_out[bi * max_len - int(cum_offsets[bi]) + seq_id]
    return out


# csrc/gpu/token_penalty_multi_scores_v2.cu:19-139 (order: min-length EOS mask, repeat penalty + temperature, bad words)
def token_penalty_multi_scores_v2(pre_ids, logits, penalty, frequency, presence, temperatures, bad_tokens, cur_len, min_len,
                                  eos_token_id):
    logits = logits.astype(np.float32).copy()
    bs, length = logits.shape
    for bi in range(bs):
        if cur_len[bi] >= 0 and cur_len[bi] < min_len[bi]:
            for e in eos_token_id:
                logits[bi, int(e)] = np.float32(-1e10)
        times = np.zeros(length, np.int32)
        if cur_len[bi] >= 0:
            for t in pre_ids[bi]:
                if t < 0:
                    break
                times[int(t)] += 1
        a, b, g = np.float32(penalty[bi]), np.float32(frequency[bi]), np.float32(presence[bi])
        for i in range(length):
            v = logits[bi, i]
            if times[i] != 0:
                v = v * a if v < 0 else v / a
                v = np.float32(v - np.float32(times[i]) * b - g)
            logits[bi, i] = np.float32(v / np.float32(1.0 if temperatures is None else temperatures[bi]))
        if bad_tokens is not None:
            for t in bad_tokens:
                if 0 <= t < length:
                    logits[bi, int(t)] = np.float32(-1e10)
    return logits


# csrc/gpu/stop_generation_multi_ends_v2.cu:35-59
def set_stop_value_multi_ends_v2(topk_ids, stop_flags, seq_lens, end_ids, next_tokens):
    topk_ids, stop_flags, next_tokens = topk_ids.copy(), stop_flags.copy(), next_tokens.copy()
    for i in range(topk_ids.shape[0]):
        if stop_flags[i]:
            if seq_lens[i] == 0:
                topk_ids[i] = -1
            else:
                topk_ids[i] = end_ids[0]
                next_tokens[i] = end_ids[0]
        else:
            next_tokens[i] = topk_ids[i]
        if topk_ids[i] in end_ids:
            stop_flags[i] = True
    return topk_ids, stop_flags, next_tokens


# csrc/gpu/stop_generation_multi_ends.cu:45-56 (mode 2)
def set_stop_value_multi_ends(topk_ids, stop_flags, end_ids):
    topk_ids, stop_flags = topk_ids.copy(), stop_flags.copy()
    for i in range(topk_ids.shape[0]):
        if stop_flags[i]:
            topk_ids[i] = end_ids[0]
        if topk_ids[i] in end_ids:
            stop_flags[i] = True
    return topk_ids, stop_flags


# csrc/gpu/set_value_by_flags_v2.cu
def set_value_by_flags_and_idx_v2(pre_ids_all, input_ids, seq_lens_encoder, seq_lens_decoder, step_idx, stop_flags):
    pre = pre_ids_all.copy()
    for i in range(pre.shape[0]):
        if stop_flags[i]:
            continue
        dec, enc = int(seq_lens_decoder[i]), int(seq_lens_encoder[i])
        if dec == 0 and enc == 0:
            continue
        if step_idx[i] >= 0:
            pre[i, int(step_idx[i])] = input_ids[i, enc - 1] if dec == 0 else input_ids[i, 0]
    return pre


# csrc/gpu/set_value_by_flags.cu:17-25
def set_value_by_flags_and_idx(pre_ids_all, pre_ids_now, step_idx, stop_flags):
    pre = pre_ids_all.copy()
    for i in range(pre.shape[0]):
        if not stop_flags[i] and step_idx[i] >= 0:
            pre[i, int(step_idx[i])] = pre_ids_now[i]
    return pre


# csrc/gpu/update_inputs.cu:18-66
def update_inputs(stop_flags, seq_lens_this_time, seq_lens_encoder, seq_lens_decoder, input_ids, stop_nums, next_tokens,
                  is_block_step):
    this_time, enc, dec, ids = seq_lens_this_time.copy(), seq_lens_encoder.copy(), seq_lens_decoder.copy(), input_ids.copy()
    bsz, max_bsz = this_time.shape[0], stop_flags.shape[0]
    stop_sum = 0
    for t in range(max_bsz):
        if t < bsz:
            stop_sum += 0 if is_block_step[t] else int(stop_flags[t])
        else:
            stop_sum += 1
    for t in range(bsz):
        stop = bool(stop_flags[t])
        dec[t] = 0 if stop else (enc[t] if dec[t] == 0 else dec[t] + 1)
        this_time[t] = 0 if stop else 1
        enc[t] = 0
        ids[t, 0] = next_tokens[t]
    return np.array([stop_sum < int(stop_nums[0])]), this_time, enc, dec, ids


def top_p_sampling_reject(probs, top_p, uniform, max_rounds=32):
    """csrc/gpu/sample_kernels/sampling.cuh:286-376 (kernel) and :197-280 (inverse-CDF step), sequential fp32.
    probs [bs, d] fp32, top_p [bs], uniform [max_rounds, bs] -> ids [bs]."""
    probs = np.asarray(probs, np.float32)
    bs, d = probs.shape
    out = np.zeros(bs, np.int64)
    for b in range(bs):
        p = probs[b]
        q, pivot, sid = np.float32(1.0), np.float32(0.0), d - 1
        for r in range(max_rounds):
            u = np.float32(uniform[r, b]) * q
            valid = p > pivot
            cdf = np.cumsum(np.where(valid, p, np.float32(0)), dtype=np.float32)
            hit = np.nonzero((cdf > u) & valid)[0]
            # deviation from :313, whose default sampled_id = d - 1 can be a token of probability 0 when the row's fp32
            # total is at most u: fall back to the largest index with p > pivot (d - 1 only if there is none)
            last = np.nonzero(valid)[0]
            sid = int(hit[0]) if hit.size else (int(last[-1]) if last.size else d - 1)
            pivot = max(pivot, p[sid])
            above = p > pivot
            q = np.float32(p[above].sum(dtype=np.float32))
            if 0 < q < np.float32(top_p[b]):                    # :362
                break
            if above.sum() < 1:                                  # :367 (top_p == 0 -> top-1)
                break
        out[b] = sid
    return out


def greedy_generate(input_ids: torch.Tensor, w, cfg: R.RefConfig, max_new: int, eos=None, mode: str = "bf16",
                    seq_lens=None):
    """Greedy decoding by full re-evaluation (no cache).  input_ids [B, S] right padded; returns [B, max_new] with the
    reference's stop semantics (after EOS a sequence keeps emitting EOS)."""
    B, S = input_ids.shape
    lens = [S] * B if seq_lens is None else [int(x) for x in seq_lens]
    seqs = [input_ids[b, : lens[b]].tolist() for b in range(B)]
    out = torch.full((B, max_new), -1, dtype=torch.int64)
    stopped = [False] * B
    margins = torch.zeros(B, max_new)
    for t in range(max_new):
        for b in range(B):
            if stopped[b]:
                out[b, t] = eos if eos is not None else -1
                continue
            logits = R.model_forward(torch.tensor([seqs[b]]), w, cfg, mode=mode)[0, -1]
            top2 = logits.topk(2).values
            margins[b, t] = (top2[0] - top2[1]) / logits.abs().max()
            tok = int(logits.argmax())
            out[b, t] = tok
            seqs[b].append(tok)
            if eos is not None and tok == eos:
                stopped[b] = True
    return out, margins


def paged_decode_attention(q, key_cache, value_cache, block_tables, seq_lens, scale=None):
    """Decode attention over a block (paged) KV cache, the layout of FusedBlockMultiTransformer / append_attention
    (fused_transformer_layers.py:2192-2354): key/value_cache [num_blocks, kvh, block_size, d], block_tables [B, max_blocks],
    sequence b attends to positions 0..seq_lens[b] (the new token already appended).  q [B, nh, d] -> [B, nh*d], fp32."""
    q = np.asarray(q, np.float32)
    B, nh, d = q.shape
    nb, kvh, bs, _ = key_cache.shape
    rep = nh // kvh
    scale = scale or 1.0 / np.sqrt(d)
    out = np.zeros((B, nh, d), np.float32)
    for b in range(B):
        total = min(int(seq_lens[b]) + 1, block_tables.shape[1] * bs)
        pos = np.arange(total)
        phys = np.asarray(block_tables[b])[pos // bs]
        K = np.asarray(key_cache, np.float32)[phys, :, pos % bs]          # [total, kvh, d]
        V = np.asarray(value_cache, np.float32)[phys, :, pos % bs]
        for h in range(nh):
            s = K[:, h // rep] @ q[b, h] * scale
            p = np.exp(s - s.max())
            out[b, h] = (p / p.sum()) @ V[:, h // rep]
    return out.reshape(B, nh * d)


# csrc/gpu/fused_get_rope.cu:40-75 (use_neox=True: value j at columns j and j + d/2) / :97-138 (interleaved pairs)
def fused_get_rotary_embedding(input_ids_shape, position_ids, head_dim, prompt_num=0, theta=10000.0, use_neox=True):
    """fp32 arithmetic like the kernel: powf(theta, -2j/d) with the exponent formed as -(2j) * (1/d), angle = float(pos) * inv_freq."""
    bsz, seq = int(input_ids_shape[0]), int(input_ids_shape[1])
    half = head_dim // 2
    inv_head_dim = np.float32(1.0) / np.float32(head_dim)
    expo = (-(2 * np.arange(half)).astype(np.float32)) * inv_head_dim
    inv_freq = np.power(np.float32(theta), expo, dtype=np.float32)
    pos = np.asarray(position_ids)[:, prompt_num:prompt_num + seq].astype(np.float32)          # [bsz, seq]
    freqs = (pos[:, :, None] * inv_freq[None, None, :]).astype(np.float32)
    c, s = np.cos(freqs, dtype=np.float32), np.sin(freqs, dtype=np.float32)
    out = np.empty((2, bsz, 1, seq, head_dim), np.float32)
    if use_neox:
        out[0, :, 0, :, :half], out[0, :, 0, :, half:] = c, c
        out[1, :, 0, :, :half], out[1, :, 0, :, half:] = s, s
    else:
        out[0, :, 0, :, 0::2], out[0, :, 0, :, 1::2] = c, c
        out[1, :, 0, :, 0::2], out[1, :, 0, :, 1::2] = s, s
    return out


# csrc/gpu/step.cu:19-214 (free_and_dispatch_block + recover_block), executed in sequence-index order.
# PARITY UNPINNED: the reference holds no test or known-answer vector for step_paddle, and its kernels order the free list with
# atomicAdd / atomicSub across threads (timing dependent).  This restatement runs the threads in index order — one of the orders
# the reference can produce — and is checked on its invariants (tests/test_generation_oracle.py): every cache block is owned by
# exactly one of {free list, one sequence's table}, requests are served iff a block is free, pre-emption picks the largest holder.
def step_paddle(st, block_size, first_token_id=0):
    """`st`: dict of numpy arrays named like the reference op's inputs; updated IN PLACE (every input aliases an output)."""
    sf, stt, ose, sle, sld = st["stop_flags"], st["seq_lens_this_time"], st["ori_seq_lens_encoder"], st["seq_lens_encoder"], st["seq_lens_decoder"]
    bt, ebl, ibs = st["block_tables"], st["encoder_block_lens"], st["is_block_step"]
    sbl, sl, rbl, rl = st["step_block_list"], st["step_lens"], st["recover_block_list"], st["recover_lens"]
    nbl, nl, ull, fl, fll = st["need_block_list"], st["need_block_len"], st["used_list_len"], st["free_list"], st["free_list_len"]
    ids, pre, sidx, nxt = st["input_ids"], st["pre_ids"], st["step_idx"], st["next_tokens"]
    bsz = stt.shape[0]
    length = ids.shape[1]
    max_decoder_block_num = length // block_size
    # 1. free finished sequences / collect requests                                   (:41-67)
    for tid in range(bsz):
        if sf[tid] and not ibs[tid]:
            e, used = int(ebl[tid]), int(ull[tid])
            if used > 0:
                ori = int(fll[0]); fll[0] += used
                for i in range(used):
                    fl[ori + i] = bt[tid, e + i]
                    bt[tid, e + i] = -1
                ebl[tid] = 0
                ull[tid] = 0
        elif sld[tid] != 0 and bt[tid, sld[tid] // block_size] == -1:
            nbl[int(nl[0])] = tid
            nl[0] += 1
    # 2. pre-empt the largest holders until the requests fit                            (:73-103; cub::ArgMax: ties -> lowest index)
    while nl[0] > fll[0]:
        used = np.array([int(ull[t]) if not ibs[t] else 0 for t in range(bsz)])
        k = int(np.argmax(used)); v = int(used[k])
        if v <= 0:
            break                      # nothing to reclaim: the reference kernel would spin; the CUDA port breaks out as well
        e = int(ebl[k])
        for i in range(v):
            fl[int(fll[0]) + i] = bt[k, e + i]
            bt[k, e + i] = -1
        sbl[int(sl[0])] = k
        sl[0] += 1
        fll[0] += v
        sf[k] = True; ibs[k] = True; stt[k] = 0; sld[k] = 0
    # 3. one block per surviving request from the tail of the free list                 (:105-117)
    for t in range(int(nl[0])):
        rid = int(nbl[t])
        if not sf[rid]:
            ull[rid] += 1
            ori = int(fll[0]); fll[0] -= 1
            bt[rid, sld[rid] // block_size] = fl[ori - 1]
        nbl[t] = -1
    # 4. which parked sequences fit again                                              (:119-150)
    ori_free, ori_step_len = int(fll[0]), int(sl[0])
    if ori_step_len > 0:
        sid = int(sbl[ori_step_len - 1]); tmp = int(ull[sid])
        used_len = tmp + 1 if tmp < max_decoder_block_num else tmp
        while ori_step_len > 0 and ori_free >= used_len:
            rbl[int(rl[0])] = sid
            ibs[sid] = False
            ull[sid] = used_len
            ori_free -= used_len
            sbl[ori_step_len - 1] = -1
            sl[0] -= 1; rl[0] += 1
            ori_step_len = int(sl[0])
            if ori_step_len > 0:
                sid = int(sbl[ori_step_len - 1]); tmp = int(ull[sid])
                used_len = tmp + 1 if tmp < max_decoder_block_num else tmp
    nl[0] = 0
    # 5. recover_block                                                                  (:154-214)
    for b in range(int(rl[0])):
        rid = int(rbl[b])
        oe, sn = int(ose[rid]), int(sidx[rid])
        seq_len = oe + sn
        e, used = int(ebl[rid]), int(ull[rid])
        ori = int(fll[0]); fll[0] -= used
        for i in range(used):
            bt[rid, e + i] = fl[ori - i - 1]
        for i in range(sn - 1):
            ids[rid, oe + i] = pre[rid, i + 1]
        stt[rid] = seq_len; sle[rid] = seq_len; sf[rid] = False
        ids[rid, oe + sn - 1] = nxt[rid]
        ids[rid, 0] = first_token_id
    rl[0] = 0
    return st
