"""CPU restatement of b200_retire_admit (TEST INFRASTRUCTURE ONLY), the continuous-batching step that runs right after
step_paddle: retire finished slots into a per-request output buffer, return their encoder blocks, and admit queued requests
into the empty slots.  The reference has no such op (its serving stack does this on the host), so there is nothing to pin it
against; it is written in the style of generation_ref.step_paddle, in slot-index order, and tested on its invariants
(tests/test_continuous_batching_cpu.py) and bit-exact against the kernel (tests/test_continuous_batching_gpu.py)."""

# int32 words of the step header (enum B200_RA_* of include/b200nlp.h)
TOKEN_NUM, MAX_Q_LEN, RUNNING, PENDING, PARKED, DONE, FREE_BLOCKS, PREEMPTIONS, RECOVERIES, ADMITTED, RETIRED = range(11)
HEADER_INTS = 16


def retire_admit(st, header, block_size):
    """`st`: dict of numpy arrays named like the op's arguments (the step_paddle state plus max_dec_len, min_dec_len,
    slot_request, the queue prompt_ids / prompt_offsets / req_max_dec_len / req_min_dec_len / cursor and the outputs
    out_ids / out_lens); `header` int32 [HEADER_INTS].  Everything is updated IN PLACE."""
    sf, ibs, stt, sle, ose, sld = (st[k] for k in ("stop_flags", "is_block_step", "seq_lens_this_time", "seq_lens_encoder",
                                                   "ori_seq_lens_encoder", "seq_lens_decoder"))
    sidx, pre, nxt, ids, bt, ebl, ull = (st[k] for k in ("step_idx", "pre_ids", "next_tokens", "input_ids", "block_tables",
                                                         "encoder_block_lens", "used_list_len"))
    fl, fll, sl, mdl, mnl, sreq = (st[k] for k in ("free_list", "free_list_len", "step_lens", "max_dec_len", "min_dec_len",
                                                   "slot_request"))
    pids, poff, qmax, qmin, cur, out, olen = (st[k] for k in ("prompt_ids", "prompt_offsets", "req_max_dec_len",
                                                             "req_min_dec_len", "cursor", "out_ids", "out_lens"))
    bsz = stt.shape[0]
    R, out_stride = qmax.shape[0], out.shape[1]
    # 0 / 1 / 2: recovered slots get their first prompt token back; parked and retiring slots return their encoder blocks
    # (a parked slot counts them as decoder blocks from now on); retiring slots record their tokens and empty
    recovered = 0
    retired = []
    for b in range(bsz):
        r = int(sreq[b])
        if r >= 0 and not sf[b] and sle[b] > 0 and sidx[b] > 0:
            ids[b, 0] = pids[poff[r]]
            recovered += 1
        parked = bool(ibs[b])
        retire = r >= 0 and bool(sf[b]) and not parked
        if parked or retire:
            # what the row still holds are the encoder blocks, a prefix of it: step_paddle cleared the decoder entries (and,
            # for a stopped slot, zeroed encoder_block_lens too)
            e = 0
            while e < bt.shape[1] and bt[b, e] >= 0:
                fl[int(fll[0])] = bt[b, e]
                fll[0] += 1
                bt[b, e] = -1
                e += 1
            ebl[b] = 0
            if parked:
                ull[b] += e
        if retire:
            n = min(int(sidx[b]), out_stride)
            if n > 0:
                out[r, :n - 1] = pre[b, 1:n]
                out[r, n - 1] = nxt[b]
            olen[r] = n
            sreq[b] = -1
            retired.append(b)
    # 3: FIFO admission into the empty slots in slot order, while nothing is parked
    # (the pool keeps one block per resident slot beyond every encoder block: step_paddle can only pre-empt decoder blocks)
    admitted = 0
    occupied = int((sreq >= 0).sum())
    held_dec = int(sum(int(ull[b]) for b in range(bsz) if sreq[b] >= 0 and not ibs[b]))
    if int(sl[0]) == 0:
        for b in range(bsz):
            if sreq[b] >= 0:
                continue
            r = int(cur[0])
            if r >= R:
                break
            plen = int(poff[r + 1] - poff[r])
            need = (plen + block_size - 1) // block_size
            if need > int(fll[0]) or need + occupied + admitted + 1 > int(fll[0]) + held_dec:
                break                                          # the head request waits: nothing overtakes it
            for j in range(need):
                bt[b, j] = fl[int(fll[0]) - 1]
                fll[0] -= 1
            ebl[b] = need
            ull[b] = 0
            stt[b] = sle[b] = ose[b] = plen
            sld[b] = 0
            sidx[b] = 0
            sf[b] = False
            mdl[b], mnl[b] = qmax[r], qmin[r]
            sreq[b] = r
            ids[b, :plen] = pids[poff[r]:poff[r + 1]]
            pre[b, :] = -1
            cur[0] += 1
            admitted += 1
    # 4: step header
    parked_now = int(sl[0])
    header[PREEMPTIONS] += parked_now - int(header[PARKED]) + recovered
    header[RECOVERIES] += recovered
    header[TOKEN_NUM] = int(stt.sum())
    header[MAX_Q_LEN] = int(stt.max()) if bsz else 0
    header[RUNNING] = int((stt > 0).sum())
    header[PENDING] = R - int(cur[0])
    header[PARKED] = parked_now
    header[FREE_BLOCKS] = int(fll[0])
    header[ADMITTED] = admitted
    header[RETIRED] = len(retired)
    header[DONE] = int(not (sreq >= 0).any() and int(cur[0]) >= R)
    return st
