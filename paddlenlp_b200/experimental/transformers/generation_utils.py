"""GenerationInferenceModel — the dense-KV-cache generate loop of
paddlenlp/experimental/transformers/generation_utils.py (:124-183 generate, :262-400 sample, :185-260 state update).

Per step the reference runs: set_value_by_flags_and_idx -> cast fp32 -> get_token_penalty_multi_scores -> /temperature
-> softmax -> top_p_sampling_reject -> set_stop_value_multi_ends -> save_with_output, with one host sync in the `while`
condition.  Here the whole decode step (embedding .. lm_head .. token choice .. state update) is device-resident and
replayed as a CUDA graph; the stop condition is polled every `sync_interval` steps.  Greedy decoding (top_p == 0, the
benchmark setting: predictor.py:1196-1199) takes the arg-max directly; top_p > 0 runs softmax + rejection top-p sampling
(`top_p_sampling_reject`) with uniforms from a torch CUDA generator (graph-safe).
"""
from __future__ import annotations

import math
import time
from typing import List, Optional

import torch

from ... import ops

# step_paddle's state tensors, in its argument order
_STEP_PADDLE_ORDER = ("stop_flags", "seq_lens_this_time", "ori_seq_lens_encoder", "seq_lens_encoder", "seq_lens_decoder",
                      "block_tables", "encoder_block_lens", "is_block_step", "step_block_list", "step_lens", "recover_block_list",
                      "recover_lens", "need_block_list", "need_block_len", "used_list_len", "free_list", "free_list_len",
                      "input_ids", "pre_ids", "step_idx", "next_tokens")


class GenerationInferenceModel:
    def _prefill(self, input_ids, seq_lens_encoder, caches):
        raise NotImplementedError

    def _decode(self, tgt_ids, seq_lens_decoder, caches):
        raise NotImplementedError

    def _choose(self, logits, st):
        """fp32 cast -> penalties -> temperature -> softmax -> top-p sampling; with top_p == 0 the arg-max is taken
        directly (identical result: the sampler degenerates to top-1)."""
        greedy = st["top_p"] is None
        if greedy and st["plain"]:
            return ops.argmax(logits)
        lf = ops.bf16_rows_to_f32(logits)
        ops.token_penalty_multi_scores(st["pre_ids"], lf, st["penalty"], st["frequency"], st["presence"], st["temperature"],
                                       None, st["step_idx"], st["min_dec_len"], st["eos"])
        if greedy:
            return ops.argmax_f32(lf)
        ops.softmax_f32_(lf)
        return ops.top_p_sampling_reject(lf, st["top_p"], generator=st["generator"])

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, seq_len_encoder: Optional[torch.Tensor] = None, max_length: int = 64,
                 eos_token_id=None, cache_kvs: Optional[List[torch.Tensor]] = None, temperature: float = 1.0,
                 top_p: float = 0.0, penalty_score: float = 1.0, frequency_score: float = 0.0, presence_score: float = 0.0,
                 min_length: int = 0, use_cuda_graph: bool = True, sync_interval: int = 16, use_pdl: bool = True, seed: int = 0,
                 token_stream=None, **kwargs):
        """input_ids [B, S] (right padded); returns (ids [B, max_length], stop_flags, seq_len_decoder).
        top_p in (0, 1]: sample from the top-p nucleus (seed != 0 makes the draw reproducible); top_p 0: greedy.
        token_stream: a token_stream.TokenStream — every step's tokens are published to its pinned-host ring from inside
        the (graph-replayed) decode step, the replacement of save_with_output / save_output (generation_utils.py:353-361,
        :711-713): a reader thread sees step t while step t+1 is computed, with no host synchronisation in this loop."""
        if top_p is not None and not (0.0 <= float(top_p) <= 1.0):
            raise ValueError(f"top_p must be in [0, 1], got {top_p}")
        dev = self.device
        B, S = input_ids.shape
        ids = input_ids.to(dev, torch.int64).contiguous()
        enc = (torch.full((B,), S, dtype=torch.int32, device=dev) if seq_len_encoder is None
               else seq_len_encoder.to(dev, torch.int32).reshape(B).contiguous())
        if cache_kvs is None:
            cache_kvs = self.allocate_caches(B, S + max_length)
        tb = getattr(self, "transformer_block", None)
        if hasattr(tb, "check_cache_scales"):
            tb.check_cache_scales(cache_kvs)
        if getattr(self, "block_attn", False):                   # paged cache: capacity = blocks per sequence x block size
            if self.block_tables is None or self.block_tables.shape[0] != B:
                raise ValueError("block_attn: allocate the caches with allocate_caches(batch, max_len) for this batch size")
            max_len = self.block_tables.shape[1] * cache_kvs[0].shape[2]
        else:
            max_len = cache_kvs[0].shape[3]
        if S + max_length > max_len:
            raise ValueError(f"cache max_len {max_len} < prompt {S} + max_length {max_length}")
        # the rotary tables must cover every position the decode steps will index (they have max_position_embeddings rows at
        # construction; the KV cache may be longer): grow them now, before any kernel or graph captures their pointers
        if tb is not None and hasattr(tb, "ensure_rope"):
            tb.ensure_rope(S + max_length)
        eos = torch.tensor([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id or [-1]),
                           dtype=torch.int64, device=dev)
        st = dict(
            stop_flags=torch.zeros(B, dtype=torch.bool, device=dev), step_idx=torch.zeros(B, dtype=torch.int64, device=dev),
            max_dec_len=torch.full((B,), max_length, dtype=torch.int64, device=dev),
            min_dec_len=torch.full((B,), min_length, dtype=torch.int64, device=dev),
            seq_len_decoder=enc.clone(), pre_ids=torch.full((B, max_length + 1), -1, dtype=torch.int64, device=dev),
            eos=eos, out=torch.full((B, max_length), -1, dtype=torch.int64, device=dev),
            stop_count=torch.zeros(1, dtype=torch.int32, device=dev), col=torch.zeros(1, dtype=torch.int64, device=dev),
            penalty=torch.full((B,), penalty_score, dtype=torch.float32, device=dev),
            frequency=torch.full((B,), frequency_score, dtype=torch.float32, device=dev),
            presence=torch.full((B,), presence_score, dtype=torch.float32, device=dev),
            temperature=torch.full((B,), temperature, dtype=torch.float32, device=dev),
            plain=(penalty_score == 1.0 and frequency_score == 0.0 and presence_score == 0.0 and min_length <= 0
                   and temperature == 1.0),
            top_p=None, generator=None,
        )
        if top_p:
            st["top_p"] = torch.full((B,), float(top_p), dtype=torch.float32, device=dev)
            if seed:
                st["generator"] = torch.Generator(device=dev)
                st["generator"].manual_seed(int(seed))

        def update(next_tokens):
            # step_idx / stop flags / pre_ids / seq_len_decoder / token log — one kernel, no host sync.
            # seq_len_decoder is advanced for running sequences AFTER their token was chosen, so that the next
            # decode step appends at the right cache position.
            ops.generate_step_update(next_tokens, st["stop_flags"], st["step_idx"], st["max_dec_len"], st["seq_len_decoder"],
                                     st["pre_ids"], st["eos"], st["out"], st["stop_count"], out_col_dev=st["col"])
            if token_stream is not None:
                token_stream.push(next_tokens, st["stop_count"])

        if token_stream is not None:
            token_stream.reset(total_steps=max_length)
        # the penalty history of the first token is the last prompt token (entry 0; update() writes generated token k at entry
        # k), as set_value_by_flags_and_idx_v2 writes it in continuous_generate: the count stops at the first -1 entry
        st["pre_ids"][:, 0] = ids.gather(1, (enc - 1).to(torch.int64)[:, None])[:, 0]
        # ---- prefill ("encoder" step) ----
        logits = self._prefill(ids, enc, cache_kvs)              # [B, V], last valid position of each prompt
        tgt = self._choose(logits, st)
        # the prompt already occupies enc[b] cache slots; the first generated token will be appended at slot enc[b]
        st["seq_len_decoder"] -= 1                                # update() adds 1 for running sequences
        update(tgt)

        # ---- decode loop ----
        def step():
            lg = self._decode(tgt, st["seq_len_decoder"], cache_kvs)
            nxt = self._choose(lg, st)
            tgt.copy_(nxt)
            update(tgt)

        from ... import _lib

        graph = None
        n_steps = max_length - 1
        done = 0
        # programmatic dependent launch: every GEMM of the decode step prefetches its weight tiles while the previous
        # kernel drains (b200_set_pdl); restored on exit
        old_pdl = _lib.load().b200_set_pdl(1 if use_pdl else 0)
        try:
            if use_cuda_graph and n_steps > 2:
                step(); done += 1                                # warm-up (sets kernel attributes, allocator pools)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                if st["generator"] is not None:                  # philox offsets of a private generator advance per replay
                    graph.register_generator_state(st["generator"])
                with torch.cuda.graph(graph):                    # capture only records: no step is executed here
                    step()
            while done < n_steps:
                if graph is not None:
                    graph.replay()
                else:
                    step()
                done += 1
                if sync_interval > 0 and done % sync_interval == 0 and int(st["stop_count"].item()) >= B:
                    break
        finally:
            _lib.load().b200_set_pdl(old_pdl)
        self.last_generate_steps = done + 1
        return st["out"], st["stop_flags"].to(torch.int32), st["seq_len_decoder"]

    @torch.no_grad()
    def continuous_generate(self, requests, *, max_batch_size: int, num_blocks: int, eos_token_id=None, temperature: float = 1.0,
                            top_p: float = 0.0, penalty_score: float = 1.0, frequency_score: float = 0.0,
                            presence_score: float = 0.0, seed: int = 0, use_cuda_graph: bool = True):
        """Continuous batching on the paged KV cache.  `requests`: a list of (input_ids 1-D, max_length[, min_length]).  At
        most `max_batch_size` requests run at once; a finished slot takes the next queued request at the end of the same step;
        the cache is a pool of `num_blocks` pages shared by all of them (step_paddle pre-empts the largest holder when the
        pool runs dry and recovers it later).  Needs a model built with block_attn=True, append_attn=True.
        Returns (one int64 tensor of generated ids per request, in request order; stats dict).

        One step: get_padding_offset -> layers over the token_num packed rows (append_attention) -> rebuild_padding -> head ->
        set_value_by_flags_and_idx_v2 -> token choice -> set_stop_value_multi_ends v2 -> update_inputs -> step_paddle ->
        retire_admit, whose header (pinned host memory) the host reads once per step for the next step's token_num.
        Decode-only steps replay a CUDA graph per token_num (captured the second time that token_num occurs).

        Admission (retire_admit): FIFO, and nothing is admitted while a sequence is parked, so recovery goes first; a request is
        admitted only while the pool keeps one spare page per resident slot beyond every prompt page, and a parked sequence
        hands back its prompt pages too (it is recovered from position 0).  step_paddle can only pre-empt the pages a sequence
        grew into: with these rules a pool of at least the largest request's pages (plus the spare) always drains the queue.
        stats["decode_step_ms"] is the mean host-clock time of a decode-only step, the per-step header read included."""
        tb = self.transformer_block
        if not (getattr(self, "block_attn", False) and tb.config.append_attn):
            raise ValueError("continuous_generate needs a model built with block_attn=True, append_attn=True")
        if top_p is not None and not (0.0 <= float(top_p) <= 1.0):
            raise ValueError(f"top_p must be in [0, 1], got {top_p}")
        if not 1 <= int(max_batch_size) <= 1024:
            raise ValueError(f"max_batch_size must be in [1, 1024], got {max_batch_size}")
        bs, N, B = self.block_size, int(num_blocks), int(max_batch_size)
        prompts, max_lens, min_lens = [], [], []
        for i, rq in enumerate(requests):
            ids = torch.as_tensor(rq[0]).reshape(-1).to(torch.int64)
            max_len, min_len = int(rq[1]), int(rq[2]) if len(rq) > 2 else 0
            if ids.numel() == 0:
                raise ValueError(f"request {i}: empty prompt")
            if max_len < 1:
                raise ValueError(f"request {i}: max_length must be >= 1, got {max_len}")
            # alone in the pool a request holds its prompt's pages plus the one spare page admission keeps per slot, and at
            # most ceil((prompt + max_length) / block_size) pages
            pages = max(math.ceil((ids.numel() + max_len) / bs), math.ceil(ids.numel() / bs) + 1)
            if pages > N:
                raise ValueError(f"request {i}: {ids.numel()} prompt + {max_len} new tokens need {pages} pages of {bs} tokens, "
                                 f"more than num_blocks {N}")
            prompts.append(ids.cpu()); max_lens.append(max_len); min_lens.append(min_len)
        R = len(prompts)
        if R == 0:
            return [], {}
        dev = self.device
        plens = [p.numel() for p in prompts]
        max_dec, max_seq = max(max_lens), max(p + m for p, m in zip(plens, max_lens))
        bnps = math.ceil(max_seq / bs) + 1          # one spare column: step_paddle recovers a sequence with used + 1 pages
        width = bnps * bs
        tb.ensure_rope(max_seq)

        def i32(*shape, fill=0):
            return torch.full(shape, fill, dtype=torch.int32, device=dev)

        def i64(*shape, fill=0):
            return torch.full(shape, fill, dtype=torch.int64, device=dev)

        st = dict(
            stop_flags=torch.ones(B, dtype=torch.bool, device=dev), is_block_step=torch.zeros(B, dtype=torch.bool, device=dev),
            seq_lens_this_time=i32(B), ori_seq_lens_encoder=i32(B), seq_lens_encoder=i32(B), seq_lens_decoder=i32(B),
            block_tables=i32(B, bnps, fill=-1), encoder_block_lens=i32(B), step_block_list=i32(B, fill=-1), step_lens=i32(1),
            recover_block_list=i32(B, fill=-1), recover_lens=i32(1), need_block_list=i32(B, fill=-1), need_block_len=i32(1),
            used_list_len=i32(B), free_list=torch.arange(N, dtype=torch.int32, device=dev), free_list_len=i32(1, fill=N),
            input_ids=i64(B, width), pre_ids=i64(B, max_dec + 1, fill=-1), step_idx=i64(B), next_tokens=i64(B, fill=-1),
            max_dec_len=i64(B), min_dec_len=i64(B), slot_request=i32(B, fill=-1),
            prompt_ids=torch.cat(prompts).to(dev),
            prompt_offsets=torch.tensor([0] + plens, dtype=torch.int64).cumsum(0).to(device=dev, dtype=torch.int32),
            req_max_dec_len=torch.tensor(max_lens, dtype=torch.int64, device=dev),
            req_min_dec_len=torch.tensor(min_lens, dtype=torch.int64, device=dev),
            cursor=i32(1), out_ids=i64(R, max_dec, fill=-1), out_lens=i32(R),
        )
        header = torch.zeros(ops.RA_HEADER_INTS, dtype=torch.int32).pin_memory()
        caches = [torch.zeros(N, tb.kvh, bs, tb.d, dtype=getattr(self, "cache_dtype", torch.bfloat16), device=dev)
                  for _ in range(2 * tb.L)]
        tb.check_cache_scales(caches)
        eos = torch.tensor([eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id or [-1]),
                           dtype=torch.int64, device=dev)
        samp = dict(pre_ids=st["pre_ids"], step_idx=st["step_idx"], min_dec_len=st["min_dec_len"], eos=eos,
                    penalty=torch.full((B,), penalty_score, dtype=torch.float32, device=dev),
                    frequency=torch.full((B,), frequency_score, dtype=torch.float32, device=dev),
                    presence=torch.full((B,), presence_score, dtype=torch.float32, device=dev),
                    temperature=torch.full((B,), temperature, dtype=torch.float32, device=dev),
                    plain=(penalty_score == 1.0 and frequency_score == 0.0 and presence_score == 0.0 and temperature == 1.0
                           and max(min_lens) <= 0),
                    top_p=None, generator=None)
        if top_p:
            samp["top_p"] = torch.full((B,), float(top_p), dtype=torch.float32, device=dev)
            if seed:
                samp["generator"] = torch.Generator(device=dev)
                samp["generator"].manual_seed(int(seed))
        not_need_stop = torch.zeros(1, dtype=torch.bool, device=dev)
        stop_nums = torch.full((1,), B, dtype=torch.int64, device=dev)

        def admit():
            ops.retire_admit(st, header, bs, max(plens), max_seq)

        def step(token_num, max_q_len):
            this_time, enc, dec = st["seq_lens_this_time"], st["seq_lens_encoder"], st["seq_lens_decoder"]
            cum = torch.cumsum(width - this_time, 0, dtype=torch.int32)
            ids, cum_out, _, cu_q, _ = ops.get_padding_offset(st["input_ids"], cum, token_num, this_time)
            logits = self._forward_packed(ids, caches, st["block_tables"], enc, dec, this_time, cu_q, cum_out, max_q_len, width)
            ops.set_value_by_flags_and_idx_v2(st["pre_ids"], st["input_ids"], this_time, enc, dec, st["step_idx"],
                                              st["stop_flags"])
            topk = self._choose(logits, samp)
            st["step_idx"].add_((~st["stop_flags"]).to(torch.int64))
            ops.set_stop_value_multi_ends(topk, st["stop_flags"], eos, seq_lens=this_time, next_tokens=st["next_tokens"])
            # the length stop comes after the EOS substitution, so that the last token of a request is the one it chose
            # (as in generate(); the reference flags the length first and replaces that token by EOS)
            torch.logical_or(st["stop_flags"], st["step_idx"] >= st["max_dec_len"], out=st["stop_flags"])
            ops.update_inputs(st["stop_flags"], not_need_stop, this_time, enc, dec, st["input_ids"], stop_nums,
                              st["next_tokens"], st["is_block_step"])
            ops.step_paddle(*[st[k] for k in _STEP_PADDLE_ORDER], block_size=bs)
            admit()

        # every captured graph bakes in the addresses of the scratch buffers its kernels use, and a buffer that grows later
        # frees the block a graph still writes to.  The append_attention and penalty buffers depend on the slot count only and
        # are sized by the first step, which always runs eagerly; the split-K GEMM buffer grows with the rows of any step up to
        # SKINNY_M, so it is sized here for the widest GEMM the step runs (layers and head)
        head_n = self.config.vocab_size
        ops.reserve_gemm_skinny_workspace(tb.SKINNY_M, max(tb.qkv_n, tb.h, 2 * tb.I, head_n), dev)
        stats = dict(steps=0, decode_steps=0, mixed_steps=0, preemptions=0, recoveries=0, peak_blocks_in_use=0,
                     free_blocks_at_exit=0, decode_step_ms=0.0)
        # one memory pool for all graphs: they never run concurrently, and no tensor a graph allocates outlives its replay
        # (the step's state lives in `st`, allocated outside every graph)
        graphs, seen, pool = {}, set(), torch.cuda.graph_pool_handle()
        stream = torch.cuda.current_stream()
        decode_s, t_decode = 0.0, None
        try:
            admit()
            while True:
                stream.synchronize()                             # the one host synchronisation per step: the header
                if t_decode is not None:
                    decode_s += time.perf_counter() - t_decode
                    t_decode = None
                h = header.tolist()
                stats["peak_blocks_in_use"] = max(stats["peak_blocks_in_use"], N - h[ops.RA_FREE_BLOCKS])
                if h[ops.RA_DONE]:
                    break
                T, Q = h[ops.RA_TOKEN_NUM], h[ops.RA_MAX_Q_LEN]
                if T == 0:
                    if h[ops.RA_PARKED] == 0:
                        raise RuntimeError(f"continuous_generate: no slot can run ({h[ops.RA_PENDING]} requests pending, "
                                           f"{h[ops.RA_FREE_BLOCKS]} free blocks)")
                    # the last running sequence was parked in the step that just ran, before retire_admit released its
                    # encoder blocks: no model rows, step_paddle alone recovers it from the now free pool
                    ops.step_paddle(*[st[k] for k in _STEP_PADDLE_ORDER], block_size=bs)
                    admit()
                    continue
                stats["steps"] += 1
                stats["decode_steps" if Q == 1 else "mixed_steps"] += 1
                if Q == 1:
                    t_decode = time.perf_counter()
                if use_cuda_graph and Q == 1 and T in seen:
                    g = graphs.get(T)
                    if g is None:                                # the first step of this token_num ran eagerly (warm-up)
                        g = torch.cuda.CUDAGraph()
                        if samp["generator"] is not None:
                            g.register_generator_state(samp["generator"])
                        with torch.cuda.graph(g, pool=pool):     # capture only records: the step runs at the replay
                            step(T, 1)
                        graphs[T] = g
                    g.replay()
                else:
                    step(T, Q)
                    if Q == 1:
                        seen.add(T)
        finally:
            stream.synchronize()
            graphs.clear()
        stats["preemptions"], stats["recoveries"] = h[ops.RA_PREEMPTIONS], h[ops.RA_RECOVERIES]
        stats["free_blocks_at_exit"] = h[ops.RA_FREE_BLOCKS]
        stats["decode_step_ms"] = 1e3 * decode_s / max(stats["decode_steps"], 1)
        self.last_block_tables = st["block_tables"]
        out, lens = st["out_ids"].cpu(), st["out_lens"].cpu()
        return [out[r, :int(lens[r])].clone() for r in range(R)], stats
