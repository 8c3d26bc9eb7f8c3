"""GPU parity of the generation path (through the C-ABI): bookkeeping ops vs the reference's known-answer vectors and
the numpy oracle; decode kernels vs the oracle; end-to-end greedy generation vs uncached oracle decoding."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import generation_ref as G
from oracle import llama_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bookkeeping.json")))


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


def t(x, dtype):
    return torch.tensor(x, dtype=dtype, device=DEV)


def test_get_padding_offset_known_answer():
    g = GOLD["get_padding_offset_v2"]
    xr, co, po, cq, ck = ops().get_padding_offset(t(g["input_ids"], torch.int64), t(g["cum_offsets"], torch.int32),
                                                  g["token_num"], t(g["seq_lens"], torch.int32))
    assert xr.tolist() == g["ref_x_remove_padding"] and co.tolist() == g["ref_cum_offsets_out"]
    assert po.tolist() == g["ref_padding_offset"] and cq.tolist() == g["ref_cu_seqlens_q"] and ck.tolist() == g["ref_cu_seqlens_k"]


def test_token_penalty_known_answer_and_random():
    g = GOLD["token_penalty_v2"]
    case = g["cases"][0]
    lg = t(case["logits"], torch.float32)
    ops().token_penalty_multi_scores(t(case["pre_ids"], torch.int64), lg, t(g["penalty_scores"], torch.float32),
                                     t(g["frequency_scores"], torch.float32), t(g["presence_scores"], torch.float32),
                                     t(g["temperatures"], torch.float32), t(g["bad_tokens"], torch.int64),
                                     t(g["cur_len"], torch.int64), t(g["min_len"], torch.int64), t(g["eos_token_id"], torch.int64))
    assert np.sum(np.abs(lg.cpu().numpy() - np.array(case["ref_logits"], np.float32))) < 1e-6
    # random case vs the numpy oracle (penalty != 1, presence != 0, -1 padded history)
    rng = np.random.default_rng(0)
    bs, V, Lh = 3, 500, 40
    pre = rng.integers(0, V, (bs, Lh)).astype(np.int64)
    pre[:, 25:] = -1
    logits = rng.standard_normal((bs, V)).astype(np.float32)
    pen, fr, pr, tp = [1.3, 1.0, 0.8], [0.2, 0.0, 0.1], [0.5, 0.0, 0.3], [0.7, 1.0, 2.0]
    cur, mn, eos, bad = [25, 3, 25], [30, 1, 1], [7, 9], [3]
    ref = G.token_penalty_multi_scores_v2(pre, logits, pen, fr, pr, tp, bad, cur, mn, eos)
    lg = t(logits, torch.float32)
    ops().token_penalty_multi_scores(t(pre, torch.int64), lg, t(pen, torch.float32), t(fr, torch.float32), t(pr, torch.float32),
                                     t(tp, torch.float32), t(bad, torch.int64), t(cur, torch.int64), t(mn, torch.int64),
                                     t(eos, torch.int64))
    assert np.allclose(lg.cpu().numpy(), ref, rtol=1e-6, atol=1e-6)


def test_stop_value_and_flags_known_answers():
    o = ops()
    g = GOLD["set_stop_value_multi_ends_v2"]
    topk, stop, nxt = t(g["topk_ids"], torch.int64), t(g["stop_flags"], torch.bool), t(g["next_tokens"], torch.int64)
    o.set_stop_value_multi_ends(topk, stop, t(g["end_ids"], torch.int64), seq_lens=t(g["seq_lens"], torch.int32), next_tokens=nxt)
    assert topk.tolist() == g["ref_topk_ids"] and nxt.tolist() == g["ref_next_tokens"] and stop.tolist() == g["ref_stop_flags"]
    # v1 (mode 2) vs oracle
    topk1 = torch.arange(10, dtype=torch.int64, device=DEV)
    stop1 = t([0, 1, 0, 0, 1, 0, 0, 0, 0, 1], torch.bool)
    rt, rs = G.set_stop_value_multi_ends(topk1.cpu().numpy(), stop1.cpu().numpy(), [2, 7])
    o.set_stop_value_multi_ends(topk1, stop1, t([2, 7], torch.int64))
    assert topk1.tolist() == rt.tolist() and stop1.tolist() == rs.tolist()
    g = GOLD["set_value_by_flags_and_idx_v2"]
    pre = t(g["pre_ids_all"], torch.int64)
    o.set_value_by_flags_and_idx_v2(pre, t(g["input_ids"], torch.int64), None, t(g["seq_lens_encoder"], torch.int32),
                                    t(g["seq_lens_decoder"], torch.int32), t(g["step_idx"], torch.int64),
                                    t(g["stop_flags"], torch.bool))
    assert pre.tolist() == g["ref_pre_ids_all"]
    pre1 = torch.full((3, 6), -1, dtype=torch.int64, device=DEV)
    o.set_value_by_flags_and_idx(pre1, t([5, 6, 7], torch.int64), t([2, -1, 4], torch.int64), t([0, 0, 1], torch.bool))
    ref1 = G.set_value_by_flags_and_idx(np.full((3, 6), -1, np.int64), [5, 6, 7], [2, -1, 4], [False, False, True])
    assert pre1.tolist() == ref1.tolist()


def test_update_inputs_known_answer():
    g = GOLD["update_inputs"]
    max_bs = len(g["stop_flags"])
    ids = torch.zeros(max_bs, 4, dtype=torch.int64, device=DEV)
    ids[:, 0] = t(g["input_ids_col0_before"], torch.int64)
    nns = torch.ones(1, dtype=torch.bool, device=DEV)
    tt, enc, dec = t(g["seq_lens_this_time"], torch.int32), t(g["seq_lens_encoder"], torch.int32), t(g["seq_lens_decoder"], torch.int32)
    ops().update_inputs(t(g["stop_flags"], torch.bool), nns, tt, enc, dec, ids, t(g["stop_nums"], torch.int64),
                        t(g["next_tokens"], torch.int64), t(g["is_block_step"], torch.bool))
    assert bool(nns.item()) == g["ref_not_need_stop"] and tt.tolist() == g["ref_seq_lens_this_time"]
    assert enc.tolist() == g["ref_seq_lens_encoder"] and dec.tolist() == g["ref_seq_lens_decoder"]
    assert ids[:, 0].tolist() == g["ref_input_ids_col0"]


def test_rebuild_padding_vs_oracle():
    rng = np.random.default_rng(1)
    max_len, seq = 10, np.array([4, 3, 6], np.int32)
    cum = np.insert(np.cumsum(max_len - seq), 0, 0)[:-1].astype(np.int32)
    tmp = torch.tensor(rng.standard_normal((int(seq.sum()), 136)), dtype=BF16)
    out = ops().rebuild_padding(tmp.to(DEV), t(cum, torch.int32), t([0, 0, 0], torch.int32), t(seq, torch.int32), max_len)
    ref = G.rebuild_padding_v2(tmp.float().numpy(), cum, np.zeros(3, np.int32), seq, max_len)
    assert np.array_equal(out.float().cpu().numpy(), ref)


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("nh,kvh", [(4, 1), (8, 2), (7, 1)])
def test_decode_rope_append_and_attention(nh, kvh, impl):
    o = ops()
    B, d, max_len = 3, 128, 96
    g = torch.Generator().manual_seed(2)
    lens = torch.tensor([5, 40, 95 - 1], dtype=torch.int32)              # tokens already cached
    cache = torch.randn(2, B, kvh, max_len, d, generator=g).to(BF16)
    qkv = torch.randn(B, (nh + 2 * kvh) * d, generator=g).to(BF16)
    cos, sin = o.rope_tables(d, max_len, 10000.0, DEV)
    qkv_d, cache_d = qkv.clone().to(DEV), cache.clone().to(DEV)
    o.decode_rope_append(qkv_d, cache_d, cos, sin, lens.to(DEV), nh, kvh, d)
    out = o.decode_attention(qkv_d, cache_d, lens.to(DEV), nh, kvh, d, impl=impl).float().cpu()
    out1 = o.decode_attention(qkv_d, cache_d, lens.to(DEV), nh, kvh, d, num_splits=1, impl=impl).float().cpu()
    out3 = o.decode_attention(qkv_d, cache_d, lens.to(DEV), nh, kvh, d, num_splits=3, impl=impl).float().cpu()
    assert (out1 - out3).abs().max() < 1e-2 * out1.abs().max()
    c, s = R.rope_tables(d, max_len, 10000.0)
    for b in range(B):
        p = int(lens[b])
        qk = qkv[b, : (nh + kvh) * d].float().view(1, 1, nh + kvh, d)
        rot = R.apply_rope(qk, c, s, "bf16", position_ids=torch.tensor([[p]]))[0, 0]
        q, knew = rot[:nh], rot[nh:]
        vnew = qkv[b, (nh + kvh) * d:].float().view(kvh, d)
        assert torch.equal(cache_d[0, b, :, p].float().cpu(), knew) or (cache_d[0, b, :, p].float().cpu() - knew).abs().max() < 2e-2
        assert torch.equal(cache_d[1, b, :, p].float().cpu(), vnew)
        K = torch.cat([cache[0, b, :, :p].float(), knew[:, None]], dim=1)       # [kvh, p+1, d]
        V = torch.cat([cache[1, b, :, :p].float(), vnew[:, None]], dim=1)
        rep = nh // kvh
        Kr, Vr = K.repeat_interleave(rep, 0), V.repeat_interleave(rep, 0)
        sc = torch.einsum("hd,htd->ht", q, Kr) / d ** 0.5
        ref = torch.einsum("ht,htd->hd", torch.softmax(sc, -1), Vr).reshape(-1)
        err = (out[b] - ref).abs().max() / ref.abs().max()
        assert err < 1.5e-2, (b, err)


@pytest.mark.parametrize("nh,kvh,B,max_len,splits", [(32, 8, 24, 700, 0), (8, 1, 200, 300, 1), (28, 4, 5, 1100, 4), (2, 2, 3, 130, 2),
                                                     (8, 1, 200, 300, 0), (28, 4, 5, 1100, 0), (4, 1, 1, 4096, 0), (2, 2, 3, 130, 0),
                                                     (32, 8, 64, 1100, 0), (16, 2, 300, 2100, 0)])
def test_decode_attention_tc_long(nh, kvh, B, max_len, splits):
    """The decode attention kernel over many work items, several 128-row tiles per item, ragged lengths (incl. 0
    cached tokens and a full cache), vs an fp32 reference and vs the CUDA-core kernel.  splits 0 = the library's own choice.
    Partial last tiles are fetched in 32-row boxes: lengths just past / just short of a tile boundary are in the ragged draw."""
    o = ops()
    d = 128
    g = torch.Generator().manual_seed(B + nh)
    lens = torch.randint(0, max_len - 1, (B,), generator=g).to(torch.int32)
    lens[0], lens[-1] = 0, max_len - 1                                   # shortest case; cache already full (clamped)
    cache = torch.randn(2, B, kvh, max_len, d, generator=g).to(BF16)
    qkv = torch.randn(B, (nh + 2 * kvh) * d, generator=g).to(BF16)
    qkv_d, cache_d, lens_d = qkv.to(DEV), cache.to(DEV), lens.to(DEV)
    out = o.decode_attention(qkv_d, cache_d, lens_d, nh, kvh, d, num_splits=splits, impl="tc").float().cpu()
    alt = o.decode_attention(qkv_d, cache_d, lens_d, nh, kvh, d, impl="simt").float().cpu()
    rep = nh // kvh
    q = qkv[:, : nh * d].float().view(B, kvh, rep, d)
    K, V = cache[0].float(), cache[1].float()                            # [B, kvh, max_len, d]
    sc = torch.einsum("bkrd,bktd->bkrt", q, K) / d ** 0.5
    total = torch.clamp(lens.long() + 1, max=max_len)
    mask = torch.arange(max_len)[None, :] >= total[:, None]
    sc = sc.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = torch.einsum("bkrt,bktd->bkrd", torch.softmax(sc, -1), V).reshape(B, nh * d)
    scale = ref.abs().max()
    assert (out - ref).abs().max() / scale < 1.5e-2
    assert (out - alt).abs().max() / scale < 1.5e-2
    assert torch.isfinite(out).all()


def _tiny(model_type="llama"):
    return R.RefConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                       num_key_value_heads=1, rope_theta=10000.0, qkv_bias=(model_type == "qwen2"), model_type=model_type,
                       max_position_embeddings=128, rms_norm_eps=1e-5)


def _infer_model(cfg, w):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    c = T.Qwen2Config(**kw) if cfg.model_type == "qwen2" else T.LlamaConfig(**kw)
    m = LlamaForCausalLMInferenceModel(c)
    m.set_state_dict(w)
    return m, c


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_prefill_logits_equal_training_path(model_type):
    """The fused-inference prefill re-associates the same kernels: its logits must equal the training-path forward."""
    import paddlenlp_b200.transformers as T

    cfg = _tiny(model_type)
    w = R.init_weights(cfg, seed=5)
    w = {k: (v * 3).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    m, c = _infer_model(cfg, w)
    train = (T.Qwen2ForCausalLM if model_type == "qwen2" else T.LlamaForCausalLM)(c)
    train.set_state_dict(w)
    ids = torch.randint(0, cfg.vocab_size, (2, 128), generator=torch.Generator().manual_seed(3)).to(DEV)
    a = m.forward_logits_prefill(ids)
    with torch.no_grad():
        b = train(input_ids=ids)[0]
    assert torch.equal(a, b)


@pytest.mark.parametrize("use_graph,use_pdl", [(False, False), (True, False), (True, True), (False, True)])
def test_greedy_generation_matches_uncached_oracle(use_graph, use_pdl):
    cfg = _tiny()
    w = R.init_weights(cfg, seed=9)
    w = {k: (v * 4).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    m, _ = _infer_model(cfg, w)
    g = torch.Generator().manual_seed(4)
    B, S, new = 3, 24, 12
    lens = torch.tensor([24, 17, 9], dtype=torch.int32)
    ids = torch.randint(1, cfg.vocab_size, (B, S), generator=g)
    for b in range(B):
        ids[b, lens[b]:] = 0                                         # right padding
    out, stop, dec = m.generate(ids.to(DEV), seq_len_encoder=lens.to(DEV), max_length=new, eos_token_id=-7,
                                use_cuda_graph=use_graph, sync_interval=4, use_pdl=use_pdl)
    ref, margins = G.greedy_generate(ids, w, cfg, new, eos=None, mode="bf16", seq_lens=lens)
    out = out.cpu()
    # token-id argmax must match wherever the oracle's top-1/top-2 margin is above bf16 noise; after a legitimate
    # near-tie divergence the sequences differ, so compare up to the first non-decisive position of each row.
    compared = 0
    for b in range(B):
        for tpos in range(new):
            if margins[b, tpos] < 2e-2:
                break
            assert int(out[b, tpos]) == int(ref[b, tpos]), (b, tpos, out[b].tolist(), ref[b].tolist())
            compared += 1
    assert compared >= 12, f"only {compared} decisive positions were compared"
    # the last generated token is never fed back: the last appended cache index is prompt + generated - 2
    assert dec.cpu().tolist() == (lens + new - 2).tolist()


def test_generation_stops_on_eos_and_penalty_path_runs():
    cfg = _tiny()
    w = R.init_weights(cfg, seed=9)
    w = {k: (v * 4).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    m, _ = _infer_model(cfg, w)
    ids = torch.randint(1, cfg.vocab_size, (2, 16), generator=torch.Generator().manual_seed(6)).to(DEV)
    free, _, _ = m.generate(ids, max_length=10, eos_token_id=-7, use_cuda_graph=False)
    eos = int(free[0, 3])                                            # make the 4th token of row 0 the EOS id
    out, stop, _ = m.generate(ids, max_length=10, eos_token_id=eos, use_cuda_graph=False, sync_interval=1)
    row = out[0].tolist()
    k = row.index(eos)
    assert k <= 3 and all(x == eos for x in row[k:]) and int(stop[0]) == 1
    # non-default penalties take the fp32 logits -> penalty -> argmax path
    out2, _, _ = m.generate(ids, max_length=6, eos_token_id=-7, use_cuda_graph=False, penalty_score=1.2, frequency_score=0.1,
                            presence_score=0.1, temperature=0.8, min_length=2)
    assert out2.shape == (2, 6) and int(out2.min()) >= 0


def test_softmax_and_top_p_sampling_reject():
    o = ops()
    rng = np.random.default_rng(7)
    # (1) softmax vs torch
    lg = torch.tensor(rng.standard_normal((5, 40080)).astype(np.float32) * 5)
    pr = o.softmax_f32_(lg.clone().to(DEV)).cpu()
    ref = torch.softmax(lg, -1)
    assert ((pr - ref).abs() <= 1e-5 * ref + 1e-12).all() and abs(float(pr.sum(-1).min()) - 1) < 1e-5   # few-ulp agreement
    # (2) dyadic probabilities (every partial sum exact in fp32, whatever the summation order): bit-exact vs the oracle
    bs, V = 6, 8192
    w = rng.integers(0, 64, size=(bs, V)).astype(np.float64)
    w[:, :7] = 0                                                      # zero-probability tokens are never sampled
    w[0, 100] = 5000; w[1, V - 1] = 9000                              # a dominant token; one at the very end
    tot = 2.0 ** 20
    w[:, 500] += tot - w.sum(-1)                                       # rows sum to exactly 2^20
    p = (w / tot).astype(np.float32)
    assert np.all(p.sum(-1, dtype=np.float64) == 1.0) and (p >= 0).all()
    u = ((rng.integers(0, 2 ** 16, size=(32, bs)) + 0.5) / 2 ** 16).astype(np.float32)   # never equal to a partial sum
    for tp in (0.0, 0.25, 0.6, 1.0):
        tpv = np.full(bs, tp, np.float32)
        got = o.top_p_sampling_reject(t(p, torch.float32), t(tpv, torch.float32), uniform=t(u, torch.float32)).cpu().numpy()
        assert np.array_equal(got, G.top_p_sampling_reject(p, tpv, u)), tp
    # (3) realistic softmax rows on the reference test's shape: sample inside the nucleus, top_p 0 == arg max, reproducible
    probs = torch.softmax(torch.tensor(rng.standard_normal((3, 40080)).astype(np.float32) * 3), -1)
    pd = probs.to(DEV)
    ids0 = o.top_p_sampling_reject(pd, t(np.zeros(3, np.float32), torch.float32), seed=11).cpu()
    assert torch.equal(ids0, probs.argmax(-1))
    tpv = np.array([0.2, 0.7, 0.95], np.float32)
    a = o.top_p_sampling_reject(pd, t(tpv, torch.float32), seed=11).cpu()
    b = o.top_p_sampling_reject(pd, t(tpv, torch.float32), seed=11).cpu()
    assert torch.equal(a, b)
    for i in range(3):
        assert float(probs[i][probs[i] > probs[i, a[i]]].sum()) < tpv[i] + 1e-6
    # (4) frequencies follow the renormalised nucleus (top_p 1 == plain sampling): 4 tokens, 20000 draws
    small = torch.tensor([[0.5, 0.25, 0.125, 0.125]], dtype=torch.float32).repeat(20000, 1).to(DEV)
    ids = o.top_p_sampling_reject(small, torch.ones(20000, dtype=torch.float32, device=DEV), seed=3).cpu()
    freq = torch.bincount(ids, minlength=4).float() / 20000
    assert (freq - torch.tensor([0.5, 0.25, 0.125, 0.125])).abs().max() < 0.015
    ids = o.top_p_sampling_reject(small, torch.full((20000,), 0.6, dtype=torch.float32, device=DEV), seed=3).cpu()
    freq = torch.bincount(ids, minlength=4).float() / 20000                 # nucleus {0, 1}: mass above token 1 is 0.5 < 0.6
    assert freq[2] == 0 and freq[3] == 0 and abs(float(freq[0]) - 2 / 3) < 0.02


def test_generate_with_top_p_sampling():
    """generate(top_p > 0): reproducible for a fixed seed, CUDA-graph and eager agree, tiny top_p reproduces greedy."""
    cfg = _tiny()
    w = R.init_weights(cfg, seed=5)
    m, _ = _infer_model(cfg, w)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, cfg.vocab_size, (3, 12), generator=g)
    greedy, _, _ = m.generate(ids, max_length=10, top_p=0.0)
    tiny_p, _, _ = m.generate(ids, max_length=10, top_p=1e-6, seed=5)
    assert torch.equal(greedy, tiny_p)
    a, _, _ = m.generate(ids, max_length=10, top_p=0.9, temperature=1.3, seed=42)
    b, _, _ = m.generate(ids, max_length=10, top_p=0.9, temperature=1.3, seed=42)
    c, _, _ = m.generate(ids, max_length=10, top_p=0.9, temperature=1.3, seed=42, use_cuda_graph=False)
    assert torch.equal(a, b) and a.shape == (3, 10) and int(a.min()) >= 0 and int(a.max()) < cfg.vocab_size
    assert torch.equal(a, c)
    d, _, _ = m.generate(ids, max_length=10, top_p=0.9, temperature=1.3, seed=43)
    assert not torch.equal(a, d)


# ----------------------------------------------------------------------------------------------------------
# paged ("block") KV cache — FusedBlockMultiTransformer / append_attention layout (SURVEY §8f rank 1)
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh,kvh,B,block_size,max_blocks,splits", [(32, 8, 9, 64, 12, 0), (8, 2, 40, 64, 5, 1), (28, 4, 3, 128, 6, 3),
                                                                    (4, 1, 2, 32, 9, 2), (8, 2, 40, 64, 5, 0), (28, 4, 3, 128, 6, 0),
                                                                    (4, 1, 2, 32, 9, 0), (32, 8, 64, 64, 18, 0)])
def test_paged_rope_append_and_attention(nh, kvh, B, block_size, max_blocks, splits):
    o = ops()
    d = 128
    rng = np.random.default_rng(nh + B)
    nb = B * max_blocks + 3
    perm = rng.permutation(nb)[: B * max_blocks].astype(np.int32).reshape(B, max_blocks)       # scattered physical blocks
    cap = block_size * max_blocks
    lens = rng.integers(0, cap - 1, size=B).astype(np.int32)
    lens[0], lens[-1] = 0, cap - 1                                        # empty history; cache already full (clamped)
    kc = torch.tensor(rng.standard_normal((nb, kvh, block_size, d)).astype(np.float32)).to(BF16)
    vc = torch.tensor(rng.standard_normal((nb, kvh, block_size, d)).astype(np.float32)).to(BF16)
    for b in range(B):                                                    # blocks past a sequence's need are unallocated
        used = (min(int(lens[b]) + 1, cap) + block_size - 1) // block_size
        perm[b, used:] = -1
    qkv = torch.tensor(rng.standard_normal((B, (nh + 2 * kvh) * d)).astype(np.float32)).to(BF16)
    cos, sin = o.rope_tables(d, cap, 10000.0, DEV)
    kc_d, vc_d, qkv_d = kc.clone().to(DEV), vc.clone().to(DEV), qkv.clone().to(DEV)
    bt, ln = t(perm, torch.int32), t(lens, torch.int32)
    o.decode_rope_append_paged(qkv_d, kc_d, vc_d, bt, cos, sin, ln, nh)
    # RoPE + append: identical bits to the dense kernel writing into a dense cache
    dense = torch.zeros(2, B, kvh, cap, d, dtype=BF16, device=DEV)
    qkv_dense = qkv.clone().to(DEV)
    o.decode_rope_append(qkv_dense, dense, cos, sin, ln, nh, kvh, d)
    assert torch.equal(qkv_d, qkv_dense)
    for b in range(B):
        p = int(lens[b])
        if p >= cap:
            continue
        blk, off = int(perm[b, p // block_size]), p % block_size
        assert torch.equal(kc_d[blk, :, off], dense[0, b, :, p]) and torch.equal(vc_d[blk, :, off], dense[1, b, :, p])
    touched = (kc_d != kc.to(DEV)).any(-1).sum().item()
    assert touched <= B * kvh                                             # nothing else in the pool was written
    out = o.decode_attention_paged(qkv_d, kc_d, vc_d, bt, ln, nh, num_splits=splits).float().cpu().numpy()
    ref = G.paged_decode_attention(qkv_d[:, : nh * d].float().cpu().numpy().reshape(B, nh, d), kc_d.float().cpu().numpy(),
                                   vc_d.float().cpu().numpy(), perm, lens)
    assert np.isfinite(out).all()
    assert np.abs(out - ref).max() / np.abs(ref).max() < 1.5e-2


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_block_attn_generation_matches_dense_cache(model_type):
    """generate() on FusedBlockMultiTransformer (scattered 64-row pages) produces the tokens of the dense-cache path."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import FusedBlockMultiTransformer, LlamaForCausalLMInferenceModel

    cfg = _tiny(model_type)
    w = R.init_weights(cfg, seed=9)
    dense, c = _infer_model(cfg, w)
    paged = LlamaForCausalLMInferenceModel(c, block_attn=True, block_size=64)
    paged.set_state_dict(w)
    assert isinstance(paged.transformer_block, FusedBlockMultiTransformer)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, cfg.vocab_size, (5, 37), generator=g)
    enc = torch.tensor([37, 20, 5, 33, 1], dtype=torch.int32)
    for i in range(5):
        ids[i, enc[i]:] = 0
    a, _, la = dense.generate(ids, seq_len_encoder=enc, max_length=40)
    caches = paged.allocate_caches(5, 37 + 40)
    assert len(caches) == 2 * cfg.num_hidden_layers and caches[0].shape == (5 * 2, cfg.num_key_value_heads, 64, 128)
    assert paged.block_tables.shape == (5, 2) and int(paged.block_tables[0, 0]) == 9        # free_list.pop(): highest id first
    b, _, lb = paged.generate(ids, seq_len_encoder=enc, max_length=40, cache_kvs=caches)
    assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.parametrize("block_attn", [False, True])
def test_generate_edge_cases(block_attn):
    """Batch 1 (split-KV auto policy with mostly empty splits), one-token prompts, max_length 1 and 2 (no graph is built),
    and a cache exactly as long as prompt + max_length; graph and eager runs agree token for token."""
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = _tiny()
    w = R.init_weights(cfg, seed=9)
    w = {k: (v * 4).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    _, c = _infer_model(cfg, w)
    m = LlamaForCausalLMInferenceModel(c, block_attn=block_attn)
    m.set_state_dict(w)
    g = torch.Generator().manual_seed(3)
    one = torch.randint(1, cfg.vocab_size, (1, 1), generator=g)
    for L in (1, 2, 5):
        a, _, _ = m.generate(one, max_length=L)
        b, _, _ = m.generate(one, max_length=L, use_cuda_graph=False, use_pdl=False)
        assert a.shape == (1, L) and torch.equal(a, b) and int(a.min()) >= 0
    ids = torch.randint(1, cfg.vocab_size, (1, 100), generator=g)
    caches = m.allocate_caches(1, 100 + 28)                               # exactly full at the last step (128 = one tile)
    a, _, dec = m.generate(ids, max_length=28, cache_kvs=caches)
    b, _, _ = m.generate(ids, max_length=28, use_cuda_graph=False)
    assert torch.equal(a, b) and int(dec[0]) == 100 + 28 - 2
    ref, margins = G.greedy_generate(ids, w, cfg, 4)
    for tpos in range(4):
        if margins[0, tpos] < 2e-2:
            break
        assert int(a[0, tpos]) == int(ref[0, tpos])
    with pytest.raises(ValueError):
        m.generate(ids, max_length=29, cache_kvs=caches)


def test_full_width_decode_matches_uncached_forward():
    """KV-cache consistency (tests/transformers/llama/test_modeling.py:171-219) at the FULL Llama-3-8B layer width, batch 64:
    prefill logits match the training-path forward, and three decode steps (swapped-operand GEMMs at N = 6144 / 4096 /
    28672, K = 14336; decode attention with 4 query heads per kv head) reproduce the uncached forward of the grown
    sequence within bf16 noise, with identical decisive arg-max."""
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    kw = dict(vocab_size=4096, hidden_size=4096, intermediate_size=14336, num_hidden_layers=1, num_attention_heads=32,
              num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=512)
    cfg = R.RefConfig(**kw)
    w = R.init_weights(cfg, seed=31)
    w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(BF16).float()
    train = T.LlamaForCausalLM(T.LlamaConfig(**kw))
    train.set_state_dict(w)
    for block_attn in (False, True):
        inf = LlamaForCausalLMInferenceModel(T.LlamaConfig(**kw), block_attn=block_attn)
        inf.set_state_dict(w)
        B, S = 64, 130
        g = torch.Generator().manual_seed(32)
        ids = torch.randint(0, cfg.vocab_size, (B, S), generator=g).to(DEV)
        enc = torch.full((B,), S, dtype=torch.int32, device=DEV)
        caches = inf.allocate_caches(B, S + 8)
        lg = inf._prefill(ids, enc, caches)
        full = train.engine.forward_logits(ids)
        # same decoder kernels in the same order; only the 64-row lm_head takes the split-K kernel (fp32 summation order)
        e0 = ((lg.float() - full[:, -1].float()).abs().max() / full[:, -1].float().abs().max()).item()
        assert e0 < 5e-3, e0
        seq = ids
        lens = enc.clone()
        for step in range(3):
            nxt = lg.float().argmax(-1)
            seq = torch.cat([seq, nxt[:, None]], dim=1)
            lg = inf._decode(nxt, lens, caches)
            lens += 1
            ref = train.engine.forward_logits(seq)[:, -1].float()
            err = ((lg.float() - ref).abs().max() / ref.abs().max()).item()
            assert err < 2e-2, (block_attn, step, err)
            top2 = ref.topk(2, dim=-1).values
            decisive = (top2[:, 0] - top2[:, 1]) > 4 * err * ref.abs().max()
            assert bool((lg.float().argmax(-1) == ref.argmax(-1))[decisive].all())
            assert decisive.float().mean().item() >= 0.4        # the check above is not vacuous


def test_generate_beyond_max_position_embeddings_grows_rope_tables():
    """ADVICE r01: the decode kernels index the fp32 cos/sin tables with the running sequence length; a KV cache longer than
    config.max_position_embeddings must not read past them.  generate() grows the tables: a model configured with 128
    positions generates, beyond position 128, the same tokens as one configured with 512."""
    import paddlenlp_b200.transformers as T
    from oracle import llama_ref as R
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    kw = dict(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
              num_key_value_heads=1, rms_norm_eps=1e-5, rope_theta=500000.0)
    cfg = R.RefConfig(max_position_embeddings=512, **kw)
    w = R.init_weights(cfg, seed=3)
    w = {k: (v * 4).to(torch.bfloat16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    prompt = torch.randint(0, 512, (2, 100), generator=torch.Generator().manual_seed(4))
    outs = []
    for mpe in (128, 512):
        m = LlamaForCausalLMInferenceModel(T.LlamaConfig(max_position_embeddings=mpe, **kw))
        m.set_state_dict(w)
        out, _, _ = m.generate(prompt, max_length=60, eos_token_id=-1)
        assert m.transformer_block.rope[0].shape[0] >= 160
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("use_neox", [True, False])
def test_fused_get_rotary_embedding_op(use_neox):
    """fused_get_rotary_embedding (csrc/gpu/fused_get_rope.cu:40-223, called experimental/transformers/llama/modeling.py:799-803)
    vs the numpy restatement.  powf / cosf / sinf are not correctly rounded on either side: one ulp of the inverse frequency
    (2^-23 relative) times the position bounds the angle error, hence the position-proportional tolerance."""
    import numpy as np

    from oracle import generation_ref as G
    from paddlenlp_b200 import ops

    bsz, seq, d, prompt_num, theta = 3, 200, 128, 7, 500000.0
    pos = torch.arange(0, 2048, dtype=torch.int64)[None].repeat(bsz, 1).contiguous()
    pos[1] += 1000                                                     # per-sequence offsets
    ids = torch.zeros(bsz, seq, dtype=torch.int64)
    out = ops.fused_get_rotary_embedding(ids.to(DEV), pos.to(DEV), torch.zeros(d), prompt_num, theta, use_neox).cpu().numpy()
    ref = G.fused_get_rotary_embedding((bsz, seq), pos.numpy(), d, prompt_num, theta, use_neox)
    assert out.shape == (2, bsz, 1, seq, d)
    p = pos[:, prompt_num:prompt_num + seq].numpy().astype(np.float64)[None, :, None, :, None]
    tol = 4e-7 * np.maximum(p, 1.0) + 2e-6
    assert (np.abs(out - ref) <= tol).all(), float(np.abs(out - ref).max())
    if use_neox:                                                       # the layout the Llama / Qwen2 rotate-half kernels expect
        assert np.array_equal(out[..., :d // 2], out[..., d // 2:])
    else:
        assert np.array_equal(out[..., 0::2], out[..., 1::2])
    with pytest.raises(Exception):
        ops.fused_get_rotary_embedding(ids.to(DEV), pos[:, :100].contiguous().to(DEV), torch.zeros(d), prompt_num, theta, use_neox)


def test_step_paddle_matches_oracle_bit_exact():
    """step_paddle (csrc/gpu/step.cu:19-283) on a tight block pool: after every call ALL 21 state tensors equal the oracle's
    (sequence-index order on both sides), through freeing, on-demand allocation, pre-emption and recovery."""
    import numpy as np

    import step_sim as sim
    from oracle import generation_ref as G
    from paddlenlp_b200 import ops

    bs, nb, max_dec = 4, 22, 24
    sim.BLOCK_SIZE_FOR_CHECK[0] = bs
    events = 0
    for seed in range(4):
        st, rng = sim.make_state(seed, block_size=bs, num_blocks=nb, max_dec=max_dec)
        for step in range(50):
            sim.between_steps(st, rng, bs, max_dec)
            dev = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in st.items()}
            ops.step_paddle(*[dev[k] for k in sim.ORDER], block_size=bs, first_token_id=1)
            parked_before = int(st["step_lens"][0])
            G.step_paddle(st, bs, first_token_id=1)
            events += int(st["step_lens"][0]) != parked_before
            for k in sim.ORDER:
                assert np.array_equal(dev[k].cpu().numpy(), st[k]), (seed, step, k, dev[k].cpu().numpy(), st[k])
            sim.check_invariants(st, nb)
    assert events > 0


def test_streaming_token_output():
    """save_output / get_output replacement (csrc/gpu/save_with_output_msg.cc:28-52, get_output.cc, llm_utils.py:753-776): a
    reader thread receives every step's {flag, bsz, tokens} message from the pinned-host ring WHILE generation is running —
    the loop itself never synchronises — and the concatenated messages equal generate()'s return value."""
    import time

    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel, TokenStream

    cfg = T.LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                        num_key_value_heads=1, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=1024)
    m = LlamaForCausalLMInferenceModel(cfg)
    m.init_random(seed=3)
    prompt = torch.randint(0, 512, (5, 16), generator=torch.Generator().manual_seed(2))
    stream = TokenStream(max_bsz=8, num_slots=64)                       # ring much shorter than the generation: slots are reused
    assert stream.get_output(False) == [-2, 0]                          # nothing yet: the reference's "read none" answer
    n_steps = 600
    arrivals = []
    reader = stream.start_reader(on_message=lambda i, msg: arrivals.append(time.time()))
    out, _, _ = m.generate(prompt, max_length=n_steps, eos_token_id=-1, token_stream=stream)
    t_enqueued = time.time()
    reader.join(timeout=60)
    torch.cuda.synchronize()
    assert reader.error is None, reader.error
    msgs = reader.result
    assert len(msgs) == n_steps and all(len(x) == 5 for x in msgs)
    got = torch.tensor(msgs).t()                                        # [bsz, steps]
    assert torch.equal(got, out.cpu())
    # streamed: the first message was on the host long before the last one (it did not wait for the end of the generation)
    assert arrivals[0] < arrivals[-1] - 0.5 * (arrivals[-1] - arrivals[0]) and arrivals[n_steps // 4] < arrivals[-1]
    print(f"[stream] first message {arrivals[0] - t_enqueued:+.3f} s, last {arrivals[-1] - t_enqueued:+.3f} s relative to generate() returning")
    # the finished flag: -1 on the final message only
    stream2 = TokenStream(max_bsz=8, num_slots=1024)
    out2, _, _ = m.generate(prompt, max_length=40, eos_token_id=-1, token_stream=stream2)
    flags = []
    while True:
        msg = stream2.get_output(True)
        flags.append(msg[0])
        if msg[0] == -1:
            break
    assert flags == [1] * 39 + [-1] and stream2.get_output(False) == [-2, 0]
    # a reader that falls a whole ring behind is told so instead of silently reading newer data
    stream3 = TokenStream(max_bsz=8, num_slots=8)
    m.generate(prompt, max_length=40, eos_token_id=-1, token_stream=stream3)
    torch.cuda.synchronize()
    with pytest.raises(Exception):
        stream3.get_output(False)


@pytest.mark.parametrize("block_size", [64, 32])
def test_append_attention_mixed_batch(block_size):
    """append_attention (csrc/gpu/append_attention.cu:428-851): ONE call serves a mixed batch over the paged cache — a fresh prompt,
    a prompt CHUNK on top of a cached prefix (chunked prefill), a decode row, a one-token prompt and an idle slot — with RoPE and
    the cache append inside the op.  Checked against the oracle's full causal attention of every sequence at absolute positions,
    and the appended cache rows against the oracle's rotated k / raw v; two chunked calls equal one whole-prompt call."""
    from paddlenlp_b200 import ops

    nh, kvh, d = 4, 2, 128
    ld = (nh + 2 * kvh) * d
    B, max_len = 5, 640
    mb = max_len // block_size
    num_blocks = B * mb + 3
    g = torch.Generator().manual_seed(7)
    perm = torch.randperm(num_blocks, generator=g)[: B * mb].to(torch.int32)          # scattered physical pages
    block_tables = perm.view(B, mb).contiguous().to(DEV)
    cos, sin = ops.rope_tables(d, max_len, 10000.0, DEV)
    rcos, rsin = R.rope_tables(d, max_len, 10000.0)

    totals = [300, 350, 78, 1, 0]                      # final lengths of the five sequences
    seqs = [torch.randn(L, ld, generator=g).to(torch.bfloat16) for L in totals]       # pre-RoPE packed projections

    def oracle(seq):
        L = seq.shape[0]
        x = seq.float()
        q = x[:, : nh * d].view(1, L, nh, d)
        k = x[:, nh * d:(nh + kvh) * d].view(1, L, kvh, d)
        v = x[:, (nh + kvh) * d:].view(1, L, kvh, d)
        qr, kr = R.apply_rope(q, rcos, rsin, "bf16"), R.apply_rope(k, rcos, rsin, "bf16")
        return R.attention(qr, kr, v, "fp32")[0], kr[0], v[0]          # [L, nh*d], [L, kvh, d], [L, kvh, d]

    def call(chunks, key_cache, value_cache):
        """chunks: per sequence (start, stop) rows of its projection to append in this call (stop == start: idle)."""
        rows = [seqs[b][s:e] for b, (s, e) in enumerate(chunks)]
        n = [e - s for s, e in chunks]
        qkv = torch.cat([r for r in rows if r.shape[0]], 0).to(DEV).contiguous()
        cu = torch.tensor([0] + list(torch.tensor(n).cumsum(0)), dtype=torch.int32, device=DEV)
        enc = torch.tensor([ni if (ni > 1 or s == 0) and ni > 0 else 0 for ni, (s, e) in zip(n, chunks)], dtype=torch.int32, device=DEV)
        dec = torch.tensor([s for s, e in chunks], dtype=torch.int32, device=DEV)
        this = torch.tensor(n, dtype=torch.int32, device=DEV)
        out = ops.append_attention(qkv, key_cache, value_cache, enc, dec, this, cu, block_tables, cos, sin, nh, max_q_len=max(n))
        return out.float().cpu(), cu.cpu().tolist()

    def caches():
        return (torch.zeros(num_blocks, kvh, block_size, d, dtype=torch.bfloat16, device=DEV),
                torch.zeros(num_blocks, kvh, block_size, d, dtype=torch.bfloat16, device=DEV))

    kc, vc = caches()
    # call 1: build the cached prefixes (seq 1: first 150 rows, seq 2: first 77 rows), seq 0 / 3 / 4 idle
    call([(0, 0), (0, 150), (0, 77), (0, 0), (0, 0)], kc, vc)
    # call 2: the mixed batch
    out, cu = call([(0, 300), (150, 350), (77, 78), (0, 1), (0, 0)], kc, vc)
    refs = [oracle(s) if s.shape[0] else None for s in seqs]
    starts = [0, 150, 77, 0, 0]
    for b in range(4):
        ref_out = refs[b][0][starts[b]:]
        got = out[cu[b]:cu[b + 1]]
        e = ((got - ref_out).abs().max() / ref_out.abs().max()).item()
        assert e < 2e-2, (b, e)
    # the appended cache rows: rotated k and raw v at every position of every sequence
    kc_c, vc_c, bt = kc.float().cpu(), vc.float().cpu(), block_tables.cpu()
    for b in range(4):
        _, kr, v = refs[b]
        for pos in (0, totals[b] // 2, totals[b] - 1):
            phys, off = int(bt[b, pos // block_size]), pos % block_size
            assert (kc_c[phys, :, off] - kr[pos]).abs().max() <= 2 ** -7 * kr[pos].abs().max(), (b, pos)   # 1 bf16 ulp (fp32 FMA order)
            assert torch.equal(vc_c[phys, :, off], v[pos]), (b, pos)
    # chunked prefill == whole prompt: sequence 1 appended in one call gives the rows of the two-call run
    kc2, vc2 = caches()
    whole, cu2 = call([(0, 0), (0, 350), (0, 0), (0, 0), (0, 0)], kc2, vc2)
    two_step = out[cu[1]:cu[2]]
    one_step = whole[cu2[1]:cu2[2]][150:]
    assert ((two_step - one_step).abs().max() / one_step.abs().max()).item() < 1e-2


def test_generate_with_append_attention_equals_block_attention():
    """`--append_attn` (FusedBlockMultiTransformer.compute_attn -> append_attention, fused_transformer_layers.py:2215-2262):
    generation through the unified op (prompt rows and decode rows through one entry point, RoPE and cache append inside it)
    produces the tokens of the block-attention path, with right-padded prompts of different lengths."""
    import paddlenlp_b200.transformers as T
    from oracle import llama_ref as R
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    kw = dict(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
              num_key_value_heads=1, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=512)
    w = R.init_weights(R.RefConfig(**kw), seed=5)
    w = {k: (v * 4).to(torch.bfloat16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}
    prompt = torch.randint(1, 512, (3, 140), generator=torch.Generator().manual_seed(6))
    lens = torch.tensor([140, 77, 129], dtype=torch.int32)
    outs = []
    for append in (False, True):
        m = LlamaForCausalLMInferenceModel(T.LlamaConfig(**kw), block_attn=True, append_attn=append)
        m.set_state_dict(w)
        out, _, _ = m.generate(prompt, seq_len_encoder=lens, max_length=24, eos_token_id=-1)
        outs.append(out.cpu())
    agree = (outs[0] == outs[1]).float().mean().item()
    # same math, different kernels (prefill: page-gathered K/V vs dense strided views; rotation before vs inside the op): the greedy
    # tokens agree except where two logits tie within bf16 noise
    assert agree > 0.9, (agree, outs[0][0].tolist(), outs[1][0].tolist())
    assert torch.equal(outs[0][:, :4], outs[1][:, :4])
