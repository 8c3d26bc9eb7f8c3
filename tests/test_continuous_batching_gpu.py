"""Continuous batching on the paged KV cache (LlamaForCausalLMInferenceModel.continuous_generate and the retire_admit kernel):
per-request greedy tokens against the uncached oracle, pre-emption and recovery on a tight pool, graph against eager replay,
block accounting, sampling, argument errors, and the kernel bit-exact against its restatement."""
import math

import numpy as np
import pytest
import torch

import continuous_sim as sim
from oracle import generation_ref as G
from oracle import llama_ref as R
from oracle import retire_admit_ref as RA

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
MARGIN = 2e-2


def _tiny(model_type="llama"):
    return R.RefConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                       num_key_value_heads=1, rope_theta=10000.0, qkv_bias=(model_type == "qwen2"), model_type=model_type,
                       max_position_embeddings=128, rms_norm_eps=1e-5)


def _weights(cfg):
    w = R.init_weights(cfg, seed=9)
    # x4: decisive top-1/top-2 margins (the 0.02 init gives near-flat logits whose arg-max is bf16 noise)
    return {k: (v * 4).to(BF16).float() if k.endswith("weight") and "norm" not in k else v for k, v in w.items()}


def _model(cfg, w, block_size):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    c = T.Qwen2Config(**kw) if cfg.model_type == "qwen2" else T.LlamaConfig(**kw)
    m = LlamaForCausalLMInferenceModel(c, block_attn=True, append_attn=True, block_size=block_size)
    m.set_state_dict(w)
    return m


def _requests(n=11, seed=3, vocab=512, prompt=(1, 70), new=(3, 40)):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        p = int(torch.randint(prompt[0], prompt[1] + 1, (1,), generator=g))
        m = int(torch.randint(new[0], new[1] + 1, (1,), generator=g))
        out.append((torch.randint(1, vocab, (p,), generator=g), m))
    return out


_ORACLE = {}


def _oracle(model_type, reqs, key):
    """Greedy tokens and top-1/top-2 margins of every request decoded alone by the uncached oracle (cached per model and
    request set)."""
    if (model_type, key) not in _ORACLE:
        cfg = _tiny(model_type)
        w = _weights(cfg)
        _ORACLE[model_type, key] = [G.greedy_generate(ids[None], w, cfg, max_new=m) for ids, m in reqs]
    return _ORACLE[model_type, key]


def _compare(outs, reqs, ref, eos=None):
    """Each request's tokens equal the oracle's up to its first near-tie; an EOS the oracle emits ends the request there."""
    compared = 0
    for r, ((ids, m), out) in enumerate(zip(reqs, outs)):
        want, margins = ref[r][0][0], ref[r][1][0]
        assert out.dtype == torch.int64 and 1 <= out.numel() <= m
        for t in range(m):
            if margins[t] < MARGIN:
                break
            assert t < out.numel() and int(out[t]) == int(want[t]), (r, t, out.tolist(), want.tolist())
            compared += 1
            if eos is not None and int(want[t]) == eos:
                assert out.numel() == t + 1, (r, t, out.tolist())
                break
        else:
            assert out.numel() == m or (eos is not None and int(out[-1]) == eos), (r, out.tolist())
    return compared


def _pages(reqs, bs):
    return max(max(math.ceil((ids.numel() + m) / bs), math.ceil(ids.numel() / bs) + 1) for ids, m in reqs)


def _check_blocks(m, stats, num_blocks):
    assert stats["free_blocks_at_exit"] == num_blocks
    assert bool((m.last_block_tables == -1).all())


@pytest.mark.parametrize("block_size", [32, 64])
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tokens_per_request_match_the_oracle(model_type, block_size):
    cfg = _tiny(model_type)
    m = _model(cfg, _weights(cfg), block_size)
    reqs = _requests()
    ref = _oracle(model_type, reqs, "mixed")
    nb = 4 * 11 * _pages(reqs, block_size)
    outs, stats = m.continuous_generate(reqs, max_batch_size=4, num_blocks=nb)
    assert len(outs) == len(reqs)
    assert _compare(outs, reqs, ref) >= 20
    assert stats["preemptions"] == 0 and stats["mixed_steps"] >= 2            # later requests were admitted into freed slots
    _check_blocks(m, stats, nb)
    # EOS: a token a request emits early (decisively) ends it there, and the queue moves on
    r, t = next((r, t) for r in range(len(reqs)) for t in range(1, reqs[r][1] - 1)
                if ref[r][1][0][:t + 1].min() >= MARGIN and int(ref[r][0][0][t]) not in ref[r][0][0][:t].tolist())
    eos = int(ref[r][0][0][t])
    outs2, stats2 = m.continuous_generate(reqs, max_batch_size=4, num_blocks=nb, eos_token_id=eos)
    assert outs2[r].numel() == t + 1 < reqs[r][1] and int(outs2[r][-1]) == eos
    assert _compare(outs2, reqs, ref, eos=eos) >= 20
    assert stats2["mixed_steps"] >= 2
    _check_blocks(m, stats2, nb)


# outputs of two to three 32-token pages on top of one-page prompts: with one spare page per resident slot, two residents
# growing at once outrun a pool one page above the largest request's need
TIGHT = dict(prompt=(1, 30), new=(60, 96))


def _tight(model_type="llama", block_size=32, use_cuda_graph=True):
    cfg = _tiny(model_type)
    m = _model(cfg, _weights(cfg), block_size)
    reqs = _requests(**TIGHT)
    nb = _pages(reqs, block_size) + 1
    outs, stats = m.continuous_generate(reqs, max_batch_size=4, num_blocks=nb, use_cuda_graph=use_cuda_graph)
    _check_blocks(m, stats, nb)
    return reqs, outs, stats


def test_tight_pool_preempts_recovers_and_graphs_equal_eager():
    reqs, outs, stats = _tight()
    assert stats["preemptions"] > 0 and stats["recoveries"] > 0, stats
    assert stats["peak_blocks_in_use"] <= _pages(reqs, 32) + 1
    assert _compare(outs, reqs, _oracle("llama", reqs, "tight")) >= 20
    _, eager, stats_e = _tight(use_cuda_graph=False)
    assert {k: v for k, v in stats_e.items() if k != "decode_step_ms"} == {k: v for k, v in stats.items() if k != "decode_step_ms"}
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)


def test_top_p_sampling_is_reproducible():
    cfg = _tiny()
    m = _model(cfg, _weights(cfg), 64)
    reqs = _requests(n=7, seed=5)
    runs = [m.continuous_generate(reqs, max_batch_size=3, num_blocks=64, top_p=0.9, temperature=1.3, seed=42)[0]
            for _ in range(2)]
    for a, b, (_, mx) in zip(*runs, reqs):
        assert torch.equal(a, b) and a.numel() == mx
        assert int(a.min()) >= 0 and int(a.max()) < cfg.vocab_size


def test_argument_errors():
    cfg = _tiny()
    m = _model(cfg, _weights(cfg), 32)
    ok = (torch.arange(1, 10), 4)
    for bad, needle in [((torch.zeros(0, dtype=torch.int64), 4), "empty prompt"), ((torch.arange(1, 5), 0), "max_length"),
                        ((torch.arange(1, 100), 40), "more than num_blocks")]:
        with pytest.raises(ValueError, match=needle):
            m.continuous_generate([ok, bad], max_batch_size=2, num_blocks=4)
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    plain = LlamaForCausalLMInferenceModel(T.LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=688,
                                                         num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1),
                                           block_attn=True)
    with pytest.raises(ValueError, match="append_attn"):
        plain.continuous_generate([ok], max_batch_size=1, num_blocks=4)


def test_retire_admit_matches_restatement_bit_exact():
    """step_paddle + retire_admit on a tight pool through whole queues: after every call every field, the outputs and the
    header equal the restatement's, and every block is owned exactly once."""
    from paddlenlp_b200 import ops

    bs = 4
    events = np.zeros(3, int)
    for seed in range(6):
        st, rng, nb, _ = sim.make_queue_state(seed, block_size=bs)
        header = sim.new_header()
        max_prompt = int(np.diff(st["prompt_offsets"]).max())
        max_seq = int((np.diff(st["prompt_offsets"]) + st["req_max_dec_len"]).max())
        emitted, steps = {}, 0
        while True:
            dev = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in st.items()}
            hdev = torch.from_numpy(header.copy()).pin_memory()
            if steps:
                ops.step_paddle(*[dev[k] for k in sim.STEP_ORDER], block_size=bs)
                G.step_paddle(st, bs)
            ops.retire_admit(dev, hdev, bs, max_prompt, max_seq)
            RA.retire_admit(st, header, bs)
            torch.cuda.synchronize()
            for k in st:
                assert np.array_equal(dev[k].cpu().numpy(), st[k]), (seed, steps, k, dev[k].cpu().numpy(), st[k])
            assert np.array_equal(hdev.numpy(), header), (seed, steps, hdev.numpy(), header)
            sim.check_blocks(st, nb)
            events += (header[RA.ADMITTED] > 0, header[RA.RETIRED] > 0, header[RA.PARKED] > 0)
            if header[RA.DONE]:
                break
            steps += 1
            assert steps < 5000
            sim.model_step(st, rng, emitted)
    assert (events > 0).all(), events
    assert header[RA.RECOVERIES] > 0 or events[2] > 0


def test_graph_replay_after_a_larger_eager_step():
    """A decode graph captured at one token_num, then an eager mixed step with more rows (<= 128: the split-K GEMMs) when two
    long prompts are admitted, then replays of that graph: every split-K call of the whole run uses one workspace address (a
    buffer regrown under a captured graph would leave the graph writing to freed memory), and the graph run equals the
    eager run token for token and the oracle up to its first near-tie."""
    import contextlib

    from paddlenlp_b200 import _lib, ops

    cfg = _tiny()
    m = _model(cfg, _weights(cfg), 64)
    g = torch.Generator().manual_seed(11)
    # slots 0-1 retire after 6 tokens while slots 2-3 decode on (token_num 4, then 2 + the prompts, then 4 again)
    lens = [(3, 6), (3, 6), (3, 24), (3, 24), (58, 12), (58, 12)]
    reqs = [(torch.randint(1, cfg.vocab_size, (p,), generator=g), n) for p, n in lens]
    ops._workspaces.pop((torch.empty(0, device=DEV).device, "splitk"), None)     # start from no buffer at all
    addrs = set()

    def hook(name, args):
        if name == "b200_gemm_bf16_splitk":
            addrs.add(args[4].value)
        return contextlib.nullcontext()

    runs = []
    for graph in (True, False):
        _lib.call_hook = hook
        try:
            outs, stats = m.continuous_generate(reqs, max_batch_size=4, num_blocks=64, use_cuda_graph=graph)
        finally:
            _lib.call_hook = None
        runs.append(outs)
        assert stats["mixed_steps"] >= 2 and stats["decode_steps"] > 10, stats
        _check_blocks(m, stats, 64)
    assert len(addrs) == 1, addrs
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    assert _compare(runs[0], reqs, _oracle("llama", reqs, "regrow")) >= 10
