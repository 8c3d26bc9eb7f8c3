"""Tied input / output embeddings (config.tie_word_embeddings) without a GPU: configs, the tied oracle pinned to the HF
golden fixtures, HF <-> Paddle conversion, and the engine's flat layout, init and checkpoint files on a CPU container.
The tied oracle (tests/tied_oracle.py) is oracle/llama_ref.py with the head bound to E^T."""
import json
import os

import pytest
import torch

from oracle import llama_ref as R
from paddlenlp_b200.transformers import conversion_utils as cu
from tied_oracle import embed_key, load_golden, tied_forward, tied_loss_and_grads


# ------------------------------------------------------------------------------------------------------------------
# configs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_config_accepts_and_round_trips_tying(tmp_path, model_type):
    import paddlenlp_b200.transformers as T

    C = T.LlamaConfig if model_type == "llama" else T.Qwen2Config
    c = C(vocab_size=64, hidden_size=256, intermediate_size=64, num_hidden_layers=1, num_attention_heads=2,
          num_key_value_heads=1, tie_word_embeddings=True)
    assert c.tie_word_embeddings is True
    assert c.to_dict()["tie_word_embeddings"] is True
    assert C.from_dict(c.to_dict()).tie_word_embeddings is True
    c.save_pretrained(str(tmp_path))
    assert json.load(open(tmp_path / "config.json"))["tie_word_embeddings"] is True
    assert C.from_pretrained(str(tmp_path)).tie_word_embeddings is True
    assert C.from_dict({**c.to_dict(), "tie_word_embeddings": False}).tie_word_embeddings is False
    # the presets stay untied unless asked
    preset = C.llama3_2_3b if model_type == "llama" else C.qwen2_1_5b
    assert preset().tie_word_embeddings is False
    assert preset(tie_word_embeddings=True).tie_word_embeddings is True
    assert "tie_word_embeddings=True" in preset.__doc__


# ------------------------------------------------------------------------------------------------------------------
# the tied oracle against HF
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["llama_tiny_tied.pt", "qwen2_tiny_tied.pt"])
def test_tied_oracle_matches_hf_golden(name):
    d, cfg, w = load_golden(name)
    assert "lm_head.weight" not in d["weights"] and "lm_head.weight" not in d["grads_fp32"]
    logits = tied_forward(d["input_ids"], w, cfg, mode="fp32")
    assert torch.allclose(logits, d["hf_logits_fp32"], rtol=1e-4, atol=2e-5)
    loss, _, grads = tied_loss_and_grads(d["input_ids"], d["labels"], w, cfg, mode="fp32")
    assert abs(float(loss) - float(d["loss_fp32"])) < 1e-5
    assert set(grads) == set(d["grads_fp32"])
    for k, g in d["grads_fp32"].items():
        assert torch.allclose(grads[k], g, rtol=1e-3, atol=1e-6), k
    # the embedding gradient includes the head term: the lookup's scatter alone is far from it
    E = embed_key(cfg)
    wu = {**w, "lm_head.weight": w[E].t().clone()}
    _, _, gu = R.loss_and_grads(d["input_ids"], d["labels"], wu, cfg, mode="fp32")
    assert not torch.allclose(gu[E], d["grads_fp32"][E], rtol=1e-2, atol=1e-4)
    assert torch.allclose(gu[E] + gu["lm_head.weight"].t(), d["grads_fp32"][E], rtol=1e-3, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------
# HF <-> Paddle conversion (llama/modeling.py:1270-1271: no lm_head mapping when tied)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tied_hf_conversion_both_ways(model_type):
    cfg = R.RefConfig(vocab_size=64, hidden_size=32, intermediate_size=48, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, qkv_bias=(model_type == "qwen2"), model_type=model_type)
    w = R.init_weights(cfg, seed=5)
    head = w.pop("lm_head.weight")
    hf = R.to_hf_state_dict(w, cfg)
    mine = cu.paddle_to_hf_state_dict(w, model_type, tie_word_embeddings=True)
    assert "lm_head.weight" not in mine and set(mine) == set(hf) and all(torch.equal(mine[k], hf[k]) for k in hf)
    # a tied state dict that still carries a head maps to the same HF dict
    assert set(cu.paddle_to_hf_state_dict({**w, "lm_head.weight": head}, model_type, tie_word_embeddings=True)) == set(hf)
    back = cu.hf_to_paddle_state_dict(hf, model_type, tie_word_embeddings=True)
    assert set(back) == set(w) and all(torch.equal(back[k], w[k]) for k in w)
    stray = cu.hf_to_paddle_state_dict({**hf, "lm_head.weight": head.t()}, model_type, tie_word_embeddings=True)
    assert set(stray) == set(w)
    # untied configs keep today's mapping: a tied HF checkpoint gets a separate head equal to E^T
    untied = cu.hf_to_paddle_state_dict(hf, model_type)
    assert torch.equal(untied["lm_head.weight"], w[f"{model_type}.embed_tokens.weight"].t())


# ------------------------------------------------------------------------------------------------------------------
# the engine's layout, init and checkpoint files (CPU container: no kernel runs)
# ------------------------------------------------------------------------------------------------------------------
def _tiny(model_type, tied, **kw):
    import paddlenlp_b200.transformers as T

    C, M = (T.LlamaConfig, T.LlamaForCausalLM) if model_type == "llama" else (T.Qwen2Config, T.Qwen2ForCausalLM)
    c = C(vocab_size=64, hidden_size=256, intermediate_size=72, num_hidden_layers=3, num_attention_heads=2,
          num_key_value_heads=1, max_position_embeddings=64, tie_word_embeddings=tied, **kw)
    return M(c, device="cpu")


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tied_layout_has_no_head(model_type):
    mt, mu = _tiny(model_type, True), _tiny(model_type, False)
    et, eu = mt.engine, mu.engine
    assert "head" not in et._offsets and "head" in eu._offsets
    V, h = et.V, et.h
    assert et.num_parameters() == eu.num_parameters() - V * h
    assert eu.numel - et.numel == V * h                               # V * h is a multiple of 8: no padding differs
    assert "lm_head.weight" not in mt.state_dict() and "lm_head.weight" not in dict(mt.named_parameters())
    assert set(mu.state_dict()) - set(mt.state_dict()) == {"lm_head.weight"}
    # same order of every other tensor; the embedding stays first in the decayed segment
    assert et._offsets["embed"][0] == 0 and et.decay_end == eu.decay_end - V * h
    # the ranges the tied backward reports (layers L-1 .. 0, embedding, vector tail) tile the buffer exactly once
    rs = [et._range(f"l{i}.qkv_w", f"l{i}.down_w") for i in range(et.L)] + [et._range("embed", "embed"),
                                                                           (et.decay_end, et.numel)]
    pos = 0
    for lo, hi in sorted(rs):
        assert lo == pos and hi > lo
        pos = hi
    assert pos == et.numel


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tied_host_init_skips_the_head_draw(model_type):
    """Host-mode init draws in the reference's parameter order; a tied model has no lm_head, which is drawn last, so
    every tensor equals the untied model's."""
    mt, mu = _tiny(model_type, True), _tiny(model_type, False)
    st, su = mt.state_dict(), mu.state_dict()
    assert all(torch.equal(st[k], su[k]) for k in st)


@pytest.mark.parametrize("hf_format", [False, True])
def test_tied_save_and_from_pretrained(tmp_path, hf_format):
    import paddlenlp_b200.transformers as T
    from safetensors.torch import load_file, save_file

    m = _tiny("qwen2", True)
    with torch.no_grad():
        m.engine.flat_params.normal_()
    m.save_pretrained(str(tmp_path), max_shard_size="200KB", hf_format=hf_format)
    idx = json.load(open(tmp_path / cu.SAFE_WEIGHTS_INDEX_NAME))["weight_map"]
    assert "lm_head.weight" not in idx
    assert json.load(open(tmp_path / "config.json"))["tie_word_embeddings"] is True
    m2 = T.Qwen2ForCausalLM.from_pretrained(str(tmp_path), device="cpu")
    assert m2.engine.tied and torch.equal(m2.engine.flat_params, m.engine.flat_params)
    # a stray lm_head.weight (e.g. written by a tool that unties on save) is accepted and ignored
    shard = sorted(set(idx.values()))[0]
    t = load_file(str(tmp_path / shard))
    t["lm_head.weight"] = torch.randn(m.engine.V, m.engine.h) if hf_format else torch.randn(m.engine.h, m.engine.V)
    save_file(t, str(tmp_path / shard))
    with open(tmp_path / cu.SAFE_WEIGHTS_INDEX_NAME, "w") as f:
        json.dump({"metadata": {}, "weight_map": {**idx, "lm_head.weight": shard}}, f)
    m3 = T.Qwen2ForCausalLM.from_pretrained(str(tmp_path), device="cpu")
    assert torch.equal(m3.engine.flat_params, m.engine.flat_params)
    # set_state_dict takes a state dict with or without the head
    m4 = _tiny("qwen2", True)
    m4.set_state_dict({**m.state_dict(), "lm_head.weight": torch.zeros(m.engine.h, m.engine.V)})
    assert torch.equal(m4.engine.flat_params, m.engine.flat_params)
    # an untied model still requires its head
    os.remove(tmp_path / cu.SAFE_WEIGHTS_INDEX_NAME)
    for f in os.listdir(tmp_path):
        if f.endswith(".safetensors"):
            os.remove(tmp_path / f)
    m.save_pretrained(str(tmp_path), hf_format=hf_format)
    untied = T.Qwen2Config.from_pretrained(str(tmp_path), tie_word_embeddings=False)
    with pytest.raises(KeyError):
        T.Qwen2ForCausalLM.from_pretrained(str(tmp_path), config=untied, device="cpu", convert_from_hf=hf_format)
