"""head_dim 64 (Llama-3.2-1B, Qwen2-0.5B, TinyLlama) without a GPU: the presets, the configuration checks, and the C-ABI
argument checks that refuse every other head_dim before any CUDA call."""
from ctypes import c_void_p

import pytest
import torch


def test_fused_transformer_config_accepts_head_dim_64_and_refuses_others():
    from paddlenlp_b200.experimental.transformers.fused_transformer_layers import FusedMultiTransformerConfig

    for h, nh in ((2048, 32), (896, 14), (4096, 32)):                     # head_dim 64, 64, 128
        FusedMultiTransformerConfig(embed_dim=h, num_heads=nh, dim_feedforward=4 * h, kv_num_heads=2, num_layers=1)
    for h, nh in ((1280, 16), (3072, 32)):                                  # head_dim 80, 96
        with pytest.raises(NotImplementedError, match="64 and 128"):
            FusedMultiTransformerConfig(embed_dim=h, num_heads=nh, dim_feedforward=4 * h, kv_num_heads=2, num_layers=1)


def test_fusion_flash_attention_refuses_head_dim_96():
    from paddlenlp_b200.transformers.llama import fusion_ops as F

    q = torch.zeros(1, 4, 2, 96, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="head_dim 96"):
        F.fusion_flash_attention(q, None, q, q, None, False)


def test_presets_carry_the_public_shapes():
    import paddlenlp_b200.transformers as T

    c = T.LlamaConfig.llama3_2_1b()
    assert (c.hidden_size, c.num_attention_heads, c.num_key_value_heads, c.intermediate_size, c.num_hidden_layers,
            c.vocab_size) == (2048, 32, 8, 8192, 16, 128256)
    assert c.hidden_size // c.num_attention_heads == 64 and c.tie_word_embeddings
    assert (c.rms_norm_eps, c.rope_theta, c.bos_token_id, c.eos_token_id) == (1e-5, 500000.0, 128000, 128001)
    assert not T.LlamaConfig.llama3_2_1b(tie_word_embeddings=False).tie_word_embeddings
    q = T.Qwen2Config.qwen2_0_5b()
    assert (q.hidden_size, q.num_attention_heads, q.num_key_value_heads, q.intermediate_size, q.num_hidden_layers,
            q.vocab_size) == (896, 14, 2, 4864, 24, 151936)
    assert q.hidden_size // q.num_attention_heads == 64 and q.tie_word_embeddings
    assert (q.rms_norm_eps, q.rope_theta) == (1e-6, 1000000.0)


# Any non-null address: the argument checks return before a pointer is dereferenced or a CUDA call is made.
P = c_void_p(1 << 20)


@pytest.mark.parametrize("name,args", [
    ("b200_fa_fwd", (P, P, P, P, P, 1, 64, 4, 2, 96, 8 * 96, 8 * 96, 8 * 96, 4 * 96, 0.1, None)),
    ("b200_fa_bwd", (P, P, P, P, P, P, P, P, P, P, 1, 64, 4, 2, 96) + (8 * 96,) * 8 + (0.1, None)),
    ("b200_decode_attention", (P, P, P, P, P, 2, 4, 2, 96, 64, 8 * 96, 0.1, 1, None)),
    ("b200_decode_attention_tc", (P, P, P, P, P, 2, 4, 2, 96, 64, 8 * 96, 0.1, 1, None)),
    ("b200_decode_attention_paged", (P, P, P, P, P, P, P, 2, 4, 2, 96, 8, 64, 4, 8 * 96, 0.1, 1, None)),
])
def test_c_abi_refuses_head_dim_96(name, args):
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    rc = getattr(lib, name)(*args)
    assert rc < 0, (name, rc)
    msg = lib.b200_last_error().decode()
    assert "head_dim must be 64 or 128 (got 96)" in msg, msg
