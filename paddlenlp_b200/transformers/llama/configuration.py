"""LlamaConfig — same constructor surface and defaults as paddlenlp/transformers/llama/configuration.py:68-209."""
from ..configuration_utils import PretrainedConfig


class LlamaConfig(PretrainedConfig):
    model_type = "llama"
    attribute_map = {"n_positions": "max_position_embeddings", "n_embd": "hidden_size", "n_layer": "num_hidden_layers",
                     "n_head": "num_attention_heads", "n_inner": "intermediate_size"}

    def __init__(self, vocab_size=32000, hidden_size=4096, intermediate_size=11008, max_position_embeddings=2048,
                 seq_length=2048, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=None,
                 initializer_range=0.02, rms_norm_eps=1e-6, rope_theta=10000.0, use_cache=True,
                 fuse_attention_qkv=False, fuse_attention_ffn=False, pad_token_id=0, bos_token_id=1, eos_token_id=2,
                 tie_word_embeddings=False, alibi=False, rope_scaling_factor=1.0, rope_scaling_type=None, rope_scaling=None,
                 **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.max_position_embeddings = max_position_embeddings
        self.seq_length = seq_length
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.num_key_value_heads = num_attention_heads if num_key_value_heads is None else num_key_value_heads
        self.initializer_range = initializer_range
        self.rms_norm_eps = rms_norm_eps
        self.rope_theta = rope_theta
        self.use_cache = use_cache
        self.fuse_attention_qkv = fuse_attention_qkv
        self.fuse_attention_ffn = fuse_attention_ffn
        self.alibi = alibi
        self.rope_scaling_factor = rope_scaling_factor
        self.rope_scaling_type = rope_scaling_type
        self.rope_scaling = rope_scaling                       # {"rope_type": "llama3", ...} (HF Llama-3.1 config.json)
        if rope_scaling_type not in (None, "linear", "ntk", "dynamic_ntk"):
            raise ValueError(f"Unknown RoPE scaling type {rope_scaling_type}")      # llama/modeling.py:864
        if alibi:
            raise NotImplementedError("alibi attention bias is outside the hot path this build covers")
        super().__init__(pad_token_id=pad_token_id, bos_token_id=bos_token_id, eos_token_id=eos_token_id,
                         tie_word_embeddings=tie_word_embeddings, **kwargs)

    @property
    def rope(self):
        return not self.alibi

    def rope_scaling_spec(self):
        """The rotary variant `_init_rope` would pick (llama/modeling.py:821-864) as a dict for ops.rope_tables, or None."""
        rs = getattr(self, "rope_scaling", None)
        if rs is not None and rs.get("rope_type", None) == "llama3":
            return dict(rs)
        t = getattr(self, "rope_scaling_type", None)
        if t is None:
            return None
        return {"type": t, "factor": float(self.rope_scaling_factor)}

    # public presets used by bench / tests (hyper-parameters from the public model cards, SURVEY.md §8)
    @classmethod
    def llama3_2_3b(cls, **kw):
        """Llama-3.2-3B shapes (head_dim 128, GQA 24/8).  The released model ties its input and output embeddings; the preset
        keeps a separate lm_head by default (the benchmarked model).  Pass `tie_word_embeddings=True` for the released layout:
        the logits then read the embedding matrix, and its V x h parameters, gradients and optimizer state exist once."""
        base = dict(vocab_size=128256, hidden_size=3072, intermediate_size=8192, num_hidden_layers=28,
                    num_attention_heads=24, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0,
                    max_position_embeddings=8192, seq_length=4096, bos_token_id=128000, eos_token_id=128001)
        base.update(kw)
        return cls(**base)

    @classmethod
    def llama3_8b(cls, **kw):
        base = dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                    num_attention_heads=32, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0,
                    max_position_embeddings=8192, seq_length=4096, bos_token_id=128000, eos_token_id=128001)
        base.update(kw)
        return cls(**base)
