"""Qwen2Config — constructor surface of paddlenlp/transformers/qwen2/configuration.py."""
from ..configuration_utils import PretrainedConfig


class Qwen2Config(PretrainedConfig):
    model_type = "qwen2"

    def __init__(self, vocab_size=151936, hidden_size=4096, intermediate_size=22016, num_hidden_layers=32,
                 num_attention_heads=32, num_key_value_heads=32, hidden_act="silu", max_position_embeddings=32768,
                 seq_length=32768, initializer_range=0.02, rms_norm_eps=1e-6, use_cache=True, tie_word_embeddings=False,
                 rope_theta=10000.0, pad_token_id=0, bos_token_id=151643, eos_token_id=151643, use_sliding_window=False,
                 sliding_window=4096, max_window_layers=28, attention_dropout=0.0, **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.num_key_value_heads = num_attention_heads if num_key_value_heads is None else num_key_value_heads
        self.hidden_act = hidden_act
        self.max_position_embeddings = max_position_embeddings
        self.seq_length = seq_length
        self.initializer_range = initializer_range
        self.rms_norm_eps = rms_norm_eps
        self.use_cache = use_cache
        self.rope_theta = rope_theta
        self.use_sliding_window = use_sliding_window
        self.sliding_window = sliding_window
        self.max_window_layers = max_window_layers
        self.attention_dropout = attention_dropout
        if use_sliding_window:
            raise NotImplementedError("sliding-window attention is outside the hot path this build covers")
        super().__init__(pad_token_id=pad_token_id, bos_token_id=bos_token_id, eos_token_id=eos_token_id,
                         tie_word_embeddings=tie_word_embeddings, **kwargs)

    @classmethod
    def qwen2_1_5b(cls, **kw):
        """Qwen2-1.5B shapes (head_dim 128, GQA 12/2).  The released model ties its input and output embeddings; the preset
        keeps a separate lm_head by default (the benchmarked model: the same shapes and FLOPs, 0.23 G more parameters).  Pass
        `tie_word_embeddings=True` for the released layout."""
        base = dict(vocab_size=151936, hidden_size=1536, intermediate_size=8960, num_hidden_layers=28,
                    num_attention_heads=12, num_key_value_heads=2, rms_norm_eps=1e-6, rope_theta=1000000.0,
                    max_position_embeddings=32768, seq_length=2048)
        base.update(kw)
        return cls(**base)

    @classmethod
    def qwen2_0_5b(cls, **kw):
        """Qwen2-0.5B / Qwen2.5-0.5B shapes (head_dim 64, GQA 14/2).  Tied input and output embeddings by default, the released
        layout (no benchmark uses this preset); pass `tie_word_embeddings=False` for a separate lm_head."""
        base = dict(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                    num_attention_heads=14, num_key_value_heads=2, rms_norm_eps=1e-6, rope_theta=1000000.0,
                    max_position_embeddings=32768, seq_length=2048, tie_word_embeddings=True)
        base.update(kw)
        return cls(**base)

    @classmethod
    def qwen2_7b(cls, **kw):
        base = dict(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                    num_attention_heads=28, num_key_value_heads=4, rms_norm_eps=1e-6, rope_theta=1000000.0,
                    max_position_embeddings=32768, seq_length=2048)
        base.update(kw)
        return cls(**base)
