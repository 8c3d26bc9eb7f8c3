"""paddlenlp.experimental.transformers surface kept by this build (fused_transformer_layers.py:67-78)."""
from .fused_transformer_layers import (FusedBlockMultiTransformer, FusedBlockMultiTransformerWeightOnly, FusedMultiTransformerBase,
                                       FusedMultiTransformerConfig, FusedMultiTransformerWeightOnly)
from .generation_utils import GenerationInferenceModel
from .llama.modeling import LlamaForCausalLMInferenceModel

from .token_stream import TokenStream, TokenStreamOverrun
