"""paddlenlp_b200 — H100-native (sm_90a) implementation of PaddleNLP's LLM decoder hot path.

Sub-packages mirror the reference's import paths for the classes on that path:
    paddlenlp_b200.transformers  ~ paddlenlp.transformers  (LlamaConfig, LlamaForCausalLM, Qwen2ForCausalLM, Auto*)
    paddlenlp_b200.trainer       ~ paddlenlp.trainer       (Trainer, TrainingArguments, PdArgumentParser)
    paddlenlp_b200.ops           — torch-tensor wrappers over the C-ABI (include/b200nlp.h)
The compute path is libb200nlp.so (paddlenlp_b200/csrc); there is no CPU or library fallback.
"""
__version__ = "0.1.0"
