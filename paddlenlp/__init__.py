"""`paddlenlp` import-path shim: `import paddlenlp.X` resolves to `paddlenlp_b200.X` (the same module object).

The H100-native implementation lives in `paddlenlp_b200/` (so that it can be installed next to the reference without
shadowing it); putting THIS directory on sys.path makes the reference's own import lines work unchanged for the hot path —
    from paddlenlp.trainer import PdArgumentParser, Trainer, TrainingArguments, get_last_checkpoint, set_seed, speed_metrics
    from paddlenlp.transformers import AutoConfig, AutoModelForCausalLM, LlamaConfig, LlamaForCausalLM, ...
    from paddlenlp.transformers.llama import fusion_ops
    from paddlenlp.experimental.transformers import FusedMultiTransformerBase, ...
(llm/run_pretrain.py:24-47, llm/run_finetune.py, llm/predict/predictor.py).  Sub-packages outside the data-parallel decoder hot
path do not exist; importing them fails with ModuleNotFoundError naming the missing `paddlenlp_b200` module.
"""
import importlib
import importlib.abc
import importlib.util
import sys

import paddlenlp_b200 as _impl

__version__ = getattr(_impl, "__version__", "0")
_PREFIX, _REAL = "paddlenlp.", "paddlenlp_b200."


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, real_name):
        self.real_name = real_name

    def create_module(self, spec):
        mod = importlib.import_module(self.real_name)     # the real module object: paddlenlp.X IS paddlenlp_b200.X
        return mod

    def exec_module(self, module):
        pass


class _AliasFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
        if not fullname.startswith(_PREFIX):
            return None
        real = _REAL + fullname[len(_PREFIX):]
        try:
            real_spec = importlib.util.find_spec(real)
        except (ImportError, ValueError):
            real_spec = None
        if real_spec is None:
            return None
        spec = importlib.util.spec_from_loader(fullname, _AliasLoader(real), is_package=real_spec.submodule_search_locations is not None)
        return spec


if not any(isinstance(f, _AliasFinder) for f in sys.meta_path):
    sys.meta_path.insert(0, _AliasFinder())
