"""The C-ABI library builds for sm_90a, loads without a GPU, and exports exactly what include/b200nlp.h declares."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "b200nlp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_library_loads_and_exports_every_declared_symbol():
    from paddlenlp_b200 import _lib

    lib = _lib.load()              # builds in-tree with nvcc if the .so is absent
    declared = header_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b200nlp.h but not exported"
    assert sorted(_lib.exported_symbols()) == declared, "ctypes signature table out of sync with the header"
    assert lib.b200_abi_version() == 2


def test_no_cuda_device_is_a_loud_error():
    """Without a GPU the product path must fail loudly, never fall back to a CPU implementation."""
    import torch

    if torch.cuda.is_available():
        return
    import pytest

    import paddlenlp_b200.transformers as T

    with pytest.raises(RuntimeError, match="CUDA"):
        T.LlamaForCausalLM(T.LlamaConfig(hidden_size=256, num_attention_heads=2, num_hidden_layers=1, vocab_size=64,
                                         intermediate_size=512))
    from paddlenlp_b200 import ops

    with pytest.raises(ValueError, match="CUDA"):
        ops.rmsnorm_fwd(torch.zeros(2, 8, dtype=torch.bfloat16), torch.ones(8, dtype=torch.bfloat16), 1e-5)


def test_sass_contains_wgmma_mma_and_tma():
    """Evidence that the contractions are Hopper-native: HGMMA (wgmma), HMMA (mma.sync), LDSM (ldmatrix), UTMALDG (TMA)."""
    lib = os.path.join(ROOT, "paddlenlp_b200", "lib", "libb200nlp.so")
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True)
    if out.returncode != 0:
        import pytest

        pytest.skip("cuobjdump unavailable")
    sass = out.stdout
    for mnemonic in ("HGMMA", "HMMA", "LDSM", "UTMALDG"):
        assert mnemonic in sass, mnemonic
    assert "arch = sm_90a" in sass and "arch = sm_100" not in sass


def test_product_path_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "paddlenlp_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), os.path.join(dirpath, f)
