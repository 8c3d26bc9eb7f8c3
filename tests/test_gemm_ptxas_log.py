"""ptxas neither serialised the wgmmas of a GEMM instantiation nor spilled in it (read from the build's ptxas log, no GPU needed)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gemm_wgmmas_not_serialised_and_no_spills():
    """A function call anywhere in the kernel (a printf in a barrier wait) makes ptxas wait for every wgmma before it issues the
    next: it says so with C7510, and the GEMMs then run about 9 % slower."""
    log = os.path.join(ROOT, "paddlenlp_b200", "build", "gemm_wgmma.o.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log: the library was not built in this tree")
    with open(log) as f:
        text = f.read()
    assert "C7510" not in text
    found = re.findall(r"Compiling entry function '(\w*gemm_bf16_kernel\w*)'.*\n.*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", text)
    assert len(found) == 8, found   # 64- and 128-row tiles x 4 operand-major combinations
    for name, stack, stores, loads in found:
        assert (stack, stores, loads) == ("0", "0", "0"), (name, stack, stores, loads)
