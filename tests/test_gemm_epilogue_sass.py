"""The 128-row wgmma GEMM epilogue stores its output tiles with TMA (checked in the built library's SASS, no GPU needed)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_contains_tma_stores():
    lib = os.path.join(ROOT, "paddlenlp_b200", "lib", "libb200nlp.so")
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "UTMASTG" in out.stdout
