"""The GEMM entry points reject an output or epilogue input whose base address is not 16-byte aligned (TMA can neither store
to nor read from it), before they encode a tensor map or make any CUDA call: called through the C-ABI with integer addresses
that are never dereferenced, no device is needed."""
import re

import pytest
import torch

# With a device, a regression that let such a call through would launch a kernel on these made-up addresses.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a machine without a CUDA device")

A, B, X, Y = 1 << 20, 2 << 20, 3 << 20, 4 << 20   # 16-byte aligned stand-ins for device addresses


def _gemm_ex(off, operand):
    c, r = (Y + off, X) if operand == "C" else (Y, X + off)
    return "b200_gemm_bf16_ex", (A, B, c, None, r, 64, 256, 128, 128, 256, 256, 256, 0, 1, 0, 0, None)


def _swiglu(off, operand):
    gu, m = (X + off, Y) if operand == "GU" else (X, Y + off)
    return "b200_gemm_swiglu_bf16", (A, B, gu, m, 64, 128, 128, 128, 256, 256, 128, None)


def _swiglu_bwd(off, operand):
    gu, dgu = (X + off, Y) if operand == "GU" else (X, Y + off)
    return "b200_gemm_swiglu_bwd_bf16", (A, B, gu, dgu, 64, 128, 128, 128, 128, 256, 256, None)


def _splitk(off, operand):
    return "b200_gemm_bf16_splitk", (A, B, Y + off, None, X, 64, 256, 128, 128, 256, 256, 0, 1, 0, None)


CASES = [(_gemm_ex, "C"), (_gemm_ex, "residual"), (_swiglu, "GU"), (_swiglu, "Mout"), (_swiglu_bwd, "GU"),
         (_swiglu_bwd, "DGU"), (_splitk, "C")]


@pytest.mark.parametrize("off", [2, 4, 8])
@pytest.mark.parametrize("case", CASES, ids=[f"{f.__name__[1:]}-{op}" for f, op in CASES])
def test_misaligned_base_is_an_argument_error(case, off):
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    name, args = case[0](off, case[1])
    rc = getattr(lib, name)(*args)
    msg = lib.b200_last_error().decode()
    assert rc < 0, (rc, msg)
    assert re.search(rf"\b{case[1]} must be 16-byte aligned", msg), msg
