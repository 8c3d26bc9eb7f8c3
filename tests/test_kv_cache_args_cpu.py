"""Every entry point that addresses the paged KV cache accepts the same block geometry (block_size 32, 64 or 128, at least one
block per sequence, a block table) and rejects any other as an argument error naming itself, before any CUDA call: called
through the C-ABI with integer addresses that are never dereferenced, no device is needed."""
import pytest
import torch

# With a device, a regression that let such a call through would launch a kernel on these made-up addresses.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a machine without a CUDA device")

QKV, KC, VC, BT, LENS, OUT, WS, COS, SIN = ((i + 1) << 20 for i in range(9))   # 16-byte aligned stand-ins for device addresses
B, NH, KVH, D = 2, 8, 2, 128
LD = (NH + 2 * KVH) * D


def _write_cache_kv_paged(block_size, max_blocks, bt):
    return (QKV, KC, VC, bt, LENS, B, 16, NH, KVH, D, block_size, max_blocks, LD, None)


def _decode_rope_append_paged(block_size, max_blocks, bt):
    return (QKV, None, None, KC, VC, bt, COS, SIN, LENS, B, NH, KVH, D, block_size, max_blocks, LD, None)


def _decode_attention_paged(block_size, max_blocks, bt):
    return (QKV, KC, VC, bt, LENS, OUT, WS, B, NH, KVH, D, 16, block_size, max_blocks, LD, 0.1, 1, None)


def _append_attention(block_size, max_blocks, bt):
    return (QKV, KC, VC, LENS, LENS, LENS, LENS, bt, COS, SIN, OUT, WS, B, 4, 3, NH, KVH, D, 16, block_size, max_blocks, 4096,
            LD, NH * D, 0.1, 1, None)


ENTRIES = [_write_cache_kv_paged, _decode_rope_append_paged, _decode_attention_paged, _append_attention]
BAD = {"block_size_16": (16, 4, BT), "block_size_0": (0, 4, BT), "no_blocks": (64, 0, BT), "null_table": (64, 4, None)}


@pytest.mark.parametrize("bad", list(BAD))
@pytest.mark.parametrize("entry", ENTRIES, ids=[f.__name__[1:] for f in ENTRIES])
def test_bad_block_geometry_is_an_argument_error(entry, bad):
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    name = entry.__name__[1:]
    rc = getattr(lib, "b200_" + name)(*entry(*BAD[bad]))
    msg = lib.b200_last_error().decode()
    assert rc < 0, (rc, msg)
    assert msg.startswith(name + ":"), msg


def test_append_attention_checks_the_decode_rows_before_any_launch():
    """A GQA group the decode kernel has no instantiation for is refused before the RoPE / cache-write kernel runs, so the cache
    is left untouched (with no device, a launch would return a CUDA error instead of the argument error)."""
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    nh, kvh = 18, 2
    args = list(_append_attention(64, 4, BT))
    args[15], args[16] = nh, kvh
    args[22], args[23] = (nh + 2 * kvh) * D, nh * D
    rc = lib.b200_append_attention(*args)
    msg = lib.b200_last_error().decode()
    assert rc < 0, (rc, msg)
    assert msg.startswith("append_attention: GQA group size 9"), msg
