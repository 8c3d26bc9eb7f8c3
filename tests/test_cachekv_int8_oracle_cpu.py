"""The fake-quantised reference forward (oracle/llama_ref.py, kv_quant=): the int8-cache models are compared with it on the
H100 (tests/test_cachekv_int8_at_scale_gpu.py), so here it is pinned on the CPU: without kv_quant it is the forward the golden
files pin, on-grid K / V pass through it unchanged, and quant_from switches exactly the rows it names."""
import os

import pytest
import torch

from oracle import cachekv_int8_ref as C
from oracle import llama_ref as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")
BF16 = torch.bfloat16


def _golden(name):
    d = torch.load(os.path.join(GOLD, name), map_location="cpu", weights_only=False)
    return d, R.RefConfig(**d["config"]), {k: v.float() for k, v in d["weights"].items()}


def _scales(cfg, seed, lo=0.5, hi=4.0):
    """Distinct per-(layer, kv head) scales from absmax values in [lo, hi)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(cfg.num_hidden_layers):
        s_k, o_k = C.scales_from_absmax(lo + (hi - lo) * torch.rand(cfg.num_key_value_heads, generator=g, dtype=torch.float64))
        s_v, o_v = C.scales_from_absmax(lo + (hi - lo) * torch.rand(cfg.num_key_value_heads, generator=g, dtype=torch.float64))
        out.append((s_k, o_k, s_v, o_v))
    return out


def test_fake_quant_is_quantize_then_dequantize():
    g = torch.Generator().manual_seed(1)
    x = (3 * torch.randn(5, 4, 64, generator=g)).to(BF16).float()
    s, o = C.scales_from_absmax(torch.tensor([0.5, 2.0, 3.0, 40.0], dtype=torch.float64))
    s, o = s.view(-1, 1), o.view(-1, 1)
    want = C.dequantize(C.quantize(x, s), o).float()
    assert torch.equal(C.fake_quant(x, s, o), want)


@pytest.mark.parametrize("name", ["llama_tiny.pt", "qwen2_tiny.pt"])
def test_without_kv_quant_the_forward_is_unchanged(name):
    """kv_quant=None and a quant_from past every position give the bits of the plain forward, which the golden files pin
    (tests/test_oracle.py)."""
    d, cfg, w = _golden(name)
    ids = d["input_ids"]
    plain = R.model_forward(ids, w, cfg)
    assert torch.equal(R.model_forward(ids, w, cfg, kv_quant=None), plain)
    late = R.KvQuant(_scales(cfg, 2), torch.full((ids.shape[0],), ids.shape[1], dtype=torch.int64))
    assert torch.equal(R.model_forward(ids, w, cfg, kv_quant=late), plain)
    early = R.KvQuant(_scales(cfg, 2), torch.zeros(ids.shape[0], dtype=torch.int64))
    assert not torch.equal(R.model_forward(ids, w, cfg, kv_quant=early), plain)


def test_on_grid_values_pass_through_unchanged(monkeypatch):
    """Every projection and rotation output snapped onto the int8 grid of s = 16 (o = 1/16 exactly): the fake-quantised forward
    then equals the plain one bit for bit; off the grid it does not."""
    d, cfg, w = _golden("llama_tiny.pt")
    ids = d["input_ids"]
    s = torch.tensor(16.0, dtype=BF16)
    o = torch.tensor(1 / 16, dtype=BF16)
    grid = [(s.repeat(cfg.num_key_value_heads), o.repeat(cfg.num_key_value_heads)) * 2] * cfg.num_hidden_layers
    q = R.KvQuant(grid, torch.zeros(ids.shape[0], dtype=torch.int64))
    off_grid = R.model_forward(ids, w, cfg, kv_quant=q)
    assert not torch.equal(off_grid, R.model_forward(ids, w, cfg))
    real_linear, real_rope = R.linear, R.apply_rope
    monkeypatch.setattr(R, "linear", lambda *a, **k: C.fake_quant(real_linear(*a, **k), s, o))
    monkeypatch.setattr(R, "apply_rope", lambda *a, **k: C.fake_quant(real_rope(*a, **k), s, o))
    plain = R.model_forward(ids, w, cfg)
    assert torch.equal(R.model_forward(ids, w, cfg, kv_quant=q), plain)
    # and the unquantised attention is not what the all-quantised forward returns: fake quantisation runs on every row
    monkeypatch.setattr(R, "fake_quant_rows", lambda x, s_, o_: torch.zeros_like(x))
    assert not torch.equal(R.model_forward(ids, w, cfg, kv_quant=q), plain)


def test_quant_from_switches_exactly_its_rows():
    """One layer: rows below quant_from[b] carry the plain forward's bits and rows from it on the all-quantised forward's.
    Two layers: rows below quant_from still carry the plain bits (causal: they see only unquantised rows) and every row from
    it on differs."""
    d, cfg, w = _golden("llama_tiny.pt")
    ids = d["input_ids"]
    B, S = ids.shape
    qf = torch.tensor([S // 3, 0] + [S - 1] * (B - 2), dtype=torch.int64)[:B]
    sc = _scales(cfg, 3)
    one = R.RefConfig(**{**d["config"], "num_hidden_layers": 1})
    for c, layers in ((one, 1), (cfg, cfg.num_hidden_layers)):
        plain = R.model_forward(ids, w, c)
        allq = R.model_forward(ids, w, c, kv_quant=R.KvQuant(sc, torch.zeros(B, dtype=torch.int64)))
        got = R.model_forward(ids, w, c, kv_quant=R.KvQuant(sc, qf))
        for b in range(B):
            f = int(qf[b])
            assert torch.equal(got[b, :f], plain[b, :f]), (layers, b)
            if layers == 1:
                assert torch.equal(got[b, f:], allq[b, f:]), (layers, b)
            assert bool((got[b, f:] != plain[b, f:]).any(dim=-1).all()), (layers, b)

