"""End-to-end parity of the native decoder path against the oracle: logits, loss, argmax, gradients.

Tolerances (north star): logits / loss within 1e-3 relative of the reference's bf16 path, argmax identical.  bf16 carries
~3 significant digits, so "relative" is the normalised error max|a-b| / max|b| and ||a-b|| / ||b|| against the oracle
evaluated WITH the reference's bf16 rounding points (SURVEY.md §7.3 item 4); the oracle's own bf16-vs-fp32 distance is
printed beside it as the noise floor.
"""
import pytest
import torch

from oracle import llama_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def maxerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def tiny_cfg(model_type="llama"):
    return R.RefConfig(vocab_size=1024, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                       num_attention_heads=2, num_key_value_heads=1, rms_norm_eps=1e-5 if model_type == "llama" else 1e-6,
                       rope_theta=500000.0 if model_type == "llama" else 1e6, qkv_bias=(model_type == "qwen2"),
                       model_type=model_type, max_position_embeddings=512)


def build(cfg: R.RefConfig, weights):
    import paddlenlp_b200.transformers as T

    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    if cfg.model_type == "qwen2":
        model = T.Qwen2ForCausalLM(T.Qwen2Config(**kw))
    else:
        model = T.LlamaForCausalLM(T.LlamaConfig(**kw))
    model.set_state_dict(weights)
    return model


def make_weights(cfg, seed=3):
    w = R.init_weights(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    for k in w:      # non-trivial norm weights so the norm-weight gradient path is exercised
        if "norm" in k:
            w[k] = (1.0 + 0.1 * torch.randn(w[k].shape, generator=g)).to(torch.bfloat16).float()
    # larger weights than the 0.02 init so logits are not degenerate (argmax margins above bf16 noise)
    for k in w:
        if k.endswith("proj.weight") or k.startswith("lm_head") or "embed" in k:
            w[k] = (w[k] * 3.0).to(torch.bfloat16).float()
    return w


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_logits_loss_argmax_and_grads(model_type):
    cfg = tiny_cfg(model_type)
    w = make_weights(cfg)
    model = build(cfg, w)
    B, S = 2, 256
    g = torch.Generator().manual_seed(1234)
    tok = torch.randint(0, cfg.vocab_size, (B, S + 1), generator=g)
    ids, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()      # reference collate: run_pretrain.py:245-255
    labels[0, :7] = -100

    # ---- forward: logits ----
    with torch.no_grad():
        logits = model(input_ids=ids.to(DEV))[0].float().cpu()
    ref16 = R.model_forward(ids, w, cfg, mode="bf16")
    ref32 = R.model_forward(ids, w, cfg, mode="fp32")
    floor, floor_rel = maxerr(ref16, ref32), relerr(ref16, ref32)
    e_max, e_rel = maxerr(logits, ref16), relerr(logits, ref16)
    e32_rel = relerr(logits, ref32)
    print(f"[{model_type}] logits vs bf16-oracle: max {e_max:.2e} rel {e_rel:.2e}; vs fp32-oracle rel {e32_rel:.2e}; "
          f"oracle bf16-vs-fp32 floor: max {floor:.2e} rel {floor_rel:.2e}")
    # Two bf16 evaluations with different fp32 accumulation orders differ by the same amount as either differs from
    # fp32 (a flipped rounding propagates through the layers): the CUDA path must be no further from the fp32 truth
    # than the bf16 oracle is, and within 2x that noise floor of the bf16 oracle itself.
    assert e32_rel <= 1.25 * floor_rel + 1e-3
    assert e_max <= max(2.0 * floor, 4e-3)
    assert e_rel <= max(2.0 * floor_rel, 5e-3)
    # ---- argmax: identical wherever the oracle's top-1 / top-2 margin exceeds the bf16 noise ----
    am, am_ref = logits.argmax(-1), ref16.argmax(-1)
    top2 = ref16.topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1])
    decisive = margin > 2 * e_max * ref16.abs().max()
    agree = (am == am_ref)
    print(f"[{model_type}] argmax agreement {agree.float().mean().item():.4f}; decisive positions {decisive.float().mean().item():.3f}")
    assert bool(agree[decisive].all())
    assert agree.float().mean().item() > 0.95

    # ---- loss ----
    loss, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    ref_loss = R.criterion(ref16, labels)
    assert abs(loss.item() - ref_loss.item()) <= 1e-3 * abs(ref_loss.item())

    # ---- backward: gradients vs autograd through the bf16-rounding oracle ----
    model.engine.clear_grad()
    (loss * 1.0).backward()
    _, _, gref = R.loss_and_grads(ids, labels, w, cfg, mode="bf16")
    grads = {k: v.grad.float().cpu() for k, v in model.named_parameters()}
    worst = 0.0
    for k, gr in gref.items():
        e = relerr(grads[k], gr)
        worst = max(worst, e)
        assert e < 3e-2, f"grad {k}: rel err {e:.3e}"     # bf16 gradients, tolerance precedent 1e-2 per op
    print(f"[{model_type}] worst gradient rel err {worst:.2e}")

    # ---- accumulation: a second backward with scale 0.5 adds half of the same gradient ----
    loss2, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    (loss2 * 0.5).backward()
    for k in ("lm_head.weight", f"{cfg.model_type}.layers.0.mlp.down_proj.weight", f"{cfg.model_type}.norm.weight"):
        g2 = dict(model.named_parameters())[k].grad.float().cpu()
        assert relerr(g2, 1.5 * gref[k]) < 3e-2


def test_single_layer_standard_init_tight():
    """One decoder layer at the reference's own init scale: the regime where bf16 noise does not compound, so the
    north-star tolerance (1e-3 relative, argmax exact) is checked directly."""
    cfg = tiny_cfg()
    cfg.num_hidden_layers = 1
    w = R.init_weights(cfg, seed=11)
    w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(torch.bfloat16).float()   # decisive logits
    model = build(cfg, w)
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(12))
    with torch.no_grad():
        logits = model(input_ids=ids.to(DEV))[0].float().cpu()
    ref16 = R.model_forward(ids, w, cfg, mode="bf16")
    ref32 = R.model_forward(ids, w, cfg, mode="fp32")
    e_rel, e_max = relerr(logits, ref16), maxerr(logits, ref16)
    floor_rel = relerr(ref16, ref32)
    mism = (logits != ref16).float().mean().item()
    print(f"[1-layer] rel {e_rel:.2e} max {e_max:.2e} (oracle bf16-vs-fp32 floor rel {floor_rel:.2e}); "
          f"elements differing from the bf16 oracle: {mism:.4f}")
    assert relerr(logits, ref32) <= 1.25 * floor_rel + 5e-4
    assert e_rel <= max(2.0 * floor_rel, 2e-3)
    am, am_ref = logits.argmax(-1), ref16.argmax(-1)
    top2 = ref16.topk(2, dim=-1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 2 * e_max * ref16.abs().max()
    assert bool((am == am_ref)[decisive].all())
    assert (am == am_ref).float().mean().item() > 0.95


def test_position_ids_default_equals_arange():
    """tests/transformers/llama/test_modeling.py:250-270 property."""
    cfg = tiny_cfg()
    model = build(cfg, make_weights(cfg))
    ids = torch.randint(0, cfg.vocab_size, (2, 128), generator=torch.Generator().manual_seed(5)).to(DEV)
    pos = torch.arange(128).unsqueeze(0).expand(2, -1).contiguous().to(DEV)
    with torch.no_grad():
        a = model(input_ids=ids)[0]
        b = model(input_ids=ids, position_ids=pos)[0]
    assert torch.equal(a, b)


def test_causality_prefix_invariance():
    """Causal attention: logits at position t do not depend on tokens after t (mask-invariance family of properties,
    tests/transformers/llama/test_modeling.py:152-169)."""
    cfg = tiny_cfg()
    model = build(cfg, make_weights(cfg))
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(0, cfg.vocab_size, (1, 256), generator=g)
    ids2 = ids.clone()
    ids2[0, 130:] = torch.randint(0, cfg.vocab_size, (126,), generator=g)
    with torch.no_grad():
        a = model(input_ids=ids.to(DEV))[0]
        b = model(input_ids=ids2.to(DEV))[0]
    assert torch.equal(a[0, :130], b[0, :130])
    assert not torch.equal(a[0, 130:], b[0, 130:])


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_flashmask_packing_invariance(model_type, request):
    """Zero-padding (sample packing, SURVEY §8f rank 3): three samples packed into one row with FlashMask start rows and per-sample
    position ids, right-padded the reference's way (indices padded with 0), give the logits, loss and gradients of the same
    samples run one by one.  Also checked against the oracle's masked attention end to end."""
    from paddlenlp_b200 import _lib
    from paddlenlp_b200.data import DataCollatorForSeq2Seq
    from paddlenlp_b200.datasets import ZeroPaddingMapDataset

    # the "same tiles, same order -> same bits" property below compares packed (FlashMask) and one-by-one (plain causal) runs
    # of the SAME attention kernel: both instantiations live in fa_fwd.cu
    cfg = tiny_cfg(model_type)
    w = make_weights(cfg)
    model = build(cfg, w)
    g = torch.Generator().manual_seed(11)
    lens = [150, 37, 201]
    recs = []
    for n in lens:
        ids = torch.randint(1, cfg.vocab_size, (n + 1,), generator=g)
        lab = ids[1:].clone()
        lab[: n // 3] = -100                                          # prompt tokens carry no loss (llm/utils/data.py:179-206)
        recs.append({"input_ids": ids[:-1].tolist(), "labels": lab.tolist()})
    packed = ZeroPaddingMapDataset(recs, max_length=512)
    assert len(packed) == 1
    batch = DataCollatorForSeq2Seq(max_length=512, pad_token_id=0)([packed[0]])
    assert batch["attn_mask_startend_row_indices"][0, 149] == 150 and batch["attn_mask_startend_row_indices"][0, 400] == 0
    dev = {k: v.to(DEV) for k, v in batch.items()}

    # packed run
    model.engine.clear_grad()
    loss, logits = model(**dev)
    logits = logits.clone()                                           # backward() reuses the logits buffer for dlogits
    loss.backward()
    g_packed = {k: v.clone() for k, v in model.engine.named_views(grads=True).items()}
    n_valid = sum(int((torch.tensor(r["labels"]) != -100).sum()) for r in recs)

    # the same samples one by one, gradients accumulated with the weights that make the sum the packed mean
    model.engine.clear_grad()
    start, loss_sum = 0, 0.0
    for r in recs:
        n = len(r["input_ids"])
        ids = torch.tensor([r["input_ids"]]).to(DEV)
        lab = torch.tensor([r["labels"]]).to(DEV)
        nv = int((lab != -100).sum())
        l1, lg1 = model(input_ids=ids, labels=lab)
        lg1 = lg1.clone()
        (l1 * (nv / n_valid)).backward()
        loss_sum += float(l1.detach()) * nv
        seg = logits[0, start:start + n].float()
        assert maxerr(seg, lg1[0]) < 2e-2, (start, maxerr(seg, lg1[0]))
        if start == 0:
            assert torch.equal(logits[0, :n], lg1[0])                  # first sample: same tiles, same order -> same bits
        start += n
    assert abs(float(loss.detach()) - loss_sum / n_valid) < 2e-3 * abs(float(loss.detach()))
    g_single = model.engine.named_views(grads=True)
    pre = cfg.model_type
    for k in (f"{pre}.layers.0.self_attn.q_proj.weight", f"{pre}.layers.1.self_attn.v_proj.weight",
              f"{pre}.layers.0.mlp.down_proj.weight", f"{pre}.layers.1.input_layernorm.weight", "lm_head.weight"):
        assert relerr(g_packed[k], g_single[k]) < 3e-2, (k, relerr(g_packed[k], g_single[k]))

    # oracle with the same mask (bf16 rounding points): logits on the real tokens
    ms = torch.maximum(batch["attn_mask_startend_row_indices"], torch.arange(1, 513, dtype=torch.int32)[None])
    wd = {k: v.float() for k, v in w.items()}
    cos, sin = R.rope_tables(cfg.hidden_size // cfg.num_attention_heads, cfg.max_position_embeddings, cfg.rope_theta)
    x = wd[f"{pre}.embed_tokens.weight"][batch["input_ids"]]
    for i in range(cfg.num_hidden_layers):
        x = R.decoder_layer(x, wd, f"{pre}.layers.{i}.", cfg, cos, sin, "bf16", position_ids=batch["position_ids"], mask_start=ms)
    ref = R.linear(R.rms_norm(x, wd[f"{pre}.norm.weight"], cfg.rms_norm_eps, "bf16"), wd["lm_head.weight"], None, "bf16")
    real = sum(lens)
    e = maxerr(logits[0, :real].cpu(), ref[0, :real])
    assert e < 3e-2, e


def test_flashmask_rejects_non_document_masks():
    cfg = tiny_cfg()
    model = build(cfg, make_weights(cfg))
    ids = torch.randint(1, cfg.vocab_size, (1, 128), generator=torch.Generator().manual_seed(1)).to(DEV)
    bad = torch.full((1, 128), 128, dtype=torch.int32)
    bad[0, 40:80] = 60                                                # a start row that decreases again: not a packed layout
    with pytest.raises(ValueError):
        model(input_ids=ids, attn_mask_startend_row_indices=bad.to(DEV))


def test_full_width_single_layer_llama3_8b_shapes():
    """SURVEY §8d parity input: one decoder layer at the FULL Llama-3-8B width (h 4096, 32 q / 8 kv heads, I 14336; vocab and
    sequence shortened so that the CPU oracle finishes in seconds) — logits, loss and the layer's weight gradients vs the
    bf16-rounding oracle, with the oracle's own bf16-vs-fp32 distance as the noise floor."""
    cfg = R.RefConfig(vocab_size=4096, hidden_size=4096, intermediate_size=14336, num_hidden_layers=1, num_attention_heads=32,
                      num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=1024)
    w = R.init_weights(cfg, seed=21)
    w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(torch.bfloat16).float()   # decisive logits at the 0.02 init scale
    model = build(cfg, w)
    tok = torch.randint(0, cfg.vocab_size, (1, 1025), generator=torch.Generator().manual_seed(22))
    ids, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    loss, logits = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    logits = logits.float().cpu().clone()
    ref16 = R.model_forward(ids, w, cfg, mode="bf16")
    ref32 = R.model_forward(ids, w, cfg, mode="fp32")
    floor_rel = relerr(ref16, ref32)
    e_rel, e_max = relerr(logits, ref16), maxerr(logits, ref16)
    print(f"[full width] logits rel {e_rel:.2e} max {e_max:.2e}; oracle bf16-vs-fp32 floor rel {floor_rel:.2e}")
    assert relerr(logits, ref32) <= 1.25 * floor_rel + 5e-4
    assert e_rel <= max(2.0 * floor_rel, 2e-3)
    am, am_ref = logits.argmax(-1), ref16.argmax(-1)
    top2 = ref16.topk(2, dim=-1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 2 * e_max * ref16.abs().max()
    assert bool((am == am_ref)[decisive].all()) and (am == am_ref).float().mean().item() > 0.95
    ref_loss = R.criterion(ref16, labels)
    assert abs(loss.item() - ref_loss.item()) <= 1e-3 * abs(ref_loss.item())
    model.engine.clear_grad()
    loss.backward()
    _, _, gref = R.loss_and_grads(ids, labels, w, cfg, mode="bf16")
    grads = model.engine.named_views(grads=True)
    for k in ("llama.layers.0.self_attn.q_proj.weight", "llama.layers.0.self_attn.v_proj.weight", "llama.layers.0.mlp.up_proj.weight",
              "llama.layers.0.mlp.down_proj.weight", "llama.layers.0.input_layernorm.weight"):
        e = relerr(grads[k].cpu(), gref[k])
        assert e < 3e-2, (k, e)


# ------------------------------------------------------------------------------------------------
# Parity at the BENCHMARKED shape (SURVEY §8d "Parity inputs"; VERDICT r01 weak #1): full Llama-3-8B layer width at S = 4096.
# The oracle is evaluated on the GPU in fp32 torch (it is a checker: cuBLAS fp32, TF32 off) — on the CPU these sizes take minutes.
# ------------------------------------------------------------------------------------------------
def _chunked_linear(x, wt, bias, mode):
    """R.linear with the K dimension summed in 4 chunks: the same rounding points, a different fp32 accumulation order."""
    K = wt.shape[0]
    step = (K + 3) // 4
    y = None
    for s0 in range(0, K, step):
        part = x[..., s0:s0 + step] @ wt[s0:s0 + step]
        y = part if y is None else y + part
    if bias is not None:
        y = y + bias
    return R.rnd(y, mode)


def _oracle_on_device(cfg, w, ids, labels, want_grads=True, reorder_grads=False):
    assert not torch.backends.cuda.matmul.allow_tf32
    wd = {k: v.to(DEV) for k, v in w.items()}
    ids_d, lab_d = ids.to(DEV), labels.to(DEV)
    with torch.no_grad():
        ref32 = R.model_forward(ids_d, wd, cfg, mode="fp32")
    if want_grads:
        ref_loss, ref16, gref = R.loss_and_grads(ids_d, lab_d, wd, cfg, mode="bf16")
    else:
        with torch.no_grad():
            ref16 = R.model_forward(ids_d, wd, cfg, mode="bf16")
        ref_loss, gref = R.criterion(ref16, lab_d), None
    if reorder_grads:
        orig = R.linear
        R.linear = _chunked_linear
        try:
            _, _, gref2 = R.loss_and_grads(ids_d, lab_d, wd, cfg, mode="bf16")
        finally:
            R.linear = orig
        return ref16, ref32, ref_loss, gref, gref2
    return ref16, ref32, ref_loss, gref


def _check_logits_loss_argmax(tag, logits, loss, ref16, ref32, ref_loss):
    floor_rel = relerr(ref16, ref32)
    e_rel, e_max = relerr(logits, ref16), maxerr(logits, ref16)
    e32 = relerr(logits, ref32)
    print(f"[{tag}] logits vs bf16-oracle rel {e_rel:.2e} max {e_max:.2e}; vs fp32-oracle rel {e32:.2e}; "
          f"oracle bf16-vs-fp32 floor rel {floor_rel:.2e}; loss {float(loss):.6f} vs {float(ref_loss):.6f}")
    assert e32 <= 1.25 * floor_rel + 5e-4
    assert e_rel <= max(2.0 * floor_rel, 2e-3)
    am, am_ref = logits.argmax(-1), ref16.argmax(-1)
    top2 = ref16.topk(2, dim=-1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 2 * e_max * ref16.abs().max()
    agree = (am == am_ref)
    print(f"[{tag}] argmax agreement {agree.float().mean().item():.4f}; decisive positions {decisive.float().mean().item():.3f}")
    assert bool(agree[decisive].all()) and agree.float().mean().item() > 0.95
    assert abs(float(loss) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))


def test_full_width_layer_at_bench_shape_b2_s4096():
    """One decoder layer at the full Llama-3-8B width with the bench's micro-batch shape: B = 2, S = 4096 (32 q tiles x 32
    heads x 2 sequences through the attention kernels, M = 8192 GEMMs): logits, loss, arg-max and the layer's weight
    gradients vs the bf16-rounding oracle."""
    cfg = R.RefConfig(vocab_size=4096, hidden_size=4096, intermediate_size=14336, num_hidden_layers=1, num_attention_heads=32,
                      num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=4096)
    w = R.init_weights(cfg, seed=31)
    w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(torch.bfloat16).float()   # decisive logits at the 0.02 init scale
    model = build(cfg, w)
    tok = torch.randint(0, cfg.vocab_size, (2, 4097), generator=torch.Generator().manual_seed(32))
    ids, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    loss, logits = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    logits = logits.float().clone()
    ref16, ref32, ref_loss, gref = _oracle_on_device(cfg, w, ids, labels)
    _check_logits_loss_argmax("full width, B=2 S=4096", logits, loss.detach(), ref16, ref32, ref_loss)
    del ref16, ref32
    model.engine.clear_grad()
    loss.backward()
    grads = model.engine.named_views(grads=True)
    worst = 0.0
    for k in ("llama.layers.0.self_attn.q_proj.weight", "llama.layers.0.self_attn.k_proj.weight",
              "llama.layers.0.self_attn.v_proj.weight", "llama.layers.0.self_attn.o_proj.weight",
              "llama.layers.0.mlp.gate_proj.weight", "llama.layers.0.mlp.up_proj.weight", "llama.layers.0.mlp.down_proj.weight",
              "llama.layers.0.input_layernorm.weight", "llama.layers.0.post_attention_layernorm.weight", "lm_head.weight",
              "llama.embed_tokens.weight"):
        e = relerr(grads[k], gref[k])
        worst = max(worst, e)
        assert e < 3e-2, (k, e)
    print(f"[full width, B=2 S=4096] worst gradient rel err {worst:.2e}")


def test_two_layer_full_width_real_vocab_s4096():
    """Two decoder layers at full width with the REAL 128 256-wide lm_head / criterion at S = 4096 (the head GEMMs with
    N = K = 128 256 and the CE kernels at the bench's row count), plus the micro-batch accumulation path: two backward
    passes accumulate into the flat gradient buffer exactly as bench.py's step does."""
    cfg = R.RefConfig(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=2, num_attention_heads=32,
                      num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=4096)
    w = R.init_weights(cfg, seed=41)
    w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(torch.bfloat16).float()
    model = build(cfg, w)
    tok = torch.randint(0, cfg.vocab_size, (2, 4097), generator=torch.Generator().manual_seed(42))
    ids, labels = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    model.engine.clear_grad()
    gsum = gsum2 = None
    for mb in range(2):                                   # two micro-batches of one sequence, loss / 2 each (bench: / accum)
        i1, l1 = ids[mb:mb + 1], labels[mb:mb + 1]
        loss, logits = model(input_ids=i1.to(DEV), labels=l1.to(DEV))
        logits = logits.float().clone()
        ref16, ref32, ref_loss, gref, gref2 = _oracle_on_device(cfg, w, i1, l1, reorder_grads=True)
        _check_logits_loss_argmax(f"2 layers, V=128256, S=4096, micro-batch {mb}", logits, loss.detach(), ref16, ref32, ref_loss)
        del ref16, ref32, logits
        (loss / 2).backward()
        gsum = {k: v / 2 for k, v in gref.items()} if gsum is None else {k: gsum[k] + gref[k] / 2 for k in gref}
        gsum2 = {k: v / 2 for k, v in gref2.items()} if gsum2 is None else {k: gsum2[k] + gref2[k] / 2 for k in gref2}
        del gref, gref2
    grads = model.engine.named_views(grads=True)
    # Gradient tolerance = the oracle's OWN sensitivity to the fp32 accumulation order, measured: with logits of magnitude ~40
    # (lm_head x 8 for decisive arg-max) one bf16 ulp of a logit is 0.25, i.e. exp(+-0.25) = +-25 % on that probability, so two
    # correct bf16 evaluations disagree on d(logits) by percents — the same oracle with every Linear summed in 4 K-chunks gives
    # the floor, and the CUDA path must stay within 2x of it (3e-2 where the floor is small).
    worst = 0.0
    for k in ("lm_head.weight", "llama.norm.weight", "llama.layers.1.mlp.down_proj.weight", "llama.layers.1.self_attn.q_proj.weight",
              "llama.layers.0.self_attn.v_proj.weight", "llama.layers.0.mlp.gate_proj.weight", "llama.layers.0.input_layernorm.weight",
              "llama.embed_tokens.weight"):
        e, floor = relerr(grads[k], gsum[k]), relerr(gsum2[k], gsum[k])
        print(f"[2 layers, V=128256] grad {k}: rel err {e:.2e}; oracle re-ordering floor {floor:.2e}")
        worst = max(worst, e)
        assert e < max(3e-2, 2.0 * floor), (k, e, floor)
    print(f"[2 layers, V=128256] worst accumulated-gradient rel err {worst:.2e}")


def test_reorder_noise_floor_at_depth():
    """How far apart do two CORRECT bf16 evaluations sit when only the fp32 accumulation order differs?  The bf16-rounding
    oracle is evaluated twice on the GPU — once with plain matmuls, once with every Linear's K dimension summed in 4 chunks —
    at depth 2, 8 and 32 (h = 1024).  This is the measured floor behind the "2 x floor" logits tolerance (VERDICT r01 weak #2):
    the CUDA path at depth 32 must sit no further from the oracle than 2 x the oracle's own re-ordering distance, and both are
    printed beside the bf16-vs-fp32 distance."""
    orig_linear = R.linear
    chunked_linear = _chunked_linear

    rows = []
    for L in (2, 8, 32):
        cfg = R.RefConfig(vocab_size=2048, hidden_size=1024, intermediate_size=2752, num_hidden_layers=L, num_attention_heads=8,
                          num_key_value_heads=2, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=512)
        w = R.init_weights(cfg, seed=50 + L)
        w["lm_head.weight"] = (w["lm_head.weight"] * 8).to(torch.bfloat16).float()
        ids = torch.randint(0, cfg.vocab_size, (2, 512), generator=torch.Generator().manual_seed(51))
        wd = {k: v.to(DEV) for k, v in w.items()}
        with torch.no_grad():
            a = R.model_forward(ids.to(DEV), wd, cfg, mode="bf16")
            f = R.model_forward(ids.to(DEV), wd, cfg, mode="fp32")
            R.linear = chunked_linear
            try:
                b = R.model_forward(ids.to(DEV), wd, cfg, mode="bf16")
            finally:
                R.linear = orig_linear
        model = build(cfg, w)
        with torch.no_grad():
            c = model(input_ids=ids.to(DEV))[0].float()
        reorder, floor32, ours = relerr(b, a), relerr(a, f), relerr(c, a)
        rows.append((L, reorder, floor32, ours, relerr(c, f)))
        print(f"[depth {L:2d}] oracle(bf16) vs oracle(bf16, K summed in 4 chunks): rel {reorder:.2e} | oracle bf16 vs fp32: {floor32:.2e} | "
              f"CUDA vs oracle(bf16): {ours:.2e} | CUDA vs fp32: {relerr(c, f):.2e}")
        assert ours <= max(2.0 * max(reorder, floor32), 2e-3), (L, ours, reorder, floor32)
        assert relerr(c, f) <= 1.25 * floor32 + 5e-4
        del model
    assert rows[-1][1] > 1e-3          # the re-ordering distance itself exceeds 1e-3 at depth: 1e-3 element-wise is not attainable in bf16


# ------------------------------------------------------------------------------------------------
# init (row a10), activation recomputation, padding masks, rotary scaling
# ------------------------------------------------------------------------------------------------
def test_init_weights_statistics_and_shared_bits():
    """LlamaPretrainedModel._init_weights (llama/modeling.py:1386-1436): N(0, 0.02) for every Linear / Embedding / lm_head,
    o_proj and down_proj scaled by 1/sqrt(2L), RMSNorm weights 1, biases 0 — for both init paths of the engine:
    the host path shares bits with the CPU restatement (same generator, same draw order, fp32 -> bf16 once), the device path
    (what an 8 B model uses) is checked on its statistics and on seed determinism."""
    import math

    import paddlenlp_b200.transformers as T

    kw = dict(vocab_size=2048, hidden_size=512, intermediate_size=1376, num_hidden_layers=4, num_attention_heads=4,
              num_key_value_heads=2, max_position_embeddings=256)
    cfg = R.RefConfig(rms_norm_eps=1e-6, rope_theta=10000.0, **kw)
    model = T.LlamaForCausalLM(T.LlamaConfig(seed=77, **kw))          # default: host path (small model)
    ref = R.init_weights(cfg, seed=77)
    sd = model.state_dict()
    assert set(sd) == set(ref)
    for k, v in ref.items():
        assert torch.equal(sd[k].float().cpu(), v), k                  # shared bits (SURVEY §8a a10)
    L, std = 4, 0.02
    for on_host in (False, True):
        model.engine.init_weights(seed=5, on_host=on_host)
        sd = {k: v.float() for k, v in model.state_dict().items()}
        for k, v in sd.items():
            if "norm" in k:
                assert bool((v == 1).all()), k
                continue
            want = std / math.sqrt(2 * L) if ("o_proj" in k or "down_proj" in k) else std
            assert abs(v.std().item() / want - 1) < 0.02, (k, on_host, v.std().item(), want)
            assert abs(v.mean().item()) < 4 * want / math.sqrt(v.numel()) + 1e-6, (k, on_host, v.mean().item())
        a = model.engine.flat_params.clone()
        model.engine.init_weights(seed=5, on_host=on_host)
        assert torch.equal(a, model.engine.flat_params)                # same seed -> same bits
        model.engine.init_weights(seed=6, on_host=on_host)
        assert not torch.equal(a, model.engine.flat_params)
    # Qwen2: q/k/v biases start at zero (Paddle nn.Linear default), weights as above
    mq = T.Qwen2ForCausalLM(T.Qwen2Config(**kw))
    for k, v in mq.state_dict().items():
        if k.endswith("bias"):
            assert bool((v == 0).all()), k


@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_recompute_matches_stored_activations(model_type):
    """recompute_enable() (model_utils.py:1140; llama/modeling.py:1706-1733 granularity "full"): every layer keeps only its input
    and is re-run inside backward.  The forward kernels are deterministic, so loss and logits are bit-identical and the gradients
    agree to the attention-backward summation noise."""
    cfg = tiny_cfg(model_type)
    w = make_weights(cfg)
    model = build(cfg, w)
    tok = torch.randint(0, cfg.vocab_size, (2, 257), generator=torch.Generator().manual_seed(9))
    ids, labels = tok[:, :-1].contiguous().to(DEV), tok[:, 1:].contiguous().to(DEV)
    model.engine.clear_grad()
    loss_a, logits_a = model(input_ids=ids, labels=labels)
    logits_a = logits_a.clone()
    loss_a.backward()
    g_a = model.engine.flat_grads.clone()
    torch.cuda.reset_peak_memory_stats()
    model.recompute_enable()
    assert model.engine.recompute and model.config.recompute
    model.engine.clear_grad()
    loss_b, logits_b = model(input_ids=ids, labels=labels)
    assert len(model.engine._saved["layers"][0]) == 1                  # only the layer input is kept
    assert torch.equal(loss_a.detach(), loss_b.detach()) and torch.equal(logits_a, logits_b)
    loss_b.backward()
    g_b = model.engine.flat_grads
    assert relerr(g_b, g_a) < 2e-3
    model.recompute_disable()
    import paddlenlp_b200.transformers as T
    with pytest.raises(NotImplementedError):
        T.LlamaForCausalLM(T.LlamaConfig(vocab_size=256, hidden_size=256, intermediate_size=512, num_hidden_layers=1,
                                         num_attention_heads=2, recompute=True, recompute_granularity="core_attn"))


def test_left_padded_batch_with_2d_attention_mask():
    """A left-padded batch (the Llama tokenizer default, llama/tokenizer.py:52) with the 2-D attention_mask the reference expands
    to a dense mask (llama/modeling.py:1517-1552, 1683-1699): logits on the real tokens equal the oracle's masked attention,
    and equal the un-padded sequence run alone at the reference's position ids (arange over the padded row)."""
    cfg = tiny_cfg()
    w = make_weights(cfg)
    model = build(cfg, w)
    S, pads = 256, [0, 37, 130]
    g = torch.Generator().manual_seed(13)
    ids = torch.randint(1, cfg.vocab_size, (3, S), generator=g)
    mask = torch.ones(3, S, dtype=torch.int64)
    for b, p in enumerate(pads):
        ids[b, :p] = 0
        mask[b, :p] = 0
    with torch.no_grad():
        logits = model(input_ids=ids.to(DEV), attention_mask=mask.to(DEV))[0].float().cpu()
        plain = model(input_ids=ids.to(DEV))[0].float().cpu()
    assert torch.isfinite(logits).all()
    assert torch.equal(logits[0], plain[0]) or maxerr(logits[0], plain[0]) < 2e-2     # row 0 has no padding
    # oracle with the same start rows
    from paddlenlp_b200.transformers.llama.modeling import _mask_rows_from_padding_mask
    ms = _mask_rows_from_padding_mask(mask)
    wd = {k: v.float() for k, v in w.items()}
    cos, sin = R.rope_tables(cfg.head_dim, S, cfg.rope_theta)
    x = wd["llama.embed_tokens.weight"][ids]
    for i in range(cfg.num_hidden_layers):
        x = R.decoder_layer(x, wd, f"llama.layers.{i}.", cfg, cos, sin, "bf16", mask_start=ms)
    ref = R.linear(R.rms_norm(x, wd["llama.norm.weight"], cfg.rms_norm_eps, "bf16"), wd["lm_head.weight"], None, "bf16")
    for b, p in enumerate(pads):
        e = maxerr(logits[b, p:], ref[b, p:])
        assert e < 3e-2, (b, e)
        if p:
            assert maxerr(plain[b, p:], ref[b, p:]) > 3 * e             # without the mask the padding leaks into the real rows
    # the un-padded sequence alone, at the same absolute positions
    b, p = 2, pads[2]
    pos = torch.arange(p, S)[None]
    with torch.no_grad():
        solo = model(input_ids=ids[b:b + 1, p:].to(DEV), position_ids=pos.to(DEV))[0].float().cpu()
    assert maxerr(logits[b, p:], solo[0]) < 2e-2
    # zeros in the middle of a row are not a padding pattern
    bad = torch.ones(1, S, dtype=torch.int64)
    bad[0, 40:50] = 0
    cfg2 = tiny_cfg()
    model2 = build(cfg2, w)
    with pytest.raises(ValueError):
        model2(input_ids=ids[:1].to(DEV), attention_mask=bad.to(DEV))


def test_llama3_rope_scaling_end_to_end():
    """Llama-3.1 rotary scaling (llama/modeling.py:520-554) through the config: logits vs the oracle with the same tables, and
    different from the unscaled model (the argument is no longer silently ignored, VERDICT r01 weak #12)."""
    import paddlenlp_b200.transformers as T

    sc = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 64}
    cfg = tiny_cfg()
    cfg.rope_scaling = sc
    w = make_weights(cfg)
    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
              max_position_embeddings=cfg.max_position_embeddings)
    scaled = T.LlamaForCausalLM(T.LlamaConfig(rope_scaling=sc, **kw))
    scaled.set_state_dict(w)
    plain = T.LlamaForCausalLM(T.LlamaConfig(**kw))
    plain.set_state_dict(w)
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(17))
    with torch.no_grad():
        a = scaled(input_ids=ids.to(DEV))[0].float().cpu()
        b = plain(input_ids=ids.to(DEV))[0].float().cpu()
    ref16 = R.model_forward(ids, w, cfg, mode="bf16")
    ref32 = R.model_forward(ids, w, cfg, mode="fp32")
    floor_rel = relerr(ref16, ref32)
    assert relerr(a, ref16) <= max(2.0 * floor_rel, 5e-3)
    assert relerr(b, ref16) > 5 * relerr(a, ref16)
