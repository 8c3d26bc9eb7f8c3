"""Tied input / output embeddings on the GPU, through the C-ABI: parity with the tied bf16 oracle, invariance against an
untied model whose head is E^T, gradient accumulation and the data-parallel ready ranges, AdamW, checkpoints, Trainer
resume, generation with every KV cache, and the benchmark width with the real 128 256-token vocabulary.

The tied oracle (tests/tied_oracle.py) is oracle/llama_ref.py with `lm_head.weight` bound to E^T; it is
pinned to HuggingFace with tied embeddings by the golden fixtures tests/golden/{llama,qwen2}_tiny_tied.pt."""
import json
import os

import pytest
import torch

from oracle import llama_ref as R
from oracle import optim_ref
from tied_oracle import bind_head, embed_key, tied_forward, tied_loss_and_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def maxerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


def ulp_bf16(x):
    """One bf16 ulp at |x| (the spacing of bf16 values at that magnitude); 2^-133 at zero."""
    a = x.float().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def tiny_cfg(model_type="llama"):
    return R.RefConfig(vocab_size=1024, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                       num_attention_heads=2, num_key_value_heads=1, rms_norm_eps=1e-5 if model_type == "llama" else 1e-6,
                       rope_theta=500000.0 if model_type == "llama" else 1e6, qkv_bias=(model_type == "qwen2"),
                       model_type=model_type, max_position_embeddings=512)


def hf_kw(cfg):
    return dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                num_key_value_heads=cfg.num_key_value_heads, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta,
                max_position_embeddings=cfg.max_position_embeddings)


def config(cfg, tied=True, **extra):
    import paddlenlp_b200.transformers as T

    C = T.Qwen2Config if cfg.model_type == "qwen2" else T.LlamaConfig
    return C(tie_word_embeddings=tied, **hf_kw(cfg), **extra)


def build(cfg, weights, tied=True):
    import paddlenlp_b200.transformers as T

    M = T.Qwen2ForCausalLM if cfg.model_type == "qwen2" else T.LlamaForCausalLM
    model = M(config(cfg, tied))
    model.set_state_dict(weights)
    return model


def make_weights(cfg, seed=3, scale=3.0):
    """Oracle init without a head; non-trivial norm weights; larger matrices for decisive logits."""
    w = R.init_weights(cfg, seed=seed)
    w.pop("lm_head.weight")
    g = torch.Generator().manual_seed(seed + 100)
    for k in w:
        if "norm" in k:
            w[k] = (1.0 + 0.1 * torch.randn(w[k].shape, generator=g)).to(BF16).float()
        elif k.endswith("proj.weight") or "embed" in k:
            w[k] = (w[k] * scale).to(BF16).float()
    return w


def batch(cfg, B, S, seed):
    tok = torch.randint(0, cfg.vocab_size, (B, S + 1), generator=torch.Generator().manual_seed(seed))
    ids, labels = tok[:, :-1].clone(), tok[:, 1:].clone()          # clones: at B = 1 the slices are contiguous views
    labels[0, :7] = -100
    return ids, labels


def _chunked_linear(x, wt, bias, mode):
    """R.linear with K summed in 4 chunks: the same rounding points, another fp32 accumulation order."""
    K = wt.shape[0]
    step = (K + 3) // 4
    y = None
    for s0 in range(0, K, step):
        part = x[..., s0:s0 + step] @ wt[s0:s0 + step]
        y = part if y is None else y + part
    if bias is not None:
        y = y + bias
    return R.rnd(y, mode)


def reordered_grads(ids, labels, w, cfg):
    orig = R.linear
    R.linear = _chunked_linear
    try:
        return tied_loss_and_grads(ids, labels, w, cfg, mode="bf16")[2]
    finally:
        R.linear = orig


def check_logits(tag, logits, ref16, ref32):
    floor, floor_rel = maxerr(ref16, ref32), relerr(ref16, ref32)
    e_max, e_rel, e32 = maxerr(logits, ref16), relerr(logits, ref16), relerr(logits, ref32)
    print(f"[{tag}] logits vs bf16-oracle max {e_max:.2e} rel {e_rel:.2e}; vs fp32-oracle rel {e32:.2e}; "
          f"floor max {floor:.2e} rel {floor_rel:.2e}")
    assert e32 <= 1.25 * floor_rel + 1e-3
    assert e_max <= max(2.0 * floor, 4e-3)
    assert e_rel <= max(2.0 * floor_rel, 5e-3)
    am, am_ref = logits.argmax(-1), ref16.argmax(-1)
    top2 = ref16.topk(2, dim=-1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 2 * e_max * ref16.abs().max()
    agree = am == am_ref
    print(f"[{tag}] argmax agreement {agree.float().mean().item():.4f}; decisive {decisive.float().mean().item():.3f}")
    assert bool(agree[decisive].all()) and agree.float().mean().item() > 0.95


# ------------------------------------------------------------------------------------------------------------------
# parity with the tied oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tied_logits_loss_argmax_and_grads(model_type):
    cfg = tiny_cfg(model_type)
    w = make_weights(cfg)
    model = build(cfg, w)
    assert model.engine.tied and "lm_head.weight" not in dict(model.named_parameters())
    ids, labels = batch(cfg, 2, 256, 1234)
    with torch.no_grad():
        logits = model(input_ids=ids.to(DEV))[0].float().cpu()
    ref16 = tied_forward(ids, w, cfg, "bf16")
    ref32 = tied_forward(ids, w, cfg, "fp32")
    check_logits(f"tied {model_type}", logits, ref16, ref32)
    loss, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    ref_loss = R.criterion(ref16, labels)
    assert abs(loss.item() - ref_loss.item()) <= 1e-3 * abs(ref_loss.item())
    model.engine.clear_grad()
    loss.backward()
    _, _, gref = tied_loss_and_grads(ids, labels, w, cfg, "bf16")
    gref2 = reordered_grads(ids, labels, w, cfg)
    grads = {k: v.grad.float().cpu() for k, v in model.named_parameters()}
    assert set(grads) == set(gref)
    for k, gr in gref.items():
        e, floor = relerr(grads[k], gr), relerr(gref2[k], gr)
        print(f"[tied {model_type}] grad {k}: rel err {e:.2e}; oracle re-ordering floor {floor:.2e}")
        assert e < max(3e-2, 2.0 * floor), (k, e, floor)


# ------------------------------------------------------------------------------------------------------------------
# invariance: tied == untied with head = E^T
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_type", ["llama", "qwen2"])
def test_tied_equals_untied_with_head_set_to_embedding_transpose(model_type):
    cfg = tiny_cfg(model_type)
    w = make_weights(cfg, seed=9)
    E = embed_key(cfg)
    tied = build(cfg, w, tied=True)
    untied = build(cfg, {**w, "lm_head.weight": w[E].t().contiguous()}, tied=False)
    ids, labels = batch(cfg, 2, 256, 77)
    with torch.no_grad():
        lt = tied(input_ids=ids.to(DEV))[0].float()
        lu = untied(input_ids=ids.to(DEV))[0].float()
    diff = (lt - lu).abs()
    n_diff = int((diff > 0).sum())
    print(f"[{model_type}] tied vs untied(E^T) logits: {'bit-identical' if n_diff == 0 else f'{n_diff} elements differ'}; "
          f"max |diff| / ulp {float((diff / ulp_bf16(lu)).max()):.2f}")
    assert bool((diff <= ulp_bf16(torch.maximum(lt.abs(), lu.abs()))).all())
    # The two head GEMMs read the same values and sum over K in the same k-block order, so the logits are expected to be
    # bit-identical (E as the K-major B operand vs head = E^T as the MN-major one); everything downstream of them then is too.
    assert n_diff == 0, "tied and untied head GEMMs no longer agree bit for bit"
    outs = {}
    for name, m in (("tied", tied), ("untied", untied)):
        m.engine.clear_grad()
        loss, _ = m(input_ids=ids.to(DEV), labels=labels.to(DEV))
        loss.backward()
        outs[name] = (float(loss), {k: v.clone() for k, v in m.engine.named_views(grads=True).items()})
    (loss_t, gt), (loss_u, gu) = outs["tied"], outs["untied"]
    print(f"[{model_type}] loss tied {loss_t!r} untied {loss_u!r}")
    assert loss_t == loss_u
    assert set(gt) == set(gu) - {"lm_head.weight"}
    for k in gt:
        if k != E:
            assert torch.equal(gt[k], gu[k]), k
    # g_E(tied) = g_E(untied) + g_head(untied)^T, up to the bf16 roundings of the sums: the tied buffer starts from the rounded
    # head term and the lookup's scatter adds one rounded bf16 atomic per token of each row, so every partial sum of a row
    # is rounded once more (its magnitude can exceed the final value's; the bound uses the row's largest term).
    want = gu[E].float() + gu["lm_head.weight"].float().t()
    err = (gt[E].float() - want).abs()
    cnt = torch.bincount(ids.reshape(-1).to(DEV), minlength=cfg.vocab_size).float()[:, None]
    unseen = cnt[:, 0] == 0
    # rows of tokens absent from the batch hold the head term alone (reported: is the [V, h] GEMM the transposed [h, V] one?)
    n_unseen_diff = int((gt[E][unseen] != gu["lm_head.weight"].t()[unseen]).sum())
    mag = (gu[E].float().abs() + gu["lm_head.weight"].float().t().abs()).amax(dim=1, keepdim=True)
    bound = (cnt + 2) * ulp_bf16(mag)
    print(f"[{model_type}] g_E tied vs g_E + g_head^T: max err / bound {float((err / bound).max()):.3f}, "
          f"rel {relerr(gt[E], want):.2e}; rows without a token: {n_unseen_diff} elements differ from g_head^T")
    assert bool((err <= bound).all())
    assert relerr(gt[E], want) < 8e-3


# ------------------------------------------------------------------------------------------------------------------
# accumulation, clear_grad, data-parallel ready ranges, AdamW
# ------------------------------------------------------------------------------------------------------------------
def test_tied_accumulation_then_clear_grad():
    """Two micro-batches accumulate both gradient terms of E once each; clear_grad() and a fresh step hold one batch's."""
    cfg = tiny_cfg("qwen2")
    w = make_weights(cfg, seed=21)
    model = build(cfg, w)
    eng = model.engine
    mbs = [batch(cfg, 1, 256, s) for s in (5, 6)]

    def step(ids, labels, scale=1.0):
        loss, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
        (loss * scale).backward()

    single = []
    for ids, labels in mbs:
        eng.clear_grad()
        step(ids, labels)
        single.append(eng.flat_grads.float().clone())
    eng.clear_grad()
    for ids, labels in mbs:
        step(ids, labels, 0.5)
    acc = eng.named_views(grads=True, flat=eng.flat_grads.float())
    want = eng.named_views(flat=(single[0] + single[1]) * 0.5)
    for k in want:
        e = relerr(acc[k], want[k])
        assert e < 1e-2, (k, e)
    # a zeroed or doubled head term of either micro-batch would move g_E by a large fraction of that term
    E = embed_key(cfg)
    head_term = eng.named_views(flat=single[0])[E].norm() / want[E].norm()
    print(f"accumulated g_E rel err {relerr(acc[E], want[E]):.2e} (one micro-batch's g_E is {float(head_term):.2f} of the sum)")
    eng.clear_grad()
    step(*mbs[0])
    fresh = eng.named_views(flat=eng.flat_grads.float())
    ref = eng.named_views(flat=single[0])
    for k in ref:
        assert relerr(fresh[k], ref[k]) < 1e-2, k


def test_tied_grad_ready_ranges():
    cfg = tiny_cfg("llama")
    model = build(cfg, make_weights(cfg, seed=4))
    eng = model.engine
    ids, labels = batch(cfg, 2, 128, 8)
    seen = []
    eng.clear_grad()
    eng.grad_ready_hook = lambda lo, hi: seen.append((lo, hi))
    loss, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    loss.backward()
    pos = 0
    for lo, hi in sorted(seen):
        assert lo == pos and hi > lo, seen
        pos = hi
    assert pos == eng.numel
    mats = [r for r in seen if r[0] < eng.decay_end]
    assert mats[-1] == eng._range("embed", "embed") and len(mats) == cfg.num_hidden_layers + 1
    assert seen[-1] == (eng.decay_end, eng.numel)


def test_tied_adamw_step_vs_optim_ref():
    from paddlenlp_b200.optimizer import AdamW, ClipGradByGlobalNorm

    cfg = tiny_cfg("qwen2")
    w = make_weights(cfg, seed=13)
    model = build(cfg, w)
    eng = model.engine
    ids, labels = batch(cfg, 2, 128, 14)
    eng.clear_grad()
    loss, _ = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    loss.backward()
    opt = AdamW(learning_rate=1e-3, weight_decay=0.1, grad_clip=ClipGradByGlobalNorm(1.0), engine=eng)
    master0 = opt.master.clone().cpu()
    grads = eng.flat_grads.float().cpu()
    opt.step()
    torch.cuda.synchronize()
    mask = torch.arange(eng.numel) < eng.decay_end
    assert bool(mask[eng._range("embed", "embed")[0]])          # E is weight-decayed
    p, m, v, _ = optim_ref.adamw_step(master0, torch.zeros_like(master0), torch.zeros_like(master0), grads, lr=1e-3,
                                      beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.1, step=1, decay_mask=mask,
                                      max_grad_norm=1.0)
    assert relerr(opt.master.cpu(), p) < 1e-6
    # fp32 kernel arithmetic: (1 - beta2) formed from an fp32 beta2 is 1.3e-5 off the fp64 value the reference uses
    assert relerr(opt.exp_avg.cpu(), m) < 1e-5 and relerr(opt.exp_avg_sq.cpu(), v) < 3e-5
    # the update follows the tied oracle's gradient: sign agreement wherever the gradient is above bf16 noise
    _, _, gref = tied_loss_and_grads(ids, labels, w, cfg, "bf16")
    upd = eng.named_views(flat=(opt.master.cpu() - master0))
    for k in (embed_key(cfg), "qwen2.layers.1.mlp.down_proj.weight"):
        g = gref[k]
        big = g.abs() > 0.1 * g.abs().max()
        agree = (torch.sign(upd[k][big]) == -torch.sign(g[big])).float().mean().item()
        assert agree > 0.95, (k, agree)


# ------------------------------------------------------------------------------------------------------------------
# checkpoints
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stray_head", [False, True])
def test_tied_hf_checkpoint_from_pretrained_reproduces_oracle(tmp_path, stray_head):
    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.transformers import conversion_utils as cu

    cfg = tiny_cfg("llama")
    w = make_weights(cfg, seed=17)
    hf = R.to_hf_state_dict(w, cfg)
    assert "lm_head.weight" not in hf
    if stray_head:
        hf["lm_head.weight"] = torch.randn(cfg.vocab_size, cfg.hidden_size)
    config(cfg).save_pretrained(str(tmp_path))
    cu.save_sharded({k: v.to(BF16) for k, v in hf.items()}, str(tmp_path))
    model = T.LlamaForCausalLM.from_pretrained(str(tmp_path))
    assert model.engine.tied
    ids, _ = batch(cfg, 2, 128, 18)
    with torch.no_grad():
        logits = model(input_ids=ids.to(DEV))[0].float().cpu()
    check_logits("from_pretrained tied", logits, tied_forward(ids, w, cfg, "bf16"), tied_forward(ids, w, cfg, "fp32"))
    out = tmp_path / "saved"
    model.save_pretrained(str(out), hf_format=True)
    saved = cu.load_sharded(str(out))
    assert "lm_head.weight" not in saved and set(saved) == set(hf) - {"lm_head.weight"}


def test_tied_trainer_checkpoint_resume(tmp_path):
    """As test_trainer_gpu.test_checkpoint_resume, for a tied model: no lm_head entries in any checkpoint file, every buffer
    restored bit for bit, the resumed run's first loss equal to the original's bit for bit."""
    import shutil

    import paddlenlp_b200.transformers as T
    from paddlenlp_b200.trainer import Trainer, TrainingArguments
    from paddlenlp_b200.transformers import conversion_utils as cu

    class Toy(torch.utils.data.Dataset):
        def __init__(self):
            self.tok = torch.randint(1, 512, (16, 129), generator=torch.Generator().manual_seed(1234))

        def __len__(self):
            return 16

        def __getitem__(self, i):
            return {"input_ids": self.tok[i, :-1].clone(), "labels": self.tok[i, 1:].clone()}

    def make(out_dir, save_steps=0):
        model = T.Qwen2ForCausalLM(T.Qwen2Config(
            vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
            num_key_value_heads=1, max_position_embeddings=256, seq_length=128, tie_word_embeddings=True))
        args = TrainingArguments(output_dir=str(out_dir), per_device_train_batch_size=2, gradient_accumulation_steps=2,
                                 max_steps=5, learning_rate=1e-3, weight_decay=0.01, warmup_steps=2, logging_steps=1,
                                 max_seq_length=128, lr_scheduler_type="cosine", save_steps=save_steps, save_total_limit=4)
        return Trainer(model=model, args=args, train_dataset=Toy())

    orig = make(tmp_path / "orig", save_steps=1)
    orig.train()
    ck = str(tmp_path / "orig" / "checkpoint-3")
    opt_file = cu.load_sharded(ck, cu.SAFE_OPTIMIZER_NAME, cu.SAFE_OPTIMIZER_INDEX_NAME)
    mw = cu.load_sharded(ck, cu.SAFE_MASTER_WEIGHTS_NAME, cu.SAFE_MASTER_WEIGHTS_INDEX_NAME)
    wt = cu.load_sharded(ck)
    assert not any(k.startswith("lm_head") for k in list(opt_file) + list(mw) + list(wt))
    assert "qwen2.embed_tokens.weight/moment1_0" in opt_file
    assert json.load(open(os.path.join(ck, "config.json")))["tie_word_embeddings"] is True

    probe = make(tmp_path / "probe")
    probe._load_from_checkpoint(ck)
    probe.create_optimizer_and_scheduler(5)
    probe._load_optimizer_and_scheduler(ck)
    assert probe.optimizer.step_count == 3
    for k, v in probe.optimizer.named_optimizer_state().items():
        assert torch.equal(v.cpu(), opt_file[k]), k
    for k, v in probe.optimizer.named_master_weights().items():
        assert torch.equal(v.cpu(), mw[k]), k
    for k, v in probe.model.state_dict().items():
        assert torch.equal(v.cpu(), wt[k]), k

    shutil.copytree(ck, tmp_path / "resumed" / "checkpoint-3")
    res = make(tmp_path / "resumed")
    out = res.train(resume_from_checkpoint=True)
    assert out.global_step == 5 and res.optimizer.step_count == 5
    lo, lr_ = [h["loss"] for h in orig.state.log_history], [h["loss"] for h in res.state.log_history]
    assert lr_[:4] == lo[:4]                                      # restored history + the bit-identical first resumed step
    assert abs(lr_[4] - lo[4]) < 2e-3
    a, b = res.optimizer.master, orig.optimizer.master
    assert ((a - b).norm() / b.norm()).item() < 1e-4


# ------------------------------------------------------------------------------------------------------------------
# generation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cache", ["dense", "paged", "append_attn"])
def test_tied_generation_greedy_matches_uncached_argmax_chain(cache):
    from oracle import generation_ref as G
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = R.RefConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=1, max_position_embeddings=256)
    w = make_weights(cfg, seed=7, scale=4.0)
    lcfg = config(cfg)
    kw = dict(block_attn=cache != "dense", append_attn=cache == "append_attn")
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    im = LlamaForCausalLMInferenceModel(lcfg, **kw)
    m_tied = torch.cuda.memory_allocated() - m0
    um = LlamaForCausalLMInferenceModel(config(cfg, tied=False), **kw)
    m_untied = torch.cuda.memory_allocated() - m0 - m_tied
    assert im.lm_head_weight is None
    assert not any(isinstance(t, torch.Tensor) and tuple(t.shape) == (cfg.hidden_size, cfg.vocab_size)
                   for t in vars(im).values())
    assert m_untied - m_tied == cfg.hidden_size * cfg.vocab_size * 2
    del um
    im.set_state_dict(w)
    im.set_state_dict({**w, "lm_head.weight": torch.zeros(cfg.hidden_size, cfg.vocab_size)})   # a stray head is ignored
    prompt = torch.randint(0, cfg.vocab_size, (4, 20), generator=torch.Generator().manual_seed(3))
    want, margins = G.greedy_generate(prompt, bind_head(w, cfg), cfg, max_new=8)
    out, _, _ = im.generate(prompt, max_length=8)
    out = out.cpu()
    compared = 0
    for b in range(prompt.shape[0]):
        for t in range(8):
            if margins[b, t] < 2e-2:
                break
            assert int(out[b, t]) == int(want[b, t]), (cache, b, t, out[b].tolist(), want[b].tolist())
            compared += 1
    print(f"[{cache}] {compared} decisive greedy tokens identical to the tied oracle's uncached argmax chain")
    assert compared >= 6
    # sampling under the CUDA graph: a seeded draw is reproducible and every token is in the vocabulary
    s1, _, _ = im.generate(prompt, max_length=8, top_p=0.9, temperature=1.0, seed=11)
    s2, _, _ = im.generate(prompt, max_length=8, top_p=0.9, temperature=1.0, seed=11)
    assert torch.equal(s1, s2) and int(s1.min()) >= 0 and int(s1.max()) < cfg.vocab_size


@pytest.mark.parametrize("vocab", [512, 128256])
@pytest.mark.parametrize("rows", [1, 16, 64])
def test_tied_init_random_and_decode_head_reads_embedding(vocab, rows):
    """init_random draws no head; the decode-step head (M <= 64 rows) equals hn @ E^T element by element.  V = 512 takes the
    split-K GEMM; the real vocabulary V = 128 256 (>= 100 column tiles) takes the persistent wgmma kernel with 64-row tiles
    and E as its K-major B operand, which must also agree bit for bit with the untied form (head = E^T, MN-major B)."""
    from paddlenlp_b200 import ops
    from paddlenlp_b200.experimental.transformers import LlamaForCausalLMInferenceModel

    cfg = R.RefConfig(vocab_size=vocab, hidden_size=3072, intermediate_size=256, num_hidden_layers=1, num_attention_heads=24,
                      num_key_value_heads=8, max_position_embeddings=256)
    im = LlamaForCausalLMInferenceModel(config(cfg))
    im.init_random(seed=5)
    assert im.lm_head_weight is None
    g = torch.Generator(device=DEV).manual_seed(rows)
    hidden = torch.randn(rows, cfg.hidden_size, generator=g, device=DEV).to(BF16)
    got = im._head(hidden)
    assert got.shape == (rows, vocab)
    hn, _ = ops.add_rmsnorm(hidden, None, im.norm_weight, cfg.rms_norm_eps, want_residual=False)
    E = im.embed_tokens
    ref = hn.double() @ E.double().t()
    # one bf16 rounding of the result plus the fp32 accumulation allowance of tests/test_kernels_at_scale_gpu.py (c = 9e-6)
    bound = 2.0 ** -8 * ref.abs() + 9e-6 * (hn.double().abs() @ E.double().abs().t())
    err = (got.double() - ref).abs()
    print(f"[decode head V={vocab} M={rows}] max err / bound {float((err / bound).max()):.3f}")
    assert bool(torch.isfinite(got).all()) and bool((err <= bound).all())
    if vocab >= 100 * 256:
        untied = im.transformer_block._mm(hn, E.t().contiguous())
        assert torch.equal(got, untied)


# ------------------------------------------------------------------------------------------------------------------
# benchmark width
# ------------------------------------------------------------------------------------------------------------------
def test_tied_two_layer_llama3_2_3b_width_real_vocab_s4096():
    """Two decoder layers at Llama-3.2-3B width with the real 128 256-token tied head at S = 4096: logits, loss, arg-max and
    gradients (E with both terms) against the tied oracle run on the device; gradient tolerance 2x the oracle's own
    re-ordering floor."""
    cfg = R.RefConfig(vocab_size=128256, hidden_size=3072, intermediate_size=8192, num_hidden_layers=2, num_attention_heads=24,
                      num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, max_position_embeddings=4096)
    w = R.init_weights(cfg, seed=61)
    w.pop("lm_head.weight")
    E = embed_key(cfg)
    w[E] = (w[E] * 8).to(BF16).float()                                    # decisive logits at the 0.02 init scale
    model = build(cfg, w)
    ids, labels = batch(cfg, 1, 4096, 62)
    model.engine.clear_grad()
    loss, logits = model(input_ids=ids.to(DEV), labels=labels.to(DEV))
    logits = logits.float().clone()
    loss.backward()
    wd = {k: v.to(DEV) for k, v in w.items()}
    ids_d, lab_d = ids.to(DEV), labels.to(DEV)
    assert not torch.backends.cuda.matmul.allow_tf32
    with torch.no_grad():
        ref32 = tied_forward(ids_d, wd, cfg, "fp32")
    ref_loss, ref16, gref = tied_loss_and_grads(ids_d, lab_d, wd, cfg, "bf16")
    check_logits("tied 2 layers, V=128256, S=4096", logits, ref16, ref32)
    assert abs(float(loss) - float(ref_loss)) <= 1e-3 * abs(float(ref_loss))
    del ref16, ref32, logits
    gref2 = reordered_grads(ids_d, lab_d, wd, cfg)
    grads = model.engine.named_views(grads=True)
    for k in (E, "llama.norm.weight", "llama.layers.1.mlp.down_proj.weight", "llama.layers.1.self_attn.q_proj.weight",
              "llama.layers.0.self_attn.v_proj.weight", "llama.layers.0.mlp.gate_proj.weight",
              "llama.layers.0.input_layernorm.weight"):
        e, floor = relerr(grads[k], gref[k]), relerr(gref2[k], gref[k])
        print(f"[tied 2 layers, V=128256] grad {k}: rel err {e:.2e}; oracle re-ordering floor {floor:.2e}")
        assert e < max(3e-2, 2.0 * floor), (k, e, floor)
