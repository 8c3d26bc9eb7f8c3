"""The training attention kernels per (row, head) against fp64, with packed-document FlashMask masks at every preset's GQA ratio.

fa_fwd_wgmma_kernel and fa_bwd_wgmma_kernel (reached through ops.flash_attn_fwd / flash_attn_bwd) skip kv tiles and q tiles
from the start rows of packed documents.  A visibility mistake that adds or drops one column of a long document moves that
row's output by about |v| / n, far below a relative error over a whole batch row or a 128-row tile (the existing attention
tests), yet it biases every packed sample of a training run.  The checker here works per element, per (row, head) and, in
the forward, on each row's log-sum-exp, which moves by ~p / n for one column and is exact to fp32 level otherwise.  Its CPU
tests (no gpu mark) run it on a bf16-rounding emulation of the kernels and show that it accepts the emulation and rejects
seven visibility and reduction bugs, and which of them the old whole-row / per-tile checks accept.

Per element, with mag the sum of the same products taken over absolute values:
  O    |err| <= 2^-8 |ref| + c * sum_j p_ij |v_j|
  dV   |err| <= 2^-8 |ref| + c * sum_i p_ij |dO_i|                                   + inherited
  dK   |err| <= 2^-8 |ref| + c * scale sum_i p_ij (|dP_ij| + |D_i|) |q_i|            + inherited + fp32
  dQ   |err| <= 2^-8 |ref| + c * scale sum_j p_ij (|dP_ij| + |D_i|) |k_j|            + inherited + fp32
2^-8 |ref| is the output's one bf16 rounding.  c covers the bf16 rounding of P (forward, dV) or dS (dK, dQ) before their
matmuls: half an ulp, at most 2^-8 of the value, so c = 2^-8, plus 2^-12 for the fp32 arithmetic and the output rounding of
the error itself.  The backward reads the forward's bf16 o and fp32 lse: the inherited terms are the exact effect of their
measured errors (D from o, P from lse) on the same sums.  The reference takes D from the exact O.  The fp32 terms bound the
dot products dP = dO V^T and D = rowsum(dO o), which cancel to ~0 on some rows: d 2^-23 (|dO| |V|^T + rowsum |dO o|).
"""
import math

import pytest
import torch

from oracle import llama_ref as R

DEV = "cuda:0"
BF16 = torch.bfloat16
F64 = torch.float64
BF16_REL = 2.0 ** -8           # one bf16 rounding: at most half an ulp, <= 2^-8 of the value rounded
# Measured on an H100 80GB HBM3 at a 700 W power limit over every GPU case below (impl 2 and impl 1):
# One bf16 rounding of P or dS before the matmul (2^-8) plus 2^-12 of room for the fp32 arithmetic.  c_need <= 3.3e-3 (O),
# 3.2e-3 (dQ), 2.8e-3 (dK), 3.8e-3 (dV, q = 0 at 128 x 300); worst element error / bound 0.97.
C_FWD = C_BWD = 2.0 ** -8 + 2.0 ** -12
# fp32 dot products of d terms (dP = dO V^T and D = rowsum(dO o) in the backward): at most d * 2^-23 of sum |a_i b_i|
FP32_DOT = 2.0 ** -23
# Relative Frobenius error of one (row, head): ||err|| / (||ref|| + 2^-8 ||mag|| + ||inherited||); the floor keeps rows
# whose exact value cancels to ~0 (dQ and dK of short documents, rows dominated by one planted column) judged by the size of
# what rounds in them.  Measured worst with N(0, 1) scores (and q = 0): O 3.7e-3, dV 4.7e-3, dK 1.8e-2, dQ 0.57 (a
# two-token document, where dQ = scale dS_1 (k_1 - k_0) cancels).  With planted, sink and rising logits the rows dominated
# by one column cancel in dK (0.25) and dQ (0.91); there the per-element bound carries the check of dQ.
HEAD_TOL = dict(o=6e-3, dq=0.85, dk=3e-2, dv=8e-3)
HEAD_TOL_SHAPED = dict(o=6e-3, dq=1.2, dk=0.4, dv=8e-3)
# LSE per (row, head), absolute: fp32 scores (their rounding grows with the largest score, which |LSE| follows), ex2.approx
# terms (~2^-22 relative) and one fp32 rescale and add per 128-column tile summed, then (m + log2 l) ln 2:
# 2^-20 (|LSE| + 2) + 2^-22 * tiles.  About 1.8e-5 at 4 096 columns of N(0, 1) scores.  Measured: |err| <= 1.5e-6 with
# N(0, 1) scores (0.20 of the bound), <= 7.6e-6 with +10 logits (0.54 of the bound).
LSE_ULP = 2.0 ** -20
LSE_TILE = 2.0 ** -22
# q = 0: P is exactly 1 on the visible set, so LSE = ln(count) to one fp32 log, and O = the mean of the visible V rows to
# fp32 sums (each element within 2^-14 of mean |v|) and one bf16 rounding.  Measured: LSE 0.10 and O 0.98 of the bound
# (the bf16 rounding alone reaches 0.98 in the CPU emulation).
EXACT_LSE = 2.0 ** -20
EXACT_C = 2.0 ** -14
# The checks the older attention tests apply
OLD_ROW, OLD_TILE, OLD_LSE = 2e-2, 1e-2, 2e-3

PLANT = 10.0                   # logit added to planted columns


def ops():
    from paddlenlp_b200 import ops as _ops

    return _ops


# ----------------------------------------------------------------------------------------------------------
# Masks
# ----------------------------------------------------------------------------------------------------------
def canonical(raw):
    """Start rows as the engine hands them to the kernels: every column visible at least to its own row."""
    S = raw.shape[-1]
    return torch.maximum(raw.to(torch.int32), torch.arange(1, S + 1, dtype=torch.int32, device=raw.device))


def doc_mask(doc_lens):
    out, pos = [], 0
    for n in doc_lens:
        out += [pos + n] * n
        pos += n
    return torch.tensor(out, dtype=torch.int32)


def visible(ms, B, S, device):
    """[B, S(row), S(col)] bool: c <= r and r < ms[b, c] (ms None: plain causal)."""
    r = torch.arange(S, device=device)[:, None]
    c = torch.arange(S, device=device)[None, :]
    vis = (c <= r)[None].expand(B, S, S)
    if ms is not None:
        vis = vis & (r[None] < ms.to(device).long()[:, None, :])
    return vis


def pipeline_mask(S, B, seed, greedy, lo=8, hi=1500, pack_len=None, front=(), empty_rows=()):
    """Start rows from the SFT pipeline: seeded records of log-uniform lengths (after `front`), packed by
    ZeroPaddingMapDataset into pack_len rows, right-padded to S by DataCollatorForSeq2Seq.  Returns (raw, canonical)."""
    from paddlenlp_b200.data import DataCollatorForSeq2Seq
    from paddlenlp_b200.datasets import ZeroPaddingMapDataset

    pack_len = pack_len or S
    g = torch.Generator().manual_seed(seed)
    mean = (hi - lo) / math.log(hi / lo)
    n_rec = int(3 * B * pack_len / mean) + 600
    lens = list(front) + torch.exp(torch.empty(n_rec).uniform_(math.log(lo), math.log(hi), generator=g)).long().tolist()
    recs = [{"input_ids": [1] * n, "labels": [1] * n} for n in lens]
    ds = ZeroPaddingMapDataset(recs, max_length=pack_len, greedy_zero_padding=greedy)
    assert len(ds) >= B
    feats = [ds[i] for i in range(B)]
    for i in empty_rows:
        feats[i] = {"input_ids": [], "labels": [], "position_ids": [], "attn_mask_startend_row_indices": []}
    raw = DataCollatorForSeq2Seq(max_length=S, pad_token_id=0)(feats)["attn_mask_startend_row_indices"]
    return raw, canonical(raw)


# ----------------------------------------------------------------------------------------------------------
# fp64 reference
# ----------------------------------------------------------------------------------------------------------
def reference(q, k, v, dout, ms, scale, o=None, lse=None, elems=2 ** 26):
    """fp64 causal GQA attention with FlashMask start rows ms [B, S] (canonical, or None), and its exact gradients.

    q [B, S, nh, d], k / v [B, S, kvh, d], dout [B, S, nh, d] or None (forward only).  o / lse: the forward outputs the
    kernel backward read; their measured errors give the inherited terms.  Vectorised over blocks of query rows and one kv
    head's group at a time ([G, rows, cols] fp64 matrices of at most `elems` elements).  Returns a dict of fp64 tensors:
    O, magO, dQ, magdQ, inhdQ [B, S, nh, d]; dK, magdK, inhdK, dV, magdV, inhdV [B, S, kvh, d]; LSE [B, nh, S]."""
    B, S, nh, d = q.shape
    kvh = k.shape[2]
    G = nh // kvh
    dev = q.device
    z = lambda h: torch.zeros(B, S, h, d, dtype=F64, device=dev)   # noqa: E731
    out = dict(O=z(nh), magO=z(nh), LSE=torch.zeros(B, nh, S, dtype=F64, device=dev))
    if dout is not None:
        out.update(dQ=z(nh), magdQ=z(nh), inhdQ=z(nh), dK=z(kvh), magdK=z(kvh), inhdK=z(kvh), dV=z(kvh), magdV=z(kvh),
                   inhdV=z(kvh))
    rows = max(16, min(S, elems // (G * S)))
    for b in range(B):
        msb = None if ms is None else ms[b].to(dev).long()
        for h in range(kvh):
            hs = slice(h * G, (h + 1) * G)
            Kh, Vh = k[b, :, h].to(F64), v[b, :, h].to(F64)
            for r0 in range(0, S, rows):
                r1 = min(S, r0 + rows)
                Kc, Vc = Kh[:r1], Vh[:r1]
                qb = q[b, r0:r1, hs].to(F64).transpose(0, 1)                       # [G, R, d]
                r = torch.arange(r0, r1, device=dev)[:, None]
                c = torch.arange(r1, device=dev)[None, :]
                vis = c <= r
                if msb is not None:
                    vis = vis & (r < msb[None, :r1])
                s = torch.matmul(qb, Kc.T).mul_(scale).masked_fill_(~vis, -math.inf)
                L = torch.logsumexp(s, dim=-1)                                      # [G, R]
                p = s.sub_(L[..., None]).exp_()
                del s
                O = p @ Vc
                out["O"][b, r0:r1, hs] = O.transpose(0, 1)
                out["magO"][b, r0:r1, hs] = (p @ Vc.abs()).transpose(0, 1)
                out["LSE"][b, hs, r0:r1] = L
                if dout is None:
                    continue
                dob = dout[b, r0:r1, hs].to(F64).transpose(0, 1)
                dD = torch.zeros_like(L) if o is None else ((o[b, r0:r1, hs].to(F64).transpose(0, 1) - O) * dob).sum(-1).abs()
                dl = torch.zeros_like(L) if lse is None else (lse[b, hs, r0:r1].to(F64) - L).abs()
                dp = dob @ Vc.T
                D = (dob * O).sum(-1)
                ds = p * (dp - D[..., None])
                w = p * (dp.abs_() + D.abs()[..., None])                            # p (|dP| + |D|)
                del dp
                # absolute terms: D from o, P from lse, and the fp32 dot products dP = dO V^T and D = rowsum(dO o), which
                # may cancel to ~0 (one-token documents, rows dominated by one column) and so are not relative to |dP|, |D|
                a = (dob.abs() @ Vc.abs().T).add_((dob.abs() * O.abs()).sum(-1)[..., None]).mul_(p).mul_(FP32_DOT * d)
                w2 = a.add_(p * dD[..., None]).add_(w * dl[..., None])
                pdl = p * dl[..., None]
                qa, doa, Ka = qb.abs(), dob.abs(), Kc.abs()
                out["dV"][b, :r1, h] += (p.transpose(1, 2) @ dob).sum(0)
                out["magdV"][b, :r1, h] += (p.transpose(1, 2) @ doa).sum(0)
                out["inhdV"][b, :r1, h] += (pdl.transpose(1, 2) @ doa).sum(0)
                out["dK"][b, :r1, h] += scale * (ds.transpose(1, 2) @ qb).sum(0)
                out["magdK"][b, :r1, h] += scale * (w.transpose(1, 2) @ qa).sum(0)
                out["inhdK"][b, :r1, h] += scale * (w2.transpose(1, 2) @ qa).sum(0)
                out["dQ"][b, r0:r1, hs] = (scale * (ds @ Kc)).transpose(0, 1)
                out["magdQ"][b, r0:r1, hs] = (scale * (w @ Ka)).transpose(0, 1)
                out["inhdQ"][b, r0:r1, hs] = (scale * (w2 @ Ka)).transpose(0, 1)
                del p, ds, w, w2, pdl
    return out


# ----------------------------------------------------------------------------------------------------------
# Checker
# ----------------------------------------------------------------------------------------------------------
def _check_elems(name, got, ref, mag, inh, c, head_tol, what):
    """got [B, S, H, d] against ref; returns the report, raises AssertionError on a violation."""
    fin = torch.isfinite(got)
    if not bool(fin.all()):
        b, s, h, _ = (~fin).nonzero()[0].tolist()
        raise AssertionError(f"{what} {name}: {int((~fin).sum())} non-finite (unwritten?) outputs, first at batch row {b} "
                             f"row {s} head {h}")
    err = (got.to(F64) - ref).abs_()
    rnd = BF16_REL * ref.abs()
    if inh is not None:
        rnd = rnd + inh
    ratio = (err / (rnd + c * mag).clamp_min_(1e-300)).amax(-1)                       # [B, S, H]
    c_need = ((err - rnd).clamp_min_(0) / mag.clamp_min(1e-300)).max().item()
    floor = BF16_REL * mag.norm(dim=-1) + (0 if inh is None else inh.norm(dim=-1))
    head = err.norm(dim=-1) / (ref.norm(dim=-1) + floor).clamp_min_(1e-300)
    del err, rnd, floor
    i = int(ratio.argmax())
    j = int(head.argmax())
    H = got.shape[2]
    S = got.shape[1]
    rep = dict(ratio=ratio.max().item(), at=(i // (S * H), i // H % S, i % H), c_need=c_need, head=head.max().item(),
               head_at=(j // (S * H), j // H % S, j % H))
    print(f"  [{what}] {name}: worst error / bound {rep['ratio']:.3f} at (b, row, head) {rep['at']}, c_need "
          f"{c_need:.2e} (c {c:.2e}), worst (row, head) rel. error {rep['head']:.2e} at {rep['head_at']}")
    assert rep["ratio"] <= 1.0, f"{what} {name}: element error exceeds its bound: {rep}"
    assert rep["head"] <= head_tol, f"{what} {name}: (row, head) relative error exceeds {head_tol}: {rep}"
    return rep


def lse_tol(L):
    S = L.shape[-1]
    tiles = (torch.arange(S, device=L.device) // 128 + 1).to(F64)
    return LSE_ULP * (L.abs() + 2) + LSE_TILE * tiles


def check_forward(o, lse, ref, what, c=C_FWD, head_tol=HEAD_TOL):
    """o [B, S, nh, d] bf16, lse [B, nh, S] fp32 against reference(); per element, per (row, head), LSE per (row, head)."""
    rep = dict(o=_check_elems("O", o, ref["O"], ref["magO"], None, c, head_tol["o"], what))
    if not bool(torch.isfinite(lse).all()):
        raise AssertionError(f"{what} LSE: non-finite values")
    e = (lse.to(F64) - ref["LSE"]).abs_()
    m = e / lse_tol(ref["LSE"])
    i = int(m.argmax())
    B, H, S = lse.shape
    rep["lse"] = dict(ratio=m.max().item(), err=e.max().item(), at=(i // (H * S), i % S, i // S % H))
    print(f"  [{what}] LSE: worst |err| {rep['lse']['err']:.2e}, error / bound {rep['lse']['ratio']:.3f} at (b, row, head) "
          f"{rep['lse']['at']}")
    assert rep["lse"]["ratio"] <= 1.0, f"{what} LSE: error exceeds its bound: {rep['lse']}"
    return rep


def check_backward(dq, dk, dv, ref, what, c=C_BWD, head_tol=HEAD_TOL):
    return dict(dq=_check_elems("dQ", dq, ref["dQ"], ref["magdQ"], ref["inhdQ"], c, head_tol["dq"], what),
                dk=_check_elems("dK", dk, ref["dK"], ref["magdK"], ref["inhdK"], c, head_tol["dk"], what),
                dv=_check_elems("dV", dv, ref["dV"], ref["magdV"], ref["inhdV"], c, head_tol["dv"], what))


def check_exact_visibility(o, lse, v, ms, what):
    """q = 0: every visible score is 0 and P is exactly 1, so for every (batch row, row, head) LSE = ln(count) and O = the
    mean of the visible V rows.  The visible set of row r is the columns [first(r), r], first(r) = the first column whose
    start row exceeds r (start rows are non-decreasing)."""
    B, S, nh, d = o.shape
    kvh = v.shape[2]
    G = nh // kvh
    dev = o.device
    r = torch.arange(S, device=dev)
    worst_l, worst_o = 0.0, 0.0
    for b in range(B):
        first = torch.zeros(S, dtype=torch.long, device=dev) if ms is None else \
            torch.searchsorted(ms[b].to(dev).long().contiguous(), r, right=True)
        n = (r - first + 1).to(F64)
        lt = lse[b].to(F64) - torch.log(n)[None]
        tol = EXACT_LSE * torch.log(n).clamp_min(1.0)
        bad = (lt.abs() > tol[None])
        worst_l = max(worst_l, (lt.abs() / tol[None]).max().item())
        if bool(bad.any()):
            h, i = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: LSE of batch row {b} row {i} head {h} is {lse[b, h, i].item():.7f}, ln(count) = "
                                 f"{math.log(n[i].item()):.7f} (count {int(n[i])})")
        vb = v[b].to(F64)                                                       # [S, kvh, d]
        cs = torch.cat([torch.zeros(1, kvh, d, dtype=F64, device=dev), vb.cumsum(0)])
        ca = torch.cat([torch.zeros(1, kvh, d, dtype=F64, device=dev), vb.abs().cumsum(0)])
        mean = ((cs[r + 1] - cs[first]) / n[:, None, None]).repeat_interleave(G, dim=1)
        mabs = ((ca[r + 1] - ca[first]) / n[:, None, None]).repeat_interleave(G, dim=1)
        err = (o[b].to(F64) - mean).abs()
        m = err / (BF16_REL * mean.abs() + EXACT_C * mabs)
        worst_o = max(worst_o, m.max().item())
        if not bool(torch.isfinite(o[b].float()).all()) or bool((m > 1).any()):
            i, h, _ = (~(m <= 1)).nonzero()[0].tolist()
            raise AssertionError(f"{what}: O of batch row {b} row {i} head {h} is not the mean of its {int(n[i])} visible V rows")
    print(f"  [{what}] exact visibility: LSE error / bound {worst_l:.3f}, O error / bound {worst_o:.3f}")
    return worst_l, worst_o


def old_checks(got, ref, tile):
    """The older attention tests' acceptance, per batch row: relative Frobenius error <= 2e-2, and <= 1e-2 over every
    `tile` rows of one head.  Returns True when they accept."""
    for b in range(got.shape[0]):
        a, r = got[b].to(F64), ref[b]
        if ((a - r).norm() / r.norm()).item() >= OLD_ROW:
            return False
        S, H = a.shape[0], a.shape[1]
        idx = torch.arange(S, device=a.device) // tile
        nt = (S + tile - 1) // tile
        e2 = torch.zeros(nt, H, dtype=F64, device=a.device).index_add_(0, idx, (a - r).pow(2).sum(-1))
        r2 = torch.zeros(nt, H, dtype=F64, device=a.device).index_add_(0, idx, r.pow(2).sum(-1))
        if (e2 / r2.clamp_min(1e-300)).sqrt().max().item() >= OLD_TILE:
            return False
    return True


# ----------------------------------------------------------------------------------------------------------
# CPU: a bf16-rounding emulation of the kernels, and the checker against it
# ----------------------------------------------------------------------------------------------------------
def emulate(q, k, v, dout, ms, scale, vis_fwd=None, vis_bwd=None, dq_drop=None, route=None):
    """The kernels' rounding points: forward P~ = exp(s - m) rounded to bf16 before P~ V, l = sum P~ unrounded,
    o = bf16(P~ V / l), lse = fp32(m + ln l); backward P = exp(s - lse), dS = P (dO V^T - rowsum(dO o)), P and dS rounded
    to bf16 before the gradient matmuls, fp32-exact sums, outputs rounded to bf16 once.
    Sabotage hooks: vis_fwd / vis_bwd [B, nh, S, S] replace the visible set of either pass; dq_drop [B, nh, S, S] pairs whose
    dS is left out of dQ; route[h] the kv head that q head h's dK / dV go to (None: dropped)."""
    B, S, nh, d = q.shape
    kvh = k.shape[2]
    G = nh // kvh
    base = visible(ms, B, S, q.device)[:, None].expand(B, nh, S, S)
    vis_fwd = base if vis_fwd is None else vis_fwd
    vis_bwd = vis_fwd if vis_bwd is None else vis_bwd
    r16 = lambda x: x.to(BF16).to(F64)   # noqa: E731
    qh = q.to(F64).transpose(1, 2)
    kh = k.to(F64).repeat_interleave(G, dim=2).transpose(1, 2)
    vh = v.to(F64).repeat_interleave(G, dim=2).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * scale
    sf = s.masked_fill(~vis_fwd, -math.inf)
    m = sf.amax(-1, keepdim=True)
    pt = (sf - m).exp()
    lsum = pt.sum(-1, keepdim=True)
    oh = r16((r16(pt) @ vh) / lsum)
    lse = (m + lsum.log()).squeeze(-1).float()                                  # [B, nh, S]
    o = oh.transpose(1, 2).to(BF16)
    doh = dout.to(F64).transpose(1, 2)
    P = (s - lse.to(F64)[..., None]).exp().masked_fill(~vis_bwd, 0.0)
    D = (doh * oh).sum(-1, keepdim=True)
    dS = r16(P * (doh @ vh.transpose(-1, -2) - D))
    dq = scale * (dS.masked_fill(dq_drop, 0.0) if dq_drop is not None else dS) @ kh
    dvh = r16(P).transpose(-1, -2) @ doh                                        # [B, nh, S, d] per q head
    dkh = scale * dS.transpose(-1, -2) @ qh
    route = [h // G for h in range(nh)] if route is None else route
    dk = torch.zeros(B, kvh, S, d, dtype=F64)
    dv = torch.zeros(B, kvh, S, d, dtype=F64)
    for h in range(nh):
        if route[h] is not None:
            dk[:, route[h]] += dkh[:, h]
            dv[:, route[h]] += dvh[:, h]
    t = lambda x: x.transpose(1, 2).to(BF16)   # noqa: E731
    return o, lse, t(dq), t(dk), t(dv)


CPU_S, CPU_NH, CPU_KVH, CPU_D = 512, 4, 2, 64
CPU_DOCS = [[100, 200, 87, 1, 1, 123], [64, 383, 65]]


def planted_columns(ms, S, B):
    """[B, S] bool: the last column of every document (start row = c + 1) and the first and last column of every 64-row tile."""
    c = torch.arange(S)
    edge = ((c % 64 == 0) | (c % 64 == 63))[None].expand(B, S)
    if ms is None:
        return edge.clone()
    return edge | (ms.cpu().long() == c[None] + 1)


def doc_first_columns(ms, S, B):
    c = torch.arange(S)
    if ms is None:
        return (c == 0)[None].expand(B, S).clone()
    prev = torch.cat([torch.zeros(B, 1, dtype=torch.long), ms.cpu().long()[:, :-1]], dim=1)
    return (c[None] == 0) | (prev == c[None])


def shape_scores(q, k, kind, ms, scale):
    """Score ranges (in place on bf16 q / k, which may be views): "planted": PLANT added to the logits of planted_columns;
    "sink": PLANT on each document's first column; "rising": logits rising by 16 along the sequence, so that every kv tile
    raises the running maximum; "zero_q": q = 0."""
    B, S, nh, d = q.shape
    if kind == "randn":
        return
    if kind == "zero_q":
        q.zero_()
        return
    a = 4.0
    q[..., 0] = a
    k[..., 0] = 0.0
    col = None
    if kind == "planted":
        col = planted_columns(ms, S, B).to(k.device)
    elif kind == "sink":
        col = doc_first_columns(ms, S, B).to(k.device)
    if col is not None:
        k[..., 0] = torch.where(col, PLANT / (a * scale), 0.0)[..., None].to(k.dtype)
    elif kind == "rising":
        ramp = torch.arange(S, device=k.device, dtype=torch.float32) * (16.0 / (a * scale * S))
        k[..., 0] = ramp[None, :, None].to(k.dtype)
    else:
        raise KeyError(kind)


def cpu_batch(kind="randn", seed=5):
    B, S, nh, kvh, d = 2, CPU_S, CPU_NH, CPU_KVH, CPU_D
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, S, nh, d, generator=g).to(BF16)
    k = torch.randn(B, S, kvh, d, generator=g).to(BF16)
    v = torch.randn(B, S, kvh, d, generator=g).to(BF16)
    dout = torch.randn(B, S, nh, d, generator=g).to(BF16)
    ms = torch.stack([doc_mask(x) for x in CPU_DOCS])
    scale = 1.0 / math.sqrt(d)
    shape_scores(q, k, kind, ms, scale)
    return q, k, v, dout, ms, scale


def first_visible_kv_tile(ms_row, q0, S, bkv=128):
    """fa_fwd.cu's prefix skip: leading kv tiles whose last column's document ends at or before q0."""
    n_kv = (S + bkv - 1) // bkv
    j = 0
    while j < n_kv - 1 and int(ms_row[min(j * bkv + bkv - 1, S - 1)]) <= q0:
        j += 1
    return j


def sabotage(name, q, k, v, dout, ms, scale):
    """Emulated kernel outputs with one bug; returns (o, lse, dq, dk, dv)."""
    B, S, nh, d = q.shape
    vis = visible(ms, B, S, q.device)[:, None].expand(B, nh, S, S).clone()
    if name == "row sees one column past its diagonal":
        r = 382                                              # batch row 1, document [64, 447): column 383 is a tile edge
        vis[1, :, r, r + 1] = True
        return emulate(q, k, v, dout, ms, scale, vis_fwd=vis)
    if name == "document's first row sees the previous document's last column":
        vis[0, :, 300, 299] = True
        return emulate(q, k, v, dout, ms, scale, vis_fwd=vis)
    if name == "one kv tile too many skipped":
        q0 = 256                                             # batch row 0, q tile 2: its first visible kv tile is hidden
        j = first_visible_kv_tile(ms[0], q0, S)
        assert bool(vis[0, 0, q0:q0 + 128, j * 128:(j + 1) * 128].any())
        vis[0, :, q0:q0 + 128, j * 128:(j + 1) * 128] = False
        return emulate(q, k, v, dout, ms, scale, vis_fwd=vis)
    if name == "backward q_hi one tile short":
        jt = 0                                               # batch row 0, kv tile 0: its last visible 64-row q tile dropped
        last = int(ms[0, min(jt * 128 + 127, S - 1)])
        qt = min((S + 63) // 64, (last + 63) // 64) - 1
        assert bool(vis[0, 0, qt * 64:qt * 64 + 64, jt * 128:jt * 128 + 128].any())
        vb = vis.clone()
        vb[0, :, qt * 64:qt * 64 + 64, jt * 128:jt * 128 + 128] = False
        return emulate(q, k, v, dout, ms, scale, vis_bwd=vb)
    if name == "one kv tile's dQ lost":
        drop = torch.zeros_like(vis)
        drop[1, :, 384:448, 128:256] = True                  # batch row 1, q tile 6 x kv tile 1
        return emulate(q, k, v, dout, ms, scale, dq_drop=drop)
    if name == "one q head's dK / dV lost":
        return emulate(q, k, v, dout, ms, scale, route=[0, None, 1, 1])
    if name == "one q head's dK / dV added to the next kv head":
        return emulate(q, k, v, dout, ms, scale, route=[0, 1, 1, 1])
    if name == "batch row reads another row's mask":
        wrong = ms.clone()
        wrong[1] = ms[0]
        return emulate(q, k, v, dout, wrong, scale)
    raise KeyError(name)


def check_all(out, q, k, v, dout, ms, scale, what, head_tol=HEAD_TOL):
    o, lse, dq, dk, dv = out
    ref = reference(q, k, v, dout, ms, scale, o, lse)
    return check_forward(o, lse, ref, what, head_tol=head_tol), check_backward(dq, dk, dv, ref, what, head_tol=head_tol)


def old_accepts(out, ref):
    """The older tests' whole-row and per-tile checks of O, dQ, dK and dV (their LSE check is 2e-3 absolute)."""
    o, lse, dq, dk, dv = out
    return (old_checks(o, ref["O"], 128) and old_checks(dq, ref["dQ"], 64) and old_checks(dk, ref["dK"], 128)
            and old_checks(dv, ref["dV"], 128))


def test_reference_matches_llama_ref_autograd():
    """The explicit fp64 backward formulas and the mask convention against oracle.llama_ref.attention (fp32, autograd)."""
    q, k, v, dout, ms, scale = cpu_batch()
    ref = reference(q, k, v, dout, ms, scale)
    for b in range(q.shape[0]):
        qf, kf, vf = (t[b:b + 1].float().requires_grad_(True) for t in (q, k, v))
        o = R.attention(qf, kf, vf, "fp32", mask_start=ms[b:b + 1])
        o.backward(dout[b:b + 1].float().reshape(1, CPU_S, -1))
        for name, got, want in (("O", o.detach().view(CPU_S, CPU_NH, CPU_D), ref["O"][b]), ("dQ", qf.grad[0], ref["dQ"][b]),
                                ("dK", kf.grad[0], ref["dK"][b]), ("dV", vf.grad[0], ref["dV"][b])):
            e = ((got.double() - want).norm() / want.norm()).item()
            assert e < 1e-5, (name, b, e)


def test_reference_lse_and_exact_visibility():
    q, k, v, dout, ms, scale = cpu_batch("zero_q")
    ref = reference(q, k, v, None, ms, scale)
    counts = visible(ms, 2, CPU_S, "cpu").sum(-1).double()
    assert torch.allclose(ref["LSE"], counts.log()[:, None].expand(-1, CPU_NH, -1), atol=1e-12)
    o, lse, *_ = emulate(q, k, v, dout, ms, scale)
    check_exact_visibility(o, lse, v, ms, "emulation, q = 0")
    bad = sabotage("row sees one column past its diagonal", q, k, v, dout, ms, scale)
    with pytest.raises(AssertionError, match="LSE of batch row 1 row 382"):
        check_exact_visibility(bad[0], bad[1], v, ms, "one column past the diagonal, q = 0")


@pytest.mark.parametrize("kind", ["randn", "planted"])
def test_checker_accepts_the_emulated_kernels(kind):
    q, k, v, dout, ms, scale = cpu_batch(kind)
    out = emulate(q, k, v, dout, ms, scale)
    fwd, bwd = check_all(out, q, k, v, dout, ms, scale, f"emulation {kind}",
                         head_tol=HEAD_TOL if kind == "randn" else HEAD_TOL_SHAPED)
    ref = reference(q, k, v, dout, ms, scale, out[0], out[1])
    if kind == "randn":          # with planted columns the old per-tile check rejects the correct dQ, whose rows cancel
        assert old_accepts(out, ref) and (out[1].to(F64) - ref["LSE"]).abs().max().item() < OLD_LSE
    assert fwd["o"]["c_need"] < C_FWD and max(r["c_need"] for r in bwd.values()) < C_BWD


SABOTAGES = [
    # name, whether the old whole-row / per-tile / LSE checks accept it on N(0, 1) inputs
    ("row sees one column past its diagonal", True),
    ("document's first row sees the previous document's last column", False),
    ("one kv tile too many skipped", False),
    ("backward q_hi one tile short", False),
    ("one kv tile's dQ lost", False),
    ("one q head's dK / dV lost", False),
    ("one q head's dK / dV added to the next kv head", False),
    ("batch row reads another row's mask", False),
]


@pytest.mark.parametrize("name,old_passes", SABOTAGES)
def test_checker_rejects_sabotage(name, old_passes):
    q, k, v, dout, ms, scale = cpu_batch()
    bad = sabotage(name, q, k, v, dout, ms, scale)
    ref = reference(q, k, v, dout, ms, scale, bad[0], bad[1])
    old = old_accepts(bad, ref)
    dl = (bad[1].to(F64) - ref["LSE"]).abs().max().item()
    print(f"[{name}] old whole-row / per-tile checks {'accept' if old else 'reject'} it; LSE moves by {dl:.1e}")
    assert old == old_passes
    with pytest.raises(AssertionError, match="exceeds"):
        check_all(bad, q, k, v, dout, ms, scale, name)


@pytest.mark.parametrize("name", [s[0] for s in SABOTAGES[:4]])
def test_checker_rejects_sabotage_on_planted_columns(name):
    """With +10 logits on the last column of every document and on the 64 / 128-row tile edges, the visibility bugs are
    rejected by the backward check alone, without the forward's LSE."""
    q, k, v, dout, ms, scale = cpu_batch("planted")
    bad = sabotage(name, q, k, v, dout, ms, scale)
    ref = reference(q, k, v, dout, ms, scale, bad[0], bad[1])
    with pytest.raises(AssertionError, match="exceeds"):
        check_backward(*bad[2:], ref, name, head_tol=HEAD_TOL_SHAPED)
    if name != "backward q_hi one tile short":
        with pytest.raises(AssertionError, match="exceeds"):
            check_forward(bad[0], bad[1], ref, name, head_tol=HEAD_TOL_SHAPED)


def test_checker_rejects_an_unwritten_row():
    q, k, v, dout, ms, scale = cpu_batch()
    o, lse, dq, dk, dv = emulate(q, k, v, dout, ms, scale)
    ref = reference(q, k, v, dout, ms, scale, o, lse)
    dk[1, 200, 1] = float("nan")
    with pytest.raises(AssertionError, match="non-finite"):
        check_backward(dq, dk, dv, ref, "nan row")


def test_pipeline_masks_have_the_layouts_the_gpu_cases_need():
    """The pipeline masks of the GPU cases: thousands of trailing one-token padding documents, an all-padding row, a
    document ending on a 128-row tile edge and one ending one row before it, runs of one-token documents, and a different
    layout in each row."""
    raw, ms = pipeline_mask(8192, 1, seed=3, greedy=True, pack_len=4096)
    assert int((ms[0] == torch.arange(1, 8193)).sum()) >= 4096
    raw, ms = pipeline_mask(2048, 4, seed=4, greedy=False, front=FRONT, empty_rows=(3,))
    assert torch.equal(ms[3], torch.arange(1, 2049, dtype=torch.int32))
    assert int(ms[0, 127]) == 128 and int(ms[0, 128]) == 255 and int(ms[0, 255]) == 256
    assert len({tuple(r.tolist()) for r in ms}) == 4
    ops().check_mask_form(raw)
    assert bool((ms[:, 1:] >= ms[:, :-1]).all())


# ----------------------------------------------------------------------------------------------------------
# The mask form, on every batch
# ----------------------------------------------------------------------------------------------------------
def test_check_mask_form():
    o = ops()
    o.check_mask_form(torch.tensor([[3, 3, 3, 0, 0], [5, 5, 5, 5, 5]], dtype=torch.int32))   # collator padding
    o.check_mask_form(torch.tensor([[1, 2, 3, 4, 5]]))                                        # one-token documents
    o.check_mask_form(torch.zeros(2, 1, 7, dtype=torch.int64))                                # all padding, [b, 1, s]
    with pytest.raises(ValueError, match="non-decreasing"):
        o.check_mask_form(torch.tensor([[3, 3, 3, 0, 0], [4, 4, 2, 4, 5]], dtype=torch.int32))
    with pytest.raises(ValueError, match="non-decreasing"):                                    # a later column, earlier end
        o.check_mask_form(torch.tensor([[5, 5, 3, 5, 5]]))


def test_packed_record_with_its_own_non_document_mask_is_rejected():
    """A record carrying its own attn_mask_startend_row_indices passes through packing and collation unchanged; a
    non-document layout in it is rejected by the check the Trainer and the engine run on every host batch."""
    from paddlenlp_b200.data import DataCollatorForSeq2Seq
    from paddlenlp_b200.datasets import ZeroPaddingMapDataset

    recs = [{"input_ids": [1] * 5, "labels": [1] * 5},
            {"input_ids": [1] * 4, "labels": [1] * 4, "attn_mask_startend_row_indices": [4, 2, 4, 4]}]
    batch = DataCollatorForSeq2Seq(max_length=16)([ZeroPaddingMapDataset(recs, max_length=16)[0]])
    with pytest.raises(ValueError, match="non-decreasing"):
        ops().check_mask_form(batch["attn_mask_startend_row_indices"])


# ----------------------------------------------------------------------------------------------------------
# GPU: the kernels against the reference
# ----------------------------------------------------------------------------------------------------------
PRESETS = {                    # nh, kvh, d
    "llama3_2_3b": (24, 8, 128),
    "llama3_8b": (32, 8, 128),
    "qwen2_1_5b": (12, 2, 128),
    "qwen2_7b": (28, 4, 128),
    "llama3_2_1b": (32, 8, 64),
    "qwen2_0_5b": (14, 2, 64),
}
# the in-order pack's first records: documents ending on the 128-row tile edge and one row before the next, one-token runs
FRONT = (128, 127, 1, 256, 1, 1, 1, 1, 1, 63, 65, 1, 1, 64)
PAD = 64


def set_impl(fwd, bwd):
    from paddlenlp_b200 import _lib

    lib = _lib.load()
    return lib.b200_set_fa_fwd_impl(fwd), lib.b200_set_fa_bwd_impl(bwd)


def run_kernels(q, k, v, dout, ms, scale):
    """Forward into a NaN-filled strided view (twice: must be bit-identical), backward twice into a NaN-filled packed dQKV
    buffer.  Returns (o, lse, [(dq, dk, dv), (dq, dk, dv)])."""
    o_ = ops()
    B, S, nh, d = q.shape
    kvh = k.shape[2]
    outs = []
    for _ in range(2):
        buf = torch.full((B, S, nh * d + 2 * PAD), float("nan"), dtype=BF16, device=DEV)
        out = buf[..., PAD:PAD + nh * d].unflatten(-1, (nh, d))
        _, lse = o_.flash_attn_fwd(q, k, v, scale, out=out, mask_start=ms)
        outs.append((buf, out, lse))
    torch.cuda.synchronize()
    (buf, o, lse), (buf2, o2, lse2) = outs
    for b in (buf, buf2):
        assert bool(torch.isnan(b[..., :PAD]).all() and torch.isnan(b[..., PAD + nh * d:]).all()), "write outside the output"
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "the forward is not deterministic"
    grads = []
    width = (nh + 2 * kvh) * d
    for _ in range(2):
        gbuf = torch.full((B, S, width + 2 * PAD), float("nan"), dtype=BF16, device=DEV)
        gv = gbuf[..., PAD:PAD + width]
        dq = gv[..., :nh * d].unflatten(-1, (nh, d))
        dk = gv[..., nh * d:(nh + kvh) * d].unflatten(-1, (kvh, d))
        dv = gv[..., (nh + kvh) * d:].unflatten(-1, (kvh, d))
        o_.flash_attn_bwd(q, k, v, o, dout, lse, dq, dk, dv, scale, mask_start=ms)
        torch.cuda.synchronize()
        assert bool(torch.isnan(gbuf[..., :PAD]).all() and torch.isnan(gbuf[..., PAD + width:]).all()), "write outside dQKV"
        grads.append((dq, dk, dv))
    return o, lse, grads


def make_inputs(B, S, nh, kvh, d, seed, kind, ms, scale):
    """q / k / v views of a packed projection [B, S, (nh + 2 kvh) d] (inside a wider buffer), dout [B, S, nh, d]."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    width = (nh + 2 * kvh) * d
    qkv = torch.randn(B, S, width + 3 * d, generator=g, device=DEV).to(BF16)[..., :width]
    q = qkv[..., :nh * d].unflatten(-1, (nh, d))
    k = qkv[..., nh * d:(nh + kvh) * d].unflatten(-1, (kvh, d))
    v = qkv[..., (nh + kvh) * d:].unflatten(-1, (kvh, d))
    dout = torch.randn(B, S, nh, d, generator=g, device=DEV).to(BF16)
    shape_scores(q, k, kind, ms, scale)
    return q, k, v, dout


def run_case(what, preset, B, S, ms, seed, kind="randn", scale=None, impl=2):
    """Forward and backward of kernel `impl` on one case, checked per element, per (row, head) and per LSE."""
    nh, kvh, d = PRESETS[preset]
    sc = 1.0 / math.sqrt(d) if scale is None else scale
    ms = None if ms is None else ms.to(DEV).contiguous()
    q, k, v, dout = make_inputs(B, S, nh, kvh, d, seed, kind, ms, sc)
    old = set_impl(impl, impl)
    try:
        o, lse, grads = run_kernels(q, k, v, dout, ms, sc)
    finally:
        set_impl(*old)
    what = f"{what} {preset} {nh}/{kvh} d{d} B{B} S{S} {kind} impl {impl}"
    print(f"\n[{what}]")
    if kind == "zero_q":
        check_exact_visibility(o, lse, v, ms, what)
    ref = reference(q, k, v, dout, ms, sc, o, lse)
    tol = HEAD_TOL if kind in ("randn", "zero_q") else HEAD_TOL_SHAPED
    fwd = check_forward(o, lse, ref, what, head_tol=tol)
    bwd = [check_backward(*gr, ref, what + f" run {i}", head_tol=tol) for i, gr in enumerate(grads)]
    same = all(torch.equal(a, b) for a, b in zip(*grads))
    print(f"  [{what}] backward runs bit-identical: {same}")
    del ref
    return fwd, bwd


def bench_mask(kind, S, B, seed):
    if kind == "causal":
        return None
    if B == 1:
        return pipeline_mask(S, B, seed, greedy=True)[1]
    return pipeline_mask(S, B, seed, greedy=False, front=FRONT, empty_rows=(B - 1,))[1]


@pytest.mark.gpu
@pytest.mark.parametrize("mask", ["docs", "causal"])
@pytest.mark.parametrize("B,S", [(1, 4096), (4, 2048)])
@pytest.mark.parametrize("preset", list(PRESETS))
def test_preset_at_benchmark_shapes(preset, B, S, mask):
    """Every preset's head layout at the pre-training benchmark's 1 x 4096 and the SFT benchmark's 4 x 2048, plain causal
    and with pipeline masks: greedy packing at 1 x 4096; in-order packing at 4 x 2048 with documents ending on and one row
    before the 128-row tile edges, one-token runs, right padding and a row that is all padding."""
    run_case(f"bench {mask}", preset, B, S, bench_mask(mask, S, B, seed=S + B), seed=list(PRESETS).index(preset) * 100 + B * 10 + (mask == "docs"))


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B,S,mask", [
    ("llama3_8b", 1, 8192, "padded"),       # 4 096 packed rows, then 4 096 one-token padding documents
    ("llama3_8b", 1, 8192, "causal"),
    ("qwen2_7b", 1, 16384, "docs"),         # Qwen2 presets allow 32k positions
    ("qwen2_1_5b", 3, 1000, "docs"),        # S not a multiple of 64 or 128
    ("qwen2_0_5b", 1, 4095, "docs"),
    ("llama3_2_3b", 2, 2047, "causal"),
    ("llama3_2_1b", 2, 1000, "causal"),
])
def test_long_and_unaligned_sequences(preset, B, S, mask):
    if mask == "padded":
        ms = pipeline_mask(S, B, seed=7, greedy=True, pack_len=4096)[1]
    elif mask == "docs":
        ms = pipeline_mask(S, B, seed=S, greedy=S > 2048, hi=min(1500, S))[1]
    else:
        ms = None
    run_case(f"long/unaligned {mask}", preset, B, S, ms, seed=S + B)


def every_offset_mask(S=300):
    """128 batch rows; row b's first document has length b + 1, so the boundaries cover every offset of the 128-row tile."""
    return torch.stack([doc_mask([b + 1, S - b - 1]) for b in range(128)])


@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["qwen2_1_5b", "qwen2_0_5b"])
def test_document_boundary_at_every_tile_offset(preset):
    run_case("boundary at every offset", preset, 128, 300, every_offset_mask(), seed=128)


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B,S,kind,mask,scale", [
    ("llama3_2_3b", 1, 4096, "planted", "docs", None),
    ("qwen2_0_5b", 4, 2048, "planted", "docs", None),
    ("llama3_8b", 4, 2048, "planted", "causal", None),
    ("llama3_8b", 4, 2048, "sink", "docs", None),
    ("qwen2_1_5b", 1, 4096, "rising", "docs", None),
    ("llama3_2_1b", 1, 4096, "rising", "causal", None),
    ("qwen2_7b", 4, 2048, "randn", "docs", 0.05),
])
def test_score_ranges(preset, B, S, kind, mask, scale):
    """Planted +10 logits on every document's last column and the tile edges (a row that wrongly sees one is dominated by
    it), attention sinks on every document's first column, logits that rise along the sequence (the running maximum and the
    rescale change on every kv tile), and a softmax scale other than 1 / sqrt(d)."""
    run_case(f"scores {mask}", preset, B, S, bench_mask(mask, S, B, seed=S + B + 1), seed=S * 3 + B, kind=kind, scale=scale)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["greedy", "in_order", "padded", "every_offset", "causal"])
@pytest.mark.parametrize("preset", ["llama3_2_3b", "qwen2_0_5b"])
def test_exact_visibility(preset, layout):
    """q = 0 pins the visible set of every row, head and batch row exactly: LSE = ln(count), O = mean of the visible V."""
    B, S = {"greedy": (1, 4096), "in_order": (4, 2048), "padded": (1, 8192), "every_offset": (128, 300),
            "causal": (2, 1000)}[layout]
    ms = {"greedy": lambda: pipeline_mask(S, B, seed=21, greedy=True)[1],
          "in_order": lambda: pipeline_mask(S, B, seed=22, greedy=False, front=FRONT, empty_rows=(B - 1,))[1],
          "padded": lambda: pipeline_mask(S, B, seed=23, greedy=True, pack_len=4096)[1],
          "every_offset": every_offset_mask, "causal": lambda: None}[layout]()
    run_case(f"exact {layout}", preset, B, S, ms, seed=B * S, kind="zero_q")


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B,S", [("llama3_2_3b", 1, 4096), ("qwen2_1_5b", 4, 2048)])
def test_mma_sync_kernels_at_benchmark_shapes(preset, B, S):
    """The mma.sync kernels (impl 1; the forward is the paged prefill kernel of append_attention) through the same checker."""
    run_case("mma.sync docs", preset, B, S, bench_mask("docs", S, B, seed=S + B), seed=S + B + 5, impl=1)


@pytest.mark.gpu
def test_fusion_flash_attention_end_to_end():
    """fusion_flash_attention and torch autograd at the SFT benchmark shape, from the collator's raw start rows (padding 0,
    canonicalised inside) and q / k / v views of a packed projection (made contiguous inside)."""
    from paddlenlp_b200.transformers.llama.fusion_ops import fusion_flash_attention

    preset, B, S = "llama3_2_3b", 4, 2048
    nh, kvh, d = PRESETS[preset]
    raw, ms = pipeline_mask(S, B, seed=31, greedy=False, front=FRONT, empty_rows=(1,))
    sc = 1.0 / math.sqrt(d)
    q, k, v, dout = make_inputs(B, S, nh, kvh, d, 31, "randn", None, sc)
    qkv = q._base if q._base is not None else q
    leaf = qkv.detach()[..., :(nh + 2 * kvh) * d].clone().requires_grad_(True)
    ql = leaf[..., :nh * d].unflatten(-1, (nh, d))
    kl = leaf[..., nh * d:(nh + kvh) * d].unflatten(-1, (kvh, d))
    vl = leaf[..., (nh + kvh) * d:].unflatten(-1, (kvh, d))
    out = fusion_flash_attention(ql, None, kl, vl, None, False, attn_mask_startend_row_indices=raw)
    out.backward(dout.reshape(B, S, nh * d))
    g = leaf.grad
    dq = g[..., :nh * d].unflatten(-1, (nh, d))
    dk = g[..., nh * d:(nh + kvh) * d].unflatten(-1, (kvh, d))
    dv = g[..., (nh + kvh) * d:].unflatten(-1, (kvh, d))
    o, lse = ops().flash_attn_fwd(q.contiguous(), k.contiguous(), v.contiguous(), sc, mask_start=ms.to(DEV))
    assert torch.equal(out.detach().view(B, S, nh, d), o)
    what = "fusion_flash_attention + autograd"
    print(f"\n[{what}]")
    ref = reference(q, k, v, dout, ms.to(DEV), sc, o, lse)
    check_forward(out.detach().view(B, S, nh, d), lse, ref, what)
    check_backward(dq, dk, dv, ref, what)


# ----------------------------------------------------------------------------------------------------------
# GPU: the mask form is checked on every host batch
# ----------------------------------------------------------------------------------------------------------
def _tiny_model():
    import paddlenlp_b200.transformers as T

    return T.LlamaForCausalLM(T.LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                                            num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=256,
                                            seq_length=128, rope_theta=500000.0, rms_norm_eps=1e-5))


def _batch(ms_row, g):
    S = len(ms_row)
    ids = torch.randint(1, 512, (2, S), generator=g)
    return {"input_ids": ids, "labels": ids.clone(),
            "attn_mask_startend_row_indices": torch.stack([doc_mask([S // 2, S - S // 2]), torch.tensor(ms_row, dtype=torch.int32)])}


@pytest.mark.gpu
def test_model_rejects_a_decreasing_start_row_on_a_later_batch():
    model = _tiny_model()
    g = torch.Generator().manual_seed(0)
    good = _batch(doc_mask([30, 98]).tolist(), g)
    model(**good)                                                    # first batch: the engine's one-time check passes
    bad_row = doc_mask([30, 98]).tolist()
    bad_row[40] = 35                                                 # column 40 ends before column 39's document
    with pytest.raises(ValueError, match="non-decreasing"):
        model(**_batch(bad_row, g))
    # a valid host mask on a later batch is checked on the host: preparing it adds no device synchronisation
    ms = good["attn_mask_startend_row_indices"].pin_memory()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        model.engine._prep_mask(ms, 2, 128)
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["batch", "record"])
def test_trainer_rejects_a_non_document_mask_on_the_second_batch(source, tmp_path):
    """The Trainer's second batch carries a decreasing start row: from the dataset directly, or from a record with its own
    attn_mask_startend_row_indices that went through ZeroPaddingMapDataset and DataCollatorForSeq2Seq."""
    from paddlenlp_b200.data import DataCollatorForSeq2Seq
    from paddlenlp_b200.datasets import ZeroPaddingMapDataset
    from paddlenlp_b200.trainer import Trainer, TrainingArguments

    S = 128
    recs = [{"input_ids": list(range(1, 61)), "labels": list(range(2, 62))},
            {"input_ids": list(range(1, 51)), "labels": list(range(2, 52))},
            {"input_ids": list(range(1, 101)), "labels": list(range(2, 102))}]
    bad = {"input_ids": list(range(1, 9)), "labels": list(range(2, 10))}
    if source == "record":
        bad["attn_mask_startend_row_indices"] = [8, 8, 3, 8, 8, 8, 8, 8]
    recs.append(bad)
    data = list(ZeroPaddingMapDataset(recs, max_length=S))
    assert len(data) == 2
    if source == "batch":
        data[1] = dict(data[1])
        rows = list(data[1]["attn_mask_startend_row_indices"])
        rows[105] = 104
        data[1]["attn_mask_startend_row_indices"] = rows

    class InOrder(torch.utils.data.IterableDataset):
        served = 0

        def __iter__(self):
            for rec in data:
                InOrder.served += 1
                yield rec

    args = TrainingArguments(output_dir=str(tmp_path), per_device_train_batch_size=1, max_steps=2, learning_rate=1e-3,
                             max_seq_length=S, logging_steps=1)
    trainer = Trainer(model=_tiny_model(), args=args, train_dataset=InOrder(),
                      data_collator=DataCollatorForSeq2Seq(max_length=S))
    with pytest.raises(ValueError, match="non-decreasing"):
        trainer.train()
    assert InOrder.served == 2                                          # the first batch trained, the second was refused
