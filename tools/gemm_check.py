"""Bring-up / regression check of the wgmma GEMM on an H100.

    python tools/gemm_check.py            # driver: one subprocess per (a_major, b_major) case
    python tools/gemm_check.py --case 0,1

Each case checks correctness against torch.matmul (fp32 accumulate reference on the same bf16 inputs) on
single-tile, ragged and multi-tile shapes, then times a large shape.  Output is appended to <--log-dir>/gemm_check.log.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_case(a_mn, b_mn, big):
    import torch

    from paddlenlp_b200 import _lib

    _lib.call("b200_device_check")
    dev = torch.device("cuda:0")
    res = []

    def gemm(A, B, C, M, N, K, acc=0, bias=None):
        _lib.call("b200_gemm_bf16_ex", _lib.ptr(A), _lib.ptr(B), _lib.ptr(C), _lib.ptr(bias), None, M, N, K,
                  A.stride(0), B.stride(0), C.stride(0), 0, a_mn, b_mn, acc, 0, _lib.stream_ptr())

    def check(M, N, K, acc=0, use_bias=False, seed=0):
        g = torch.Generator(device="cpu").manual_seed(seed)
        Al = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
        Bl = (torch.randn(K, N, generator=g) * 0.5).to(torch.bfloat16)
        C0 = (torch.randn(M, N, generator=g)).to(torch.bfloat16)
        bias = torch.randn(N, generator=g).float() if use_bias else None
        A = (Al.t().contiguous() if a_mn else Al).to(dev)       # a_mn: stored [K, M]
        B = (Bl if b_mn else Bl.t().contiguous()).to(dev)        # b_mn: stored [K, N]; else [N, K]
        C = C0.clone().to(dev)
        bias_d = bias.to(dev) if use_bias else None
        gemm(A, B, C, M, N, K, acc, bias_d)
        torch.cuda.synchronize()
        ref = Al.float().to(dev) @ Bl.float().to(dev)
        if use_bias:
            ref = ref + bias_d
        if acc:
            ref = ref + C0.float().to(dev)
        got = C.float()
        err = (got - ref).abs()
        scale = ref.abs().max().item() + 1e-9
        maxerr = err.max().item()
        # bf16 rounding of the result: half-ulp relative 2^-9
        tol = scale * 2.0 ** -8 + 1e-3
        ok = bool(maxerr <= tol) and bool(torch.isfinite(got).all())
        info = dict(case=[a_mn, b_mn], M=M, N=N, K=K, acc=acc, bias=use_bias, maxerr=maxerr, scale=scale, ok=ok)
        if not ok:
            bad = err > tol
            rows = bad.any(dim=1).nonzero().flatten()
            cols = bad.any(dim=0).nonzero().flatten()
            info["bad_frac"] = bad.float().mean().item()
            info["bad_rows"] = [int(rows.min()), int(rows.max()), int(rows.numel())] if rows.numel() else []
            info["bad_cols"] = [int(cols.min()), int(cols.max()), int(cols.numel())] if cols.numel() else []
            info["sample_got"] = got[:2, :4].tolist()
            info["sample_ref"] = ref[:2, :4].tolist()
        res.append(info)
        print(json.dumps(info), flush=True)
        return ok

    shapes = [
        (128, 256, 64), (128, 256, 128), (128, 256, 512),
        (256, 512, 256), (512, 768, 320), (384, 256, 64),
        (1024, 1024, 1024), (136, 264, 72), (2048, 6144, 4096),
    ]
    allok = True
    for (M, N, K) in shapes:
        allok &= check(M, N, K)
    allok &= check(512, 512, 256, acc=1, seed=3)
    allok &= check(512, 512, 256, use_bias=True, seed=4)
    allok &= check(1000, 520, 136, acc=1, use_bias=True, seed=5)

    if big and allok:
        for (M, N, K) in [(4096, 4096, 4096), (8192, 8192, 8192), (4096, 28672, 4096), (4096, 4096, 14336)]:
            A = torch.randn((K, M) if a_mn else (M, K), device=dev).to(torch.bfloat16)
            B = torch.randn((K, N) if b_mn else (N, K), device=dev).to(torch.bfloat16)
            C = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for _ in range(3):
                gemm(A, B, C, M, N, K)
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            iters = 10
            e0.record()
            for _ in range(iters):
                gemm(A, B, C, M, N, K)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            tf = 2.0 * M * N * K / ms / 1e9
            # cuBLAS reference for the same op
            At = A.t() if a_mn else A
            Bt = B if b_mn else B.t()
            for _ in range(3):
                torch.matmul(At, Bt, out=C)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(iters):
                torch.matmul(At, Bt, out=C)
            e1.record()
            torch.cuda.synchronize()
            ms2 = e0.elapsed_time(e1) / iters
            tf2 = 2.0 * M * N * K / ms2 / 1e9
            info = dict(case=[a_mn, b_mn], perf=[M, N, K], ms=ms, tflops=tf, cublas_ms=ms2, cublas_tflops=tf2)
            print(json.dumps(info), flush=True)
    return allok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    ap.add_argument("--no-big", action="store_true")
    ap.add_argument("--cases", default=None, help="semicolon separated list of a,b")
    ap.add_argument("--log-dir", default=".", help="directory of gemm_check.log")
    a = ap.parse_args()
    if a.case:
        am, bm = [int(x) for x in a.case.split(",")]
        ok = run_case(am, bm, not a.no_big)
        sys.exit(0 if ok else 1)
    os.makedirs(a.log_dir, exist_ok=True)
    log = open(os.path.join(a.log_dir, "gemm_check.log"), "a")
    if a.cases:
        cases = [tuple(int(x) for x in c.split(",")) for c in a.cases.split(";")]
    else:
        cases = [(am, bm) for am in (0, 1) for bm in (0, 1)]
    summary = {}
    for (am, bm) in cases:
        cmd = [sys.executable, os.path.abspath(__file__), "--case", f"{am},{bm}"] + (["--no-big"] if a.no_big else [])
        t0 = time.time()
        try:
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=240)
            out, rc = r.stdout + r.stderr[-3000:], r.returncode
        except subprocess.TimeoutExpired as e:
            out, rc = (e.stdout or b"").decode(errors="replace") + "\nTIMEOUT", -9
        hdr = f"=== case a_mn={am} b_mn={bm} rc={rc} ({time.time() - t0:.1f}s)"
        print(hdr)
        print(out[-6000:])
        log.write(hdr + "\n" + out + "\n")
        log.flush()
        summary[f"{am},{bm}"] = rc
    print("SUMMARY", json.dumps(summary))
    log.write("SUMMARY " + json.dumps(summary) + "\n")


if __name__ == "__main__":
    main()
