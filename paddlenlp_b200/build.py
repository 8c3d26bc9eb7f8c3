"""Build libb200nlp.so (the C-ABI library of hand-written sm_90a kernels) in-tree with nvcc.

    python -m paddlenlp_b200.build            # incremental (per-file objects, timestamp based)
    python -m paddlenlp_b200.build --force

nvcc cross-compiles for sm_90a (H100) without a GPU.  The .so lands in paddlenlp_b200/lib/ (git-ignored: every checkout
builds its own).
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
LIBDIR = os.path.join(ROOT, "lib")
OBJDIR = os.path.join(ROOT, "build")
LIB = os.path.join(LIBDIR, "libb200nlp.so")
INCLUDE = os.path.join(os.path.dirname(ROOT), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
    "-I", INCLUDE,
]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime() -> float:
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return max(os.path.getmtime(h) for h in hdrs)


def _compile(src: str, obj: str, verbose: bool) -> str:
    cmd = [nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    with open(obj + ".log", "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{log}")
    if verbose:
        print(log)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_t = _deps_mtime()
    jobs = []
    objs = []
    for src in _sources():
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        stale = force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_t)
        if stale:
            jobs.append((src, obj))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = [ex.submit(_compile, s, o, verbose) for s, o in jobs]
            for f in futs:
                f.result()
    need_link = bool(jobs) or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs)
    if need_link:
        cmd = [nvcc(), "-shared", NVCC_FLAGS[0], NVCC_FLAGS[1], "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("-v", "--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
