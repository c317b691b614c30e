"""Builds libiblb200.so in-tree with nvcc for sm_90a (H100); the library is loaded from openibl_b200/lib."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libiblb200.so")
SOURCES = ["engine.cu", "simt_conv.cu", "netvlad.cu", "gemm_simt.cu", "topk.cu", "tc_conv.cu", "tc_gemm.cu", "tc_netvlad.cu", "tc_conv1.cu", "tc_probe.cu", "netvlad_bwd.cu", "tc_dist1.cu", "tc_conv_bwd.cu", "resize.cu", "sort_rows.cu", "rerank.cu", "jpeg.cu", "png.cu", "color_jitter.cu", "tc_pca_bwd.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libiblb200 cannot be built (there is no CPU fallback)")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "iblb200.h"))
    objs = []
    procs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [sp, os.path.abspath(__file__)] + headers):   # new flags rebuild too
            cmd = [nvcc(), *NVCC_FLAGS, "-c", sp, "-o", obj]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed on {src} ---\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"--- {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if force or procs or _stale(LIB, objs):
        # link next to the target and rename: the library is replaced atomically (a copy of the tree or a running
        # process never sees a half-written .so)
        tmp = LIB + ".tmp"
        cmd = [nvcc(), "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
        subprocess.check_call(cmd)
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
