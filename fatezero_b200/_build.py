"""Build libfatezero_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libfatezero_b200.so")
SOURCES = ["fz_capi.cu", "fz_gemm.cu", "fz_elem.cu", "fz_attn.cu", "fz_p2p.cu", "fz_clip.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "--use_fast_math" if False else "-DFZ_NO_FAST_MATH"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "fatezero_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = True, variant: str = "", extra_flags=()) -> str:
    """variant/extra_flags: development builds (libfatezero_b200_<variant>.so with extra -D flags) for A/B measurements."""
    if variant:
        return _build(os.path.join(HERE, f"libfatezero_b200_{variant}.so"), os.path.join(HERE, "build", variant), list(extra_flags), verbose)
    if not force and not needs_build():
        return LIB
    return _build(LIB, os.path.join(HERE, "build"), [], verbose)


def _build(lib: str, objdir: str, extra_flags, verbose: bool) -> str:
    objs = []
    procs = []
    os.makedirs(objdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, *extra_flags, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out.decode()}")
    cmd = [_nvcc(), "-shared", "-o", lib, *objs, *ARCH]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return lib


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--variant", default="")
    ap.add_argument("--flags", default="")
    a = ap.parse_args()
    print(build(force=a.force, variant=a.variant, extra_flags=a.flags.split()))
