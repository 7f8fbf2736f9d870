"""Builds libsplashsurf_b200.so (sm_90a, H100) in-tree with nvcc.  No torch involved: the library is plain CUDA + cub."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsplashsurf_b200.so")
SOURCES = ["ss_pipeline.cu"]


def deps():
    """Every file of csrc/ plus the public header: editing any of them makes the library stale."""
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(HERE, "..", "include", "splashsurf_b200.h")]


NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    # parity: no implicit FMA contraction, IEEE division / square root, denormals kept
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fno-fast-math", "--shared", "-Xptxas", "-v",
    "--extended-lambda",
]


def source_hash(only=None) -> str:
    """sha256 (first 16 hex digits) over the CUDA sources and the public header: identifies the code a profile was taken on.
    `only`: restrict to these file names of csrc/ (e.g. the files that define one stage's kernels)."""
    import hashlib
    h = hashlib.sha256()
    for d in deps():
        if only is not None and os.path.basename(d) not in only:
            continue
        if d.endswith((".cu", ".cuh", ".inc", ".h")):
            h.update(open(d, "rb").read())
    return h.hexdigest()[:16]


# the files that define the level-set kernels (certification, exact pass, shared device helpers): a DRAM-traffic capture of the
# level-set stage stays valid while these are unchanged
LEVELSET_SOURCES = ("ss_brick.cuh", "ss_certify.cuh", "ss_exact.cuh", "ss_kernels.cuh", "ss_sm90.cuh", "ss_common.cuh")


def levelset_source_hash() -> str:
    return source_hash(only=LEVELSET_SOURCES)


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in deps()) or os.path.getmtime(__file__) > t


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES] + ["-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = os.path.join(HERE, "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed (see {log})")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
