"""Build libmdgpu.so (hand-written CUDA for sm_90a + C ABI) in-tree with nvcc. No GPU needed to compile."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmdgpu.so")
STAMP = os.path.join(HERE, "build", "flags.txt")   # the flags libmdgpu.so was built with
SOURCES = ["cells.cu", "rdf.cu", "sdf.cu", "props.cu", "within.cu", "synth.cu", "xtc.cu", "rama.cu", "porosity.cu", "expr.cu", "dssp.cu", "plan.cu"]
ARCH = "arch=compute_90a,code=sm_90a"   # H100 (Hopper)
NVCC_FLAGS = [
    "-gencode", ARCH, "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",            # no implicit FMA contraction: float results must match the reference's scalar/AVX code
    "-Xcompiler", "-fPIC,-O2,-fno-fast-math,-ffp-contract=off",
    "-Xptxas", "-v",
]


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _flags_stamp() -> str:
    return " ".join([ARCH, *NVCC_FLAGS, *SOURCES])


def needs_build() -> bool:
    """True when the library is missing, older than a source, or was built with other flags (another architecture, say)."""
    if not os.path.exists(LIB):
        return True
    try:
        with open(STAMP) as f:
            if f.read() != _flags_stamp():
                return True
    except OSError:
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "mdgpu.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    log = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    cmd = [nvcc(), "-shared", "-o", LIB, *objs, "-gencode", ARCH]
    subprocess.check_call(cmd)
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    with open(STAMP, "w") as f:
        f.write(_flags_stamp())
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
