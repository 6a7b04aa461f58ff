"""Build and run tests/count_lower.c (TEST INFRASTRUCTURE): the reference's md_script.c + the shim in one unit, compiled as
tests/test_range_selections.py compiles tests/range_lower.c. Needs the reference sources and oracle/_ref (make -C oracle ref)."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/ext/mdlib"   # REF of oracle/Makefile


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "src")) and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "obj_strict"))


def build(out_dir) -> str:
    objs = os.path.join(ROOT, "oracle", "_ref", "obj_strict")
    inc = [f"-I{REF}/{d}" for d in ("src", "ext/simde", "ext/xxhash", "ext/svd3", "ext/fastlz", "ext/xtc", "ext/stb", "ext/libdivide", "ext/hy36")]
    defs = ["-D__FMA__", "-D__LITTLE_ENDIAN__", "-D__FORCE_ASSERTIONS__=0", "-DMD_GL_SPLINE_SUBDIVISION_COUNT=8", "-D_GNU_SOURCE", "-DNDEBUG"]
    exe = os.path.join(str(out_dir), "count_lower")
    o = sorted(os.path.join(objs, f) for f in os.listdir(objs) if f.endswith(".o") and f != "md_script.o")
    subprocess.check_call(["gcc", "-std=gnu2x", "-w", "-mavx2", "-mfma", *defs, *inc, "-O2", "-fno-fast-math", "-ffp-contract=off", "-fno-strict-aliasing",
                           f"-I{ROOT}/include", os.path.join(ROOT, "tests", "count_lower.c"), *o, "-o", exe, f"-L{ROOT}/viamd_b200", "-lmdgpu",
                           f"-Wl,-rpath,{ROOT}/viamd_b200", "-lm", "-lpthread"])
    return exe


def lower(exe, sys_path, script):
    """(return code, [one dict per lowered property], stderr)"""
    p = subprocess.run([exe, "lower", "--sys", sys_path, "--script", script], capture_output=True, text=True)
    return p.returncode, [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")], p.stdout + p.stderr


def groups(exe, sys_path) -> dict:
    """the system's component offsets, instance atom ranges and structure CSR as the reference loads them"""
    return json.loads(subprocess.check_output([exe, "groups", "--sys", sys_path]).decode())
