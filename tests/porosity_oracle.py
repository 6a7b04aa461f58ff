"""ctypes binding of the plain-C restatement of porosity() (oracle/md_porosity.c). TEST INFRASTRUCTURE ONLY.

Builds oracle/build/libporosity.so on first use (gcc, the strict IEEE flags of liboracle.so)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

SRC = os.path.join(O.ORACLE_DIR, "md_porosity.c")
LIB = os.path.join(O.ORACLE_DIR, "build", "libporosity.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        deps = [SRC, os.path.join(O.ORACLE_DIR, "md_oracle.c"), os.path.join(O.ORACLE_DIR, "md_oracle.h")]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            subprocess.check_call(["gcc", "-std=gnu11", "-O2", "-fno-fast-math", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-w", "-o", LIB, SRC, "-lm"])
        _lib = C.CDLL(LIB)
    return _lib


def porosity(x, y, z, radius, idx, cell):
    """one frame -> dict(value, com, bmin, bmax, dim, set, n, tests, grid): n = the grid's voxel count N, tests = sphere-voxel tests the
    reference's loop executes; grid False for a triclinic cell or an empty selection (value 0)"""
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    x, y, z, radius = f32(x), f32(y), f32(z), f32(radius); idx = np.ascontiguousarray(idx, np.int32)
    v = C.c_float(); com, bmin, bmax = (np.zeros(3, np.float32) for _ in range(3)); dim = np.zeros(3, np.int32); s = C.c_uint64(); t = C.c_uint64()
    p = lambda a, ty: a.ctypes.data_as(C.POINTER(ty))
    rc = lib().mdo_porosity(p(x, C.c_float), p(y, C.c_float), p(z, C.c_float), p(radius, C.c_float), p(idx, C.c_int32), C.c_size_t(len(idx)), C.byref(cell),
                            C.byref(v), p(com, C.c_float), p(bmin, C.c_float), p(bmax, C.c_float), p(dim, C.c_int32), C.byref(s), C.byref(t))
    return dict(value=np.float32(v.value), com=com, bmin=bmin, bmax=bmax, dim=dim, set=int(s.value), n=int(np.prod(dim.astype(np.int64))) if rc == 0 else 0,
                tests=int(t.value), grid=rc == 0)


def set_from_value(value, n):
    """the occupied-voxel count the float value pins when n <= 2^23: the one count c with (float)((n - c) / n) == value"""
    assert n <= 1 << 23
    c = int(round(n - float(value) * n))
    hits = [k for k in range(max(c - 2, 1), min(c + 3, n + 1)) if np.float32((n - k) / n) == np.float32(value)]
    assert len(hits) == 1, (value, n, hits)
    return hits[0]
