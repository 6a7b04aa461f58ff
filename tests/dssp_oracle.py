"""ctypes binding of the plain-C restatement of the secondary-structure inference (oracle/md_dssp.c). TEST INFRASTRUCTURE ONLY.

Builds oracle/build/libdssp.so on first use (gcc, the strict IEEE flags of liboracle.so)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as O

SRC = os.path.join(O.ORACLE_DIR, "md_dssp.c")
LIB = os.path.join(O.ORACLE_DIR, "build", "libdssp.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        deps = [SRC, os.path.join(O.ORACLE_DIR, "md_oracle.c"), os.path.join(O.ORACLE_DIR, "md_oracle.h")]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            subprocess.check_call(["gcc", "-std=gnu11", "-O2", "-fno-fast-math", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-w", "-o", LIB, SRC, "-lm"])
        _lib = C.CDLL(LIB)
        _lib.mdo_dssp.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint64]
    return _lib


def dssp(x, y, z, cell, atoms, range_off, shuffle_seed=0):
    """one frame -> (status, int32 [S] md_secondary_structure_t); status 0, -1 malformed input, -3 unsupported cell"""
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    x, y, z = f32(x), f32(y), f32(z)
    atoms = np.ascontiguousarray(atoms, np.int32).reshape(-1, 5); ro = np.ascontiguousarray(range_off, np.uint32)
    out = np.zeros(len(atoms), np.int32)
    rc = lib().mdo_dssp(out.ctypes.data, x.ctypes.data, y.ctypes.data, z.ctypes.data, C.addressof(cell), atoms.ctypes.data, len(atoms),
                        ro.ctypes.data, len(ro) - 1, shuffle_seed)
    return rc, out
