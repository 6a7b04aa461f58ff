"""Generate tests/golden/props_edges.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict `eval` on raw trajectories, as
make_golden_sdf_edges.py does): the per-frame values of distance / angle / dihedral / com and density_x/_y/_z on geometries of
tests/test_props_edges.py, built by that file's case builders:
  far_images    dihedrals whose bond vectors span 65 and 200 box lengths along each axis, one orthorhombic and one triclinic frame
  nonperiodic   one non-periodic axis per frame, then a periodic frame; atoms outside the box
  shear_npt     distance() of atoms and of selections in triclinic cells whose shear (up to L/2) and box change every frame
  masses        centres of mass of atoms the reference gives mass 0 (atom name X), 16 and 7 of them, and of a mixed selection, with no cell,
                an orthorhombic and a triclinic cell
  simd_split    com(atom(1:n)) and distance(atom(1:n), 400) for n = 1, 7, 8, 9, 15, 16, 17, 67, with the same three cells
  collinear     angles whose normalised dot product rounds past +-1, and dihedrals of four collinear atoms
  density_tric  density_x/_y/_z of every atom on bin edges, one ulp either side and at rc +- ext/2 of a triclinic initial cell
The system file is a .gro of one-atom residues named C (or X for the zero-mass atoms); the reference's masses are stored with the frames, and
the raw trajectory supplies every coordinate and cell. Selections are atom ranges (atom(a:b)), as the script addresses them.

Left out, because the reference never returns on them: a dihedral bond vector with an infinite component, or one so large that a minimum-image
step leaves it unchanged (dx - box == dx, from about 2^24 box lengths on); the library returns NaN there (include/mdgpu.h).

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_props_edges.py
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import refio  # noqa: E402
from make_golden import HARNESS, run  # noqa: E402
import test_props_edges as T  # noqa: E402


def rng_(a, b):
    return [int(a), int(b)]


def cases():
    """name -> (frames, cells, atoms named X, [(statement, kind, args)]); args: 0-based atoms or [lo, hi) ranges, density (axis, range)"""
    out = {}
    fr, cells, meta = T.far_geometry()
    out["far_images"] = (fr, cells, (), [(f"t{k}_{ax}", "dihedral", [int(i) for i in at]) for k, ax, _, at in meta if k in (65, 200)])
    c = T.case_nonperiodic()
    out["nonperiodic"] = (c.frames, c.cells, (), [("d", "distance", [100, 101]), ("d_sel", "distance", [rng_(0, 20), rng_(20, 52)]),
                                                   ("a", "angle", [104, 105, 106]), ("t", "dihedral", [108, 109, 110, 111]), ("c", "com", [rng_(20, 52)])])
    c = T.case_shear_npt()
    out["shear_npt"] = (c.frames, c.cells, (), [("d", "distance", [0, 90]), ("d_sel", "distance", [rng_(0, 16), rng_(40, 64)]), ("t", "dihedral", [0, 1, 2, 3])])
    c = T.case_masses()
    zero = list(range(0, 23)) + list(range(30, 56, 2))
    out["masses"] = (c.frames, c.cells, zero, [("c_zero", "com", [rng_(0, 16)]), ("c_zero7", "com", [rng_(16, 23)]), ("c_mixed", "com", [rng_(30, 56)]),
                                               ("d_zero", "distance", [rng_(0, 16), 200]), ("t_zero", "dihedral", [rng_(16, 23), 202, 203, rng_(0, 16)])])
    c = T.case_simd_split()
    out["simd_split"] = (c.frames, c.cells, (), [(f"c{n}", "com", [rng_(0, n)]) for n in T.SIMD_SIZES] + [(f"d{n}", "distance", [rng_(0, n), 399]) for n in T.SIMD_SIZES])
    c = T.case_degenerate()
    col = [p for p in c.props if p.name.startswith("a_col") or p.name.startswith("t_line")]
    out["collinear"] = (c.frames, c.cells, (), [(p.name, p.kind, [int(a) for a in p.args]) for p in col])
    fr, cells = T.density_tric_geometry()
    N = fr.shape[2]
    out["density_tric"] = (fr, cells, (), [(f"d{a}", "density", [k, rng_(0, N)]) for k, a in enumerate("xyz")])
    return out


def script_arg(v):
    return f"atom({v[0] + 1}:{v[1]})" if isinstance(v, list) else str(v + 1)


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (frames, cells, zero, stmts) in cases().items():
            frames = np.ascontiguousarray(frames, np.float32); F, _, N = frames.shape
            cell_rows = np.array([c[:6] for c in cells], np.float64); flags = np.array([c[6] for c in cells], np.uint32)
            gro, raw, o, si = (os.path.join(tmp, name + e) for e in (".gro", ".raw", ".out", ".sys"))
            names = ["C"] * N
            for i in zero: names[i] = "X"
            refio.write_gro(gro, np.arange(1, N + 1), ["ATM"] * N, names, np.clip(frames[0].T, -900.0, 9000.0), (100.0, 100.0, 100.0))
            refio.write_raw_traj(raw, frames, cell_rows, flags)
            script = " ".join(f"{s} = {'density_' + 'xyz'[a[0]] + '(' + script_arg(a[1]) + ')' if k == 'density' else k + '(' + ', '.join(script_arg(v) for v in a) + ')'};"
                              for s, k, a in stmts)
            run(HARNESS, "eval", "--sys", gro, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--perframe", f"0:{F}", "--full", f"0:{F}")
            run(HARNESS, "sysinfo", "--sys", gro, "--out", si)
            s = refio.read_sysinfo(si); res = refio.read_refout(o)
            mass = s["mass"]
            assert (mass[list(zero)] == 0).all() and (np.delete(mass, list(zero)) > 0).all(), name
            for st, kind, _ in stmts:
                p = res[st]
                out[f"{name}/{st}"] = np.stack([p.perframe[f][:T.BINS] for f in range(F)]) if kind == "density" else np.asarray(p.full, np.float32).reshape(F, -1)
            out.update({f"{name}/frames": frames, f"{name}/cells": cell_rows, f"{name}/flags": flags, f"{name}/mass": mass,
                        f"{name}/stmts": np.array(json.dumps(stmts))})
            print(name, "ok", script[:120], flush=True)
    path = os.path.join(HERE, "props_edges.npz")
    np.savez_compressed(path, **out)
    print("props_edges.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
