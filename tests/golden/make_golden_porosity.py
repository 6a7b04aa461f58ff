"""Generate tests/golden/porosity.npz from the UNMODIFIED reference sources: porosity() evaluated per frame by oracle/_ref/ref_harness_zt
(`eval --perframe`; ref_harness_strict with cleared temporary allocations, without which the reference's bit grid starts from stale memory,
see oracle/porosity.mk), the radii of each system from oracle/_ref/radii_harness (md_atom_extract_radii; `make -C oracle -f porosity.mk`). Needs
/root/reference. The fixture stores the inputs (frames, cells, radii, selections, scripts) with the reference's values, so the tests need neither.

  porosity.npz, per case <c> in CASES:
    <c>_script, <c>_frames [F, 3, N], <c>_cells [F, 6], <c>_flags [F], <c>_radius [N], and per property <p> of the script
    <c>_<p>_idx (the selection's atoms, ascending) and <c>_<p>_values [F] (the reference's per-frame values).

  wx : water box (n = 6, 648 atoms, orthorhombic, x shifted by -3 A and wrapped): porosity(residue(1:6)), a prefix selection (one row of
       molecules) whose box is a thin slab, so that the grid has at most 2^23 voxels and the float value pins the occupied count; the row crosses
       the periodic boundary in x, so the spheres must be deperiodised about their centre of mass; and porosity(all) (512^3 grid: float regime).
  ala: porosity(all) on the first 6 frames of 1ALA-500 (153 atoms, float regime).
  tri: the water box sheared into a triclinic cell: the reference returns 0.

  python tests/golden/make_golden_porosity.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import refio  # noqa: E402

HARNESS = os.path.join(ROOT, "oracle", "_ref", "ref_harness_zt")   # ref_harness_strict with cleared temporaries (oracle/porosity.mk)
RADII = os.path.join(ROOT, "oracle", "_ref", "radii_harness")
SYNTH = os.path.join(ROOT, "oracle", "build", "synth_tool")
ALA = "/root/reference/datasets/1ALA-500.pdb"


def run(*a):
    subprocess.check_call(list(a), stdout=subprocess.DEVNULL)


def radii(tmp, sysfile):
    o = os.path.join(tmp, "r.bin"); run(RADII, "radii", "--sys", sysfile, "--out", o)
    b = open(o, "rb").read(); assert b[:8] == b"MDRADII\0"
    n = int(np.frombuffer(b, np.uint64, 1, 8)[0]); return np.frombuffer(b, np.float32, n, 16).copy()


def evaluate(tmp, sysfile, raw, script, F):
    o = os.path.join(tmp, "p.out")
    run(HARNESS, "eval", "--sys", sysfile, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--perframe", f"0:{F}")
    return {name: np.array([p.perframe[f][0] for f in range(F)], np.float32) for name, p in refio.read_refout(o).items()}


def case(out, tag, tmp, sysfile, frames, cells, flags, script, sels):
    raw = os.path.join(tmp, f"{tag}.raw"); refio.write_raw_traj(raw, frames, cells, flags)
    vals = evaluate(tmp, sysfile, raw, script, len(frames))
    out.update({f"{tag}_script": np.array(script), f"{tag}_frames": frames, f"{tag}_cells": cells, f"{tag}_flags": flags, f"{tag}_radius": radii(tmp, sysfile)})
    for name, idx in sels.items():
        out[f"{tag}_{name}_idx"] = np.asarray(idx, np.int32); out[f"{tag}_{name}_values"] = vals[name]


def main(tmp):
    out = {}
    n, seed, F = 6, 77, 4
    gro, raw0 = os.path.join(tmp, "w.gro"), os.path.join(tmp, "w0.raw")
    run(SYNTH, "water-gro", str(n), str(seed), gro); run(SYNTH, "water-raw", str(n), str(seed), str(F), raw0)
    fr, cells, flags = refio.read_raw_traj(raw0)
    fr[:, 0] = np.mod(fr[:, 0].astype(np.float64) - 3.0, cells[:, :1]).astype(np.float32)   # shift x by -3 A and wrap: the first row of molecules straddles x = 0
    na = fr.shape[2]
    case(out, "wx", tmp, gro, fr, cells, flags, "px = porosity(residue(1:6)); pa = porosity(all);", {"px": np.arange(18), "pa": np.arange(na)})
    tcells = cells.copy(); tcells[:, 1] = 3.1; tcells[:, 2] = -2.2; tcells[:, 4] = 4.3   # xy, xz, yz
    case(out, "tri", tmp, gro, fr[:2], tcells[:2], np.full(2, 2 | 4 | 8 | 16, np.uint32), "pt = porosity(all);", {"pt": np.arange(na)})
    araw = os.path.join(tmp, "a.raw"); run(HARNESS, "dumptraj", "--sys", ALA, "--traj", "sys", "--frames", "0:6", "--out", araw)
    afr, acells, aflags = refio.read_raw_traj(araw)
    case(out, "ala", tmp, ALA, afr, acells, aflags, "pa = porosity(all);", {"pa": np.arange(afr.shape[2])})
    np.savez_compressed(os.path.join(HERE, "porosity.npz"), **out)


if __name__ == "__main__":
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "-f", "porosity.mk"])
    with tempfile.TemporaryDirectory() as tmp:
        main(tmp)
    print("porosity.npz", os.path.getsize(os.path.join(HERE, "porosity.npz")), "bytes")
