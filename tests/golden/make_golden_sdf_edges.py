"""Generate tests/golden/sdf_edges.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict `eval` on raw trajectories, as
make_golden_within_edges.py does): the per-frame voxels of sdf(residue(a:b), atom(c:d), r) on geometries of tests/test_sdf_edges.py,
built by that file's case builders:
  ring_ortho      16 twelve-atom rings (1.4 A bonds) + 500 single atoms in a 26 A box, rings 0 and 1 across the periodic faces
  ring_triclinic  the same in a sheared cell whose shear changes every frame
  tree_ortho      16 ten-atom branched trees (1.5 A bonds) across the faces of a 26 A box
  shear           120 three-atom molecules in a triclinic cell whose shear changes every frame
  npt             150 three-atom molecules in a cubic box of 22.0, 20.4, 23.6 and 21.2 A (the initial frame unwrapped with each frame's box)
  nonperiodic     one non-periodic axis per frame, then a frame without a cell; 15 % of the atoms outside the box on each side
  cellless        the same 800 atoms without a cell in every frame
  large_cutoff    cutoffs 8 and 9.5 in a 14.4 A box (a one-cell grid)
The system file is a .gro whose residues are the molecules (or the atom triples) of the case, written whole (frame 0 unwrapped along
the molecules), so the bonds the reference infers from it are the molecules' own: the ring and tree bonds are at covalent spacing and
the generator checks that the inferred bonds among the atoms of the first ring or tree are exactly the template's. The reference's masses, bonds and residue
offsets are stored with the frames; the raw trajectory supplies every coordinate and cell.

Left out: frames without a cell beyond about 1 000 atoms, on which the reference harness faults (see make_golden_within_edges.py); the
non-periodic and cell-less systems here have 800 atoms. Targets are atom ranges (atom(c:d)), as the script addresses them.

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_sdf_edges.py
"""
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
from make_golden import HARNESS, run, sparse  # noqa: E402
import test_sdf_edges as T  # noqa: E402


def whole(p, cell, mol_size, n_mol):
    """frame [3, N] -> molecules 0 .. n_mol - 1 of mol_size atoms made whole about their first atom (minimum image in the cell)"""
    p = p.astype(np.float64).copy()
    x, xy, xz, y, yz, z, flags = cell
    if not flags & T.PBC_ALL: return p
    A = np.array([[x, 0, 0], [xy, y, 0], [xz, yz, z]], np.float64); Ai = np.linalg.inv(A)
    for m in range(n_mol):
        s = slice(m * mol_size, (m + 1) * mol_size)
        d = (p[:, s] - p[:, s][:, :1]).T @ Ai
        d -= np.round(d)
        p[:, s] = (d @ A).T + p[:, s][:, :1]
    return p


def cases():
    """name -> (case, molecule size, molecule count, template bonds to check (() for molecules not checked, None for atom triples that are not
    molecules), [(statement, res_a, res_b, trg_a, trg_b, cutoff)])"""
    out = {}
    for name, make, tmpl in (("ring_ortho", T.case_ring_ortho, T.ring), ("ring_triclinic", T.case_ring_triclinic, T.ring), ("tree_ortho", T.case_tree_ortho, T.tree)):
        c = make(); n = len(tmpl()[0]); N = c.frames.shape[2]
        out[name] = (c, n, 16, tmpl()[1], [("v", 1, 16, 1, N, 6.0), ("vs", 1, 8, 16 * n + 1, N, 4.5)])
    c = T.case_shear(); N = c.frames.shape[2]
    out["shear"] = (c, 3, 120, (), [("v", 1, 120, 1, N, 5.0), ("v7", 1, 30, 361, N, 7.0)])
    c = T.case_npt(); N = c.frames.shape[2]
    out["npt"] = (c, 3, 150, (), [("v", 1, 150, 1, N, 5.0), ("v8", 1, 20, 1, N, 8.0)])
    c = T.case_nonperiodic(); N = c.frames.shape[2]
    out["nonperiodic"] = (c, 3, 100, None, [("v", 1, 100, 1, N, 5.0), ("v7", 1, 30, 1, 400, 7.0)])
    c = T.case_nonperiodic(); c.cells = [T.NO_CELL] * c.frames.shape[0]
    out["cellless"] = (c, 3, 100, None, [("v", 1, 100, 1, N, 5.0), ("v7", 1, 30, 1, 400, 7.0)])
    c = T.case_large_cutoff(); N = c.frames.shape[2]
    out["large_cutoff"] = (c, 3, 40, (), [("c8", 1, 40, 1, N, 8.0), ("c95", 1, 20, 1, N, 9.5)])
    return out


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (case, n, n_mol, tbonds, stmts) in cases().items():
            frames = case.frames; F, _, N = frames.shape
            cell_rows = np.array([c[:6] for c in case.cells], np.float64); flags = np.array([c[6] for c in case.cells], np.uint32)
            gro, raw, o, si = (os.path.join(tmp, name + e) for e in (".gro", ".raw", ".out", ".sys"))
            resid = np.concatenate([np.repeat(np.arange(1, n_mol + 1), n), n_mol + 1 + np.arange(N - n * n_mol)])
            pos = whole(frames[0], case.cells[0], n, n_mol) if tbonds is not None else frames[0].astype(np.float64)
            refio.write_gro(gro, resid, ["MOL"] * (n * n_mol) + ["ATM"] * (N - n * n_mol), ["C"] * N, pos.T, (100.0, 100.0, 100.0))
            refio.write_raw_traj(raw, frames, cell_rows, flags)
            script = " ".join(f"{s} = sdf(residue({a}:{b}), atom({ta}:{tb}), {r:.2f});" for s, a, b, ta, tb, r in stmts)
            run(HARNESS, "eval", "--sys", gro, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--perframe", f"0:{F}")
            run(HARNESS, "sysinfo", "--sys", gro, "--out", si)
            s = refio.read_sysinfo(si); res = refio.read_refout(o)
            comp = s["comp_off"]
            assert np.array_equal(comp[:n_mol + 1], np.arange(n_mol + 1) * n), name
            co, ci = s["conn_off"], s["conn_idx"]
            if tbonds:   # the inferred bonds among atoms 0 .. n - 1 (those the walk follows) are the template's
                got = {(a, int(b)) for a in range(n) for b in ci[co[a]:co[a + 1]] if b < n}
                assert got == {(a, b) for a, b in tbonds} | {(b, a) for a, b in tbonds}, (name, sorted(got))
            for st, *_ in stmts:
                p = res[st]
                assert p.flags & refio.FLAG_VOLUME, (name, st, p.flags)
                for f in range(F):
                    i, v = sparse(p.perframe[f]); out[f"{name}/{st}/pf{f}_idx"] = i; out[f"{name}/{st}/pf{f}_val"] = v
                    assert v.sum() > 0, (name, st, f)
            out.update({f"{name}/frames": frames, f"{name}/cells": cell_rows, f"{name}/flags": flags, f"{name}/mass": s["mass"],
                        f"{name}/conn_off": co, f"{name}/conn_idx": ci, f"{name}/comp_off": comp, f"{name}/stmts": np.array([x[0] for x in stmts]),
                        f"{name}/res_a": np.array([x[1] for x in stmts], np.int32), f"{name}/res_b": np.array([x[2] for x in stmts], np.int32),
                        f"{name}/trg_a": np.array([x[3] for x in stmts], np.int32), f"{name}/trg_b": np.array([x[4] for x in stmts], np.int32),
                        f"{name}/cutoff": np.array([x[5] for x in stmts], np.float32)})
            print(name, "ok", flush=True)
    path = os.path.join(HERE, "sdf_edges.npz")
    np.savez_compressed(path, **out)
    print("sdf_edges.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
