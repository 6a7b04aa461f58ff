"""Generate tests/golden/rmsdctx.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict, `eval`, as make_golden_range.py does):
rmsd() inside `in` contexts (_rmsd md_script_functions.inl:4287-4345 under evaluate_context md_script.c:3418-3500), one value per context and
frame with the per-frame aggregates (mean / variance / extent), on three frame sets:
  a : the ala50 frames of 1ALA (15 residues with bonds: the unwrap's local-index-as-atom quirk walks the bonds of atoms 0..n-1, which belong
      to the first residue, whichever residue the group is)
  w : the water6 frames (orthorhombic cell)
  t : the tric6 frames (triclinic cell changing every frame)
The statements cover the whole residue, an array argument (residue(1:3)), one atom per group (the oxygens of water), two atoms per group
(the hydrogens), a single context, contexts by residue name, a context-relative argument (atom(1:2)) and, on 1ALA, empty groups: the
N-terminal hydrogens H1 / H2 / H3 are in its first residue only. The reference rejects a selection written inside `in` that is empty in some
context ("did not match any atom label within the structure"), so they come through an identifier, which is evaluated once for the system.
residue() and atom() inside a context count from the context's first residue / atom (_comp md_script_functions.inl:3157 remaps and clamps
its range to the context): residue(1:3) in a one-residue context is that residue, so `rr` equals `r`.

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_rmsdctx.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import refio  # noqa: E402
from make_golden import HARNESS, SYNTH, run  # noqa: E402

PDB = "/root/reference/datasets/1ALA-500.pdb"


def script_for(resname, terminal):
    return ("r = rmsd(all) in residue(:); rr = rmsd(residue(1:3)) in residue(:); ro = rmsd(element('O')) in residue(:); "
            "rh = rmsd(element('H')) in residue(:); r7 = rmsd(all) in residue(7); "
            f"rn = rmsd(all) in resname('{resname}'); ra = rmsd(atom(1:2)) in residue(:); "
            + (" nt = name('H1') or name('H2') or name('H3'); re = rmsd(nt) in residue(:);" if terminal else ""))


def main():
    a = np.load(os.path.join(HERE, "ala50.npz")); w = np.load(os.path.join(HERE, "water6.npz")); t = np.load(os.path.join(HERE, "tric6.npz"))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, g, sysfile, resname in (("a", a, PDB, "ALA"), ("w", w, "77", "SOL"), ("t", t, "91", "SOL")):
            if sysfile != PDB:
                gro = os.path.join(tmp, tag + ".gro"); run(SYNTH, "water-gro", "6", sysfile, gro); sysfile = gro
            raw, o = os.path.join(tmp, tag + ".raw"), os.path.join(tmp, tag + ".out")
            F = g["frames"].shape[0]
            refio.write_raw_traj(raw, g["frames"], g["cells"], g["cell_flags"])
            script = script_for(resname, tag == "a")
            run(HARNESS, "eval", "--sys", sysfile, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--full", f"0:{F}")
            for name, p in refio.read_refout(o).items():
                k = f"{tag}_{name}"
                out[k + "__dim"] = np.array(p.dim, np.int32); out[k + "__full"] = p.full
                if p.aggregate is not None: out[k + "__mean"] = p.aggregate["mean"]; out[k + "__var"] = p.aggregate["var"]; out[k + "__ext"] = p.aggregate["ext"]
            out[f"{tag}_script"] = np.array(script)
    path = os.path.join(HERE, "rmsdctx.npz")
    np.savez_compressed(path, **out)
    print("rmsdctx.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
