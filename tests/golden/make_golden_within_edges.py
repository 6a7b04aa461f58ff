"""Generate tests/golden/within_edges.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict `eval` on raw trajectories, as
make_golden_count.py does): count(within(r, atom(1:k))) and count(within(a:b, atom(1:k))) per frame on the adversarial geometries of
tests/test_dynamic_selection_edges.py, built by that file's frame builders from the seeds stored below:
  pileup        coordinates from {0, -0, 3, 6, 12, 18, L, nextafter(L, 0)} in a 24 A box; radii 6, 5.99, 3 and the window 3:6
  large_radius  an 18.6 A box (frames 0-1) and a 17.2 A box (frame 2); radii 9.4, 12, 17 (one cell, reach 1) and 40 (reach 3: no pairs)
  triclinic     a shear changing every frame, atoms wrapped into the cell
  nonperiodic   one non-periodic axis per frame, then a frame without a cell; 30 % of the atoms outside the cell
  cellless      1 000 atoms over 320 A without a cell, radius 2
The system file is a .gro of single-atom residues (the raw trajectory supplies every coordinate and cell).

Left out because the reference harness faults (SIGSEGV) on them, so their reference behaviour is undefined (and the device table leaves them out):
  - neighbour reach 2 on a one-cell grid: within(25, ...) in an 18.6 A box, within(12 or 17, ...) in an 11 A box;
  - unwrapped triclinic frames (20 % of the atoms moved by +a, with or without -b as well), at radius 3.5 and 7;
  - frames without a cell with 1 200 atoms or more, whatever their extent (100 A to 320 A), at radius 2 and 6.

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_within_edges.py
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
from make_golden import HARNESS, run  # noqa: E402
import test_dynamic_selection_edges as T  # noqa: E402

SEEDS = {"pileup": 501, "large_radius": 502, "triclinic": 503, "nonperiodic": 504, "cellless": 505}


def cases():
    """name -> (frames [F, 3, N], cells [(x, xy, xz, y, yz, z, flags)] per frame, [(statement name, k, rmin, rmax)])"""
    fr, L = T.frames_pileup(SEEDS["pileup"])
    out = {"pileup": (fr, [T.ortho(L, L, L)] * len(fr), [("c6", 40, 0.0, 6.0), ("c599", 40, 0.0, 5.99), ("c3", 40, 0.0, 3.0), ("m36", 40, 3.0, 6.0)])}
    boxes = [(18.6,) * 3] * 2 + [(17.2,) * 3]
    out["large_radius"] = (T.frames_box(SEEDS["large_radius"], 260, boxes, 0.05), [T.ortho(*b) for b in boxes],
                           [(f"c{r:g}".replace(".", "_"), 3, 0.0, r) for r in (9.4, 12.0, 17.0, 40.0)] + [("m912", 3, 9.0, 12.0), ("m1217", 3, 12.0, 17.0)])
    fr, cells = T.frames_triclinic(SEEDS["triclinic"])
    out["triclinic"] = (fr, cells, [("c35", 20, 0.0, 3.5), ("c7", 20, 0.0, 7.0), ("m27", 20, 2.0, 7.0)])
    fr, cells = T.frames_nonperiodic(SEEDS["nonperiodic"])
    out["nonperiodic"] = (fr, cells, [("c4", 20, 0.0, 4.0), ("c75", 20, 0.0, 7.5), ("m2575", 20, 2.5, 7.5)])
    out["cellless"] = (T.frames_cellless_large(SEEDS["cellless"]), [T.NO_CELL] * 2, [("c2", 50, 0.0, 2.0), ("m12", 50, 1.0, 2.0)])
    return out


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (frames, cells, stmts) in cases().items():
            frames = np.ascontiguousarray(frames, np.float32); F, _, N = frames.shape
            cell_rows = np.array([c[:6] for c in cells], np.float64); flags = np.array([c[6] for c in cells], np.uint32)
            gro, raw, o = (os.path.join(tmp, name + e) for e in (".gro", ".raw", ".out"))
            refio.write_gro(gro, np.arange(1, N + 1), ["ATM"] * N, ["C"] * N, np.zeros((N, 3)), (100.0, 100.0, 100.0))
            refio.write_raw_traj(raw, frames, cell_rows, flags)
            script = " ".join(f"{s} = count(within({f'{rmin:.2f}:' if rmin else ''}{rmax:.2f}, atom(1:{k})));" for s, k, rmin, rmax in stmts)
            run(HARNESS, "eval", "--sys", gro, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--full", f"0:{F}")
            res = refio.read_refout(o)
            for s, k, rmin, rmax in stmts:
                p = res[s]
                assert p.flags & refio.FLAG_TEMPORAL and tuple(p.dim[:2]) == (F, 1), (name, s, p.flags, p.dim)
                out[f"{name}/{s}"] = np.asarray(p.full, np.float32).reshape(F)
            out.update({f"{name}/frames": frames, f"{name}/cells": cell_rows, f"{name}/flags": flags, f"{name}/seed": np.int32(SEEDS[name]),
                        f"{name}/stmts": np.array([s for s, *_ in stmts]), f"{name}/k": np.array([k for _, k, _, _ in stmts], np.int32),
                        f"{name}/rmin": np.array([r for _, _, r, _ in stmts], np.float32), f"{name}/rmax": np.array([r for *_, r in stmts], np.float32)})
    path = os.path.join(HERE, "within_edges.npz")
    np.savez_compressed(path, **out)
    print("within_edges.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
