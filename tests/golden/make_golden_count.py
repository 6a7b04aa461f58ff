"""Generate tests/golden/count6.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict `eval`, as make_golden_range.py does):
count(x, 'atom' | 'residue' | 'chain' | 'structure') (_count_with_arg md_script_functions.inl:5536 -> internal_count :5465-5531) for every dynamic
x the device lowers — within(r, sel), within(a:b, sel), a coordinate range, and `static and <dynamic>` in both orders — on four frame sets:
  w : the water6 frames (orthorhombic cell)
  t : the tric6 frames (triclinic cell changing every frame)
  d : ext/mdlib/test_data/dppc64.pdb (64 DPPC, 3 846 SOL, 14 738 atoms, orthorhombic), 3 frames: only some lipids carry a chain letter, so
      'chain' differs from 'residue'; every lipid and water is one residue and one structure, so 'residue' and 'structure' agree
  p : ext/mdlib/test_data/1a64.pdb (two protein chains, 1 549 atoms), 4 frames: a structure spans many residues
The frames of d and p are the file's coordinates jittered from a stored seed, in the file's cell. Each set also has an empty selection, a range
that holds every atom (the values are the numbers of non-empty groups) and the one-argument count next to 'atom'.

Besides the values, the fixture holds what the Python mirror needs to lower the same statements without the reference: atom names, atomic
numbers, masses, residue offsets, bonds (ref_harness sysinfo), the instance atom ranges and the structures as the reference holds them after
loading (tests/count_lower.c `groups`: md_system_instance_atom_range, md_util_system_infer_structures).

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_count.py
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
import count_lower  # noqa: E402
import refio  # noqa: E402
from make_golden import HARNESS, SYNTH, run  # noqa: E402

TEST_DATA = os.path.join(count_lower.REF, "test_data")
TYPES = ("atom", "residue", "chain", "structure")


def script_for(tag):
    """the statements of one set: every count type x {within, within min:max, range, static and within, range and static}, an empty selection,
    a range holding every atom, and the one-argument form"""
    sel, r, rmin, rng, stat_a, rng_b, stat_b = {
        "w": ("residue(1:5)", "4.5", "2.5:5", "within_z(6:9)", "element('O')", "within_x(3:12)", "element('H')"),
        "t": ("residue(1:5)", "4.5", "2.5:5", "within_z(6:9)", "element('O')", "within_x(3:12)", "element('H')"),
        "d": ("residue(1:3)", "6.0", "3:6", "within_z(40:60)", "element('O')", "within_x(10:25)", "element('C')"),
        "p": ("residue(1:6)", "5.0", "2.5:5", "within_z(0:10)", "element('N')", "within_x(0:15)", "element('C')"),
    }[tag]
    out = []
    for t in TYPES:
        c = t[0]
        out += [f"{c}w = count(within({r}, {sel}), '{t}');",
                f"{c}m = count(within({rmin}, {sel}), '{t}');",
                f"{c}r = count({rng}, '{t}');",
                f"{c}s = count({stat_a} and within({r}, {sel}), '{t}');",
                f"{c}t = count({rng_b} and {stat_b}, '{t}');",
                f"{c}e = count(within_x(9000:9999), '{t}');",
                f"{c}a = count(within_xyz(:, :, :), '{t}');"]
    out.append(f"one = count(within({r}, {sel}));")
    return " ".join(out)


def pdb_set(tmp, name, seed, F):
    """the file's coordinates jittered by N(0, 0.25 A) per frame, in the file's cell"""
    info = os.path.join(tmp, name + ".sys"); pdb = os.path.join(TEST_DATA, name + ".pdb")
    run(HARNESS, "sysinfo", "--sys", pdb, "--out", info)
    s = refio.read_sysinfo(info)
    rng = np.random.default_rng(seed)
    base = np.stack([s["x"], s["y"], s["zc"]]).astype(np.float64)
    frames = np.stack([base + rng.normal(0.0, 0.25, base.shape) for _ in range(F)]).astype(np.float32)
    cells = np.tile(np.asarray(s["cell"][:6], np.float64), (F, 1)); flags = np.full(F, s["cell"][6], np.uint32)
    return pdb, s, frames, cells, flags


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    w = np.load(os.path.join(HERE, "water6.npz")); t = np.load(os.path.join(HERE, "tric6.npz"))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        lower = count_lower.build(tmp)
        sets = []
        for tag, g, seed in (("w", w, "77"), ("t", t, "91")):
            gro = os.path.join(tmp, tag + ".gro"); run(SYNTH, "water-gro", "6", seed, gro)
            info = os.path.join(tmp, tag + ".sys"); run(HARNESS, "sysinfo", "--sys", gro, "--out", info)
            sets.append((tag, gro, refio.read_sysinfo(info), g["frames"][:4], g["cells"][:4], g["cell_flags"][:4], int(seed)))
        for tag, name, seed, F in (("d", "dppc64", 5101, 3), ("p", "1a64", 5102, 4)):
            sets.append((tag, *pdb_set(tmp, name, seed, F), seed))
        for tag, path, s, frames, cells, flags, seed in sets:
            F = len(frames); script = script_for(tag)
            raw, o = os.path.join(tmp, tag + ".raw"), os.path.join(tmp, tag + ".out")
            refio.write_raw_traj(raw, frames, cells, flags)
            run(HARNESS, "eval", "--sys", path, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--full", f"0:{F}")
            for k, p in refio.read_refout(o).items():
                assert p.flags & refio.FLAG_TEMPORAL and tuple(p.dim[:2]) == (F, 1), (tag, k, p.flags, p.dim)
                out[f"{tag}_{k}"] = p.full
            grp = count_lower.groups(lower, path)
            assert np.array_equal(np.asarray(grp["components"], np.uint32), s["comp_off"]), tag
            out.update({f"{tag}_script": np.array(script), f"{tag}_frames": frames, f"{tag}_cells": cells, f"{tag}_cell_flags": flags,
                        f"{tag}_seed": np.int32(seed), f"{tag}_mass": s["mass"], f"{tag}_z": s["z"].astype(np.uint8),
                        f"{tag}_names": np.array(s["names"]), f"{tag}_comp_off": s["comp_off"], f"{tag}_conn_off": s["conn_off"],
                        f"{tag}_conn_idx": s["conn_idx"], f"{tag}_chains": np.asarray(grp["instances"], np.int64).reshape(-1, 2),
                        f"{tag}_struct_off": np.asarray(grp["structure_offsets"], np.uint32), f"{tag}_struct_atoms": np.asarray(grp["structure_atoms"], np.int32)})
            # the forms differ where the set is meant to tell them apart, and every statement selects something in some frame but the empty one
            for c in "arcs":
                assert out[f"{tag}_{c}e"].sum() == 0 and out[f"{tag}_{c}w"].sum() > 0, (tag, c)
            assert np.array_equal(out[f"{tag}_aw"], out[f"{tag}_one"]), tag
            if tag == "d": assert not np.array_equal(out["d_ca"], out["d_ra"]) and np.array_equal(out["d_ra"], out["d_sa"]), "dppc: chain vs residue / structure"
            if tag == "p": assert not np.array_equal(out["p_sw"], out["p_rw"]), "1a64: structure vs residue"
    path = os.path.join(HERE, "count6.npz")
    np.savez_compressed(path, **out)
    print("count6.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
