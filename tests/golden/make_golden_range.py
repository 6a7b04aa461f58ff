"""Generate tests/golden/range6.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict, `eval`, as make_golden.py's dyn6 does):
coordinate-range selections within_x / within_y / within_z / within_xyz (md_script_functions.inl:668-671, coordinate_range :2394-2476) as the
argument of every consumer the device path lowers — rdf reference and target, sdf target, density_x / _z, the centre of mass of distance /
angle / com, distance_min / _max, count() — alone and `and` a static selection in both orders, on three sets of 4 frames:
  w : the water6 frames (orthorhombic cell)
  t : the tric6 frames (triclinic cell changing every frame)
  u : the tric6 frames with residues 1-40 moved by +a, residues 100-130 by -c and residues 150-160 by +b - c: an unwrapped trajectory whose
      atoms lie outside the unit cell; a range selects them by their raw coordinates. Its script has no rdf(): the reference's rdf faults
      (SIGSEGV) on such frames, with or without a range.
Each set has its own script, because some bounds are copied from atom coordinates of its frame 2 (bounds exactly on an atom: both ends are
inclusive). The script also holds a slab that is empty on some frames, ranges that hold every atom, an empty static side and open-ended
ranges: the parser accepts `a:`, `:b` and `:` (an integer range keeps INT32_MIN / INT32_MAX for open ends, cast to float; a float range uses
-FLT_MAX / FLT_MAX). It rejects negative bounds (`within_x(-5:10)`: no unary minus on a range), so none appear.

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_range.py
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
from make_golden import HARNESS, SYNTH, run, pack  # noqa: E402

F = 4


def f32(v):
    """the shortest decimal that reads back as this float32 (through the parser's double -> float)"""
    return np.format_float_positional(np.float32(v), unique=True, trim="-")


def script_for(frames, with_rdf):
    """the statements of one frame set; bounds marked `on atom` are coordinates of frame 2"""
    x, y, z = frames[2]
    zs = np.sort(z[z > 0])   # the script language has no negative range bounds
    thin_lo = zs[100]; thin_hi = np.nextafter(thin_lo, np.float32(np.inf))   # one or two atoms of frame 2, none on most other frames
    assert min(x[10], x[30], y[50], y[70], x[5], y[5], z[5]) > 0
    rdf = [   # range as reference (static side before / after), as target, on both sides, every atom
        "rr = rdf(element('O') and within_z(4:12), element('O'), 6.0);",
        "rt = rdf(element('O'), within_x(2.5:9.5) and element('H'), 5.0);",
        "rb = rdf(within_z(0:9), within_z(9:19), 4.0);",
        "ra = rdf(within_z(:), element('O'), 5.0);",
    ]
    return " ".join((rdf if with_rdf else []) + [
        # bounds exactly on atom coordinates (frame 2): atom 11's x .. atom 31's x, atom 51's y .. atom 71's y, the point of atom 6
        f"cx = count(within_x({f32(min(x[10], x[30]))}:{f32(max(x[10], x[30]))}));",
        f"cy = count(element('H') and within_y({f32(min(y[50], y[70]))}:{f32(max(y[50], y[70]))}));",
        f"cz = count(within_xyz({f32(x[5])}:{f32(x[5])}, {f32(y[5])}:{f32(y[5])}, {f32(z[5])}:{f32(z[5])}));",
        # a slab that is empty on some frames
        f"ce = count(within_z({f32(thin_lo)}:{f32(thin_hi)}));",
        f"de = density_z(within_z({f32(thin_lo)}:{f32(thin_hi)}) and element('O'));",
        # sdf target, density
        "vs = sdf(residue(1:20), within_y(3:14) and element('O'), 5.0);",
        "dz = density_z(element('O') and within_x(0:9));",
        "dx = density_x(within_xyz(0:10, 2:16, 5:15));",
        # centre of mass of a range selection: distance / angle / com; distance_min / _max
        "dr = distance(within_z(2:6) and element('O'), 200);",
        "ar = angle(within_x(1:5), 10, residue(7));",
        "cm = com(within_y(5.5:7.25));",
        "dm = distance_min(within_z(0:3), residue(30));",
        "dn = distance_max(element('H') and within_y(10:12), residue(3));",
        # count: bare, `and` in both orders, empty static side, every atom, open ends
        "c1 = count(within_z(6:9));",
        "c2 = count(element('O') and within_z(6:9));",
        "c3 = count(within_x(3:15) and element('H'));",
        "c4 = count((atom(1:3) and residue(10)) and within_z(:));",
        "c5 = count(within_xyz(:, :, :));",
        "c6 = count(within_z(10:));",
        "c7 = count(within_y(:5));",
        "c8 = count(within_x(7.5:));",
    ])


def shifted_tric(t):
    """tric6 frames with some residues moved by lattice vectors: the same periodic system, atoms outside the unit cell"""
    fr = t["frames"].astype(np.float64).copy(); cells = t["cells"]
    for f in range(F):
        L, xy, xz, Ly, yz, Lz = (float(v) for v in cells[f])
        a, b, c = np.array([L, 0, 0]), np.array([xy, Ly, 0]), np.array([xz, yz, Lz])
        for (r0, r1), v in (((1, 40), a), ((100, 130), -c), ((150, 160), b - c)):   # residues of 3 atoms, 1-based inclusive
            s = slice(3 * (r0 - 1), 3 * r1)
            for k in range(3): fr[f, k, s] += v[k]
    return fr.astype(np.float32)


def main():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    w = np.load(os.path.join(HERE, "water6.npz")); t = np.load(os.path.join(HERE, "tric6.npz"))
    out = {}
    sets = (("w", w["frames"][:F], w["cells"][:F], w["cell_flags"][:F], "77"), ("t", t["frames"][:F], t["cells"][:F], t["cell_flags"][:F], "91"),
            ("u", shifted_tric(t), t["cells"][:F], t["cell_flags"][:F], "91"))
    with tempfile.TemporaryDirectory() as tmp:
        for tag, frames, cells, flags, seed in sets:
            script = script_for(frames, tag != "u")
            gro, raw, o = os.path.join(tmp, tag + "r.gro"), os.path.join(tmp, tag + "r.raw"), os.path.join(tmp, tag + "r.out")
            run(SYNTH, "water-gro", "6", seed, gro); refio.write_raw_traj(raw, frames, cells, flags)
            run(HARNESS, "eval", "--sys", gro, "--traj", f"raw:{raw}", "--script", script, "--out", o, "--perframe", f"0:{F}", "--full", f"0:{F}")
            sub = {}; pack(sub, refio.read_refout(o), list(range(F)))
            for k, v in sub.items(): out[f"{tag}_{k}"] = v
            out[f"{tag}_script"] = np.array(script); out[f"{tag}_frames"] = frames; out[f"{tag}_cells"] = cells; out[f"{tag}_cell_flags"] = flags
            out[f"{tag}_seed"] = np.int32(int(seed))
    path = os.path.join(HERE, "range6.npz")
    np.savez_compressed(path, **out)
    print("range6.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
