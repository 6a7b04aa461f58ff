"""The per-frame temporal and distribution kernels against the plain-C oracle on adversarial geometries.

props.cu evaluates distance / angle / dihedral / com (k_arg_com, k_arg_com_parts -> k_arg_combine, k_temporal, k_temporal_ctx, k_com_rows),
distance_min / _max / _pair (k_min_distance, k_distance_pair), coord (k_coord_rows) and density_x/_y/_z (k_density, k_density_finalize); sdf.cu
evaluates rmsd (k_rmsd, k_rmsd_groups), plane (k_plane) and shape_weights (k_shape_weights); pbcmath.cuh holds the cell routines they share.
The case table below drives the paths where these go wrong:
  simd split   selections of 1, 7, 8, 9, 15, 16, 17 and 67 atoms as an argument of distance, angle, dihedral and com, with no cell, an
               orthorhombic and a triclinic cell: periodic_com_warp runs only the double tail below 8 atoms, the 8 emulated lanes + reduce8 +
               the tail above
  masses       all-zero masses (the periodic centre takes theta = pi, the plain one and com_vec4 divide 0 by 0), some zero, masses below 1 u,
               masses of 256 u and more (k_density's high limb directly)
  cells        each axis non-periodic in turn, a strong triclinic shear (|xy|, |xz|, |yz| up to L/2) and a box that change inside one batch,
               distance() in a triclinic cell (deperiodises nothing)
  far images   single-atom dihedrals whose bond vectors span 3, 64, 65, 200 and 1 000 box lengths along each axis, orthorhombic and triclinic
               (the minimum-image loop runs that many steps); distances, pair distances and density of atoms as far outside the cell
  faces, ties  atoms on cell faces, at rc +- ext/2 of density's deperiodisation (rintf ties to even), on density bin edges and one float ulp
               either side, in bins 0 and 1023 and beyond (the clamp)
  degenerate   coincident atoms (normalize3 below 1e-5), collinear angles whose dot product rounds past +-1 (acosf -> NaN), collinear
               dihedrals (w = 0, atan2f(0, +0)), planar and collinear sets for plane() (which rejects fewer than 3 atoms), planar and
               single-atom sets for shape_weights(), an rmsd structure equal to the initial frame and one whose bonds cross a periodic face
  arg forms    atoms, selections, arrays of selections, `in` contexts with empty context groups (k_temporal_ctx, k_rmsd_groups), a within()
               argument that is empty in some frames
  pairs        distance_min / _max / _pair at 200, 256, 260 and 75 000 pairs (below, at and above the CTA, above 2^16), an empty dynamic side
               (FLT_MAX), exact ties on a lattice
  density      5 000 atoms (three CTAs per frame merge through the global atomics), 40 atoms of 16 u in one bin of one CTA (the low limb wraps
               and carries), a zero-extent axis of the initial cell (inv_ext = 0: every atom in bin 0), a triclinic initial cell (rc holds the
               shear), a within() selection

Each case is compared with oracle_lib frame by frame (plan.clear(), one frame) and as whole runs at batch_frames 1 and the default with one
and two stream slots. Under the CPU emulation (tests/emul) every value equals the oracle's bit for bit (NaN equals NaN, the sign of a zero
counts). On the device the values that pass through no libm function are bit-equal as well: distance and com of atoms or without a cell,
distance_min / _max / _pair, coord and the density counts. angle, dihedral, the periodic centre of mass, plane, rmsd and shape_weights go
through acosf / atan2f / double atan2, whose CUDA results can differ from glibc's in the last ulp: they are held to 1e-5 (relative above 1),
NaN must match NaN and +-pi count as equal; the test prints how many of them were bit-equal.

Density counts are checked exactly: k_density's bin of every atom restated in numpy in its float32 operation order, plus round(mass * 2^24)
summed as integers. The restatement's bins equal the oracle's (the oracle run with unit masses counts atoms, exactly); with integer masses the
oracle's float sums are exact, and the counts scaled back equal the oracle's bins value for value.

Geometries on which the reference itself never terminates (an infinite coordinate difference, or one so large that dx - box == dx in the
dihedral's minimum-image loop) are left out of the table: the library returns NaN there instead, which
test_dihedral_minimum_image_loop_stops_with_nan checks without the oracle. tests/golden/props_edges.npz pins the oracle to the unmodified
reference on a part of the table (make_golden_props_edges.py).
"""
import os
import sys

import numpy as np
import pytest

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
PBC_X, PBC_Y, PBC_Z, ORTHO, TRICLINIC = 4, 8, 16, 1, 2
PBC_ALL = PBC_X | PBC_Y | PBC_Z
NO_CELL = (0.0,) * 6 + (0,)
BINS = 1024
TOL = 1e-5          # DESIGN.md section 2: values that pass through libm
SIMD_SIZES = (1, 7, 8, 9, 15, 16, 17, 67)
FAR = (3, 64, 65, 200, 1000)


def ortho(x, y, z, flags=ORTHO | PBC_ALL):
    return (float(x), 0.0, 0.0, float(y), 0.0, float(z), flags)


def tric(L, sxy, sxz, syz, Ly=None, Lz=None):
    return (float(L), sxy * L, sxz * L, float(Ly or L), syz * L, float(Lz or L), TRICLINIC | PBC_ALL)


def basis(cell):
    """rows a, b, c of the cell as float64 [3, 3]"""
    x, xy, xz, y, yz, z, _ = cell
    return np.array([[x, 0, 0], [xy, y, 0], [xz, yz, z]], np.float64)


def in_cell(rng, N, cell):
    """[3, N] points uniformly inside the cell (inside [0, 20)^3 without one)"""
    A = basis(cell) if cell[6] else np.eye(3) * 20.0
    return (rng.random((N, 3)) @ A).T


def csr(N, bonds):
    nb = [[] for _ in range(N)]
    for a, b in bonds: nb[a].append(b); nb[b].append(a)
    off = np.zeros(N + 1, np.uint32); off[1:] = np.cumsum([len(n) for n in nb])
    idx = np.array([j for n in nb for j in sorted(n)], np.int32)
    return off, (idx if len(idx) else np.zeros(1, np.int32))


class Within:
    def __init__(self, radius, sel):
        self.radius, self.sel = float(radius), np.asarray(sel, np.int32)

    def vb(self):
        import viamd_b200 as vb
        return vb.Within(self.radius, self.sel)

    def oracle(self, x, y, z, cell):
        return O.within(x, y, z, self.sel, self.radius, cell)


# ----------------------------------------------------------------------------------------------------------------------------- properties
class P:
    """one property of a case: kind in distance, angle, dihedral, com, dmin, dmax, dpair, coord, plane, rmsd, shape, ctx, density.
    Position arguments: an int (an atom), an index array (a selection), a list of index arrays (an array of selections) or a Within."""
    def __init__(self, name, kind, *args):
        self.name, self.kind, self.args = name, kind, args

    def prop(self):
        import viamd_b200 as vb
        from viamd_b200 import api
        k, a = self.kind, [x.vb() if isinstance(x, Within) else x for x in self.args]
        if k in ("distance", "angle", "dihedral", "com"): return getattr(vb, k)(self.name, *a)
        if k == "dmin": return vb.distance_min(self.name, *a)
        if k == "dmax": return vb.distance_max(self.name, *a)
        if k == "dpair": return vb.distance_pair(self.name, *a)
        if k == "coord": return vb.coord(self.name, a[0], a[1])
        if k == "plane": return vb.plane(self.name, a[0])
        if k == "rmsd": return vb.rmsd(self.name, a[0])
        if k == "shape": return vb.shape_weights(self.name, a[0], a[1])
        if k == "ctx": return vb.in_contexts(self.name, {"distance": api.OP_DISTANCE, "angle": api.OP_ANGLE, "dihedral": api.OP_DIHEDRAL}[a[0]], a[1], a[2])
        if k == "density": return vb.density(self.name, a[0], a[1])
        raise ValueError(k)

    def exact(self, flags):
        """True where the device value passes through no libm function in a frame with these cell flags"""
        if self.kind in ("dmin", "dmax", "dpair", "coord", "density"): return True
        if self.kind in ("distance", "com"): return flags == 0 or all(isinstance(x, (int, np.integer)) for x in self.args)
        if self.kind == "ctx": return self.args[0] == "distance" and (flags == 0 or all(isinstance(x, (int, np.integer)) for x in self.args[1]))
        return False


def _pos_arg(a, x, y, z, oc):
    return a.oracle(x, y, z, oc) if isinstance(a, Within) else a


def oracle_values(case, p, f):
    """float32 values of temporal p in frame f"""
    x, y, z = case.frames[f]; oc = O.UnitCell(*case.cells[f]); m = case.mass
    a = [_pos_arg(v, x, y, z, oc) for v in p.args]
    k = p.kind
    if k == "distance": v = [O.distance_args(x, y, z, m, a[0], a[1], oc)]
    elif k == "angle": v = [O.angle_args(x, y, z, m, *a, oc)]
    elif k == "dihedral": v = [O.dihedral_args(x, y, z, m, *a, oc)]
    elif k == "com": v = O.arg_position(x, y, z, m, a[0], oc)
    elif k in ("dmin", "dmax"): v = [O.min_distance(x, y, z, a[0], a[1], oc)]
    elif k == "dpair": v = O.distance_pair_args(x, y, z, m, a[0], a[1], oc)
    elif k == "coord": v = case.frames[f][a[0]][np.asarray(a[1])]
    elif k == "plane": v = O.plane_frame(x, y, z, a[0], case.conn_off, case.conn_idx, oc)
    elif k == "rmsd":
        groups = a[0] if isinstance(a[0], list) else [a[0]]
        v = [O.rmsd_frame(x, y, z, case.frames[0], m, g, case.conn_off, case.conn_idx, oc) if len(g) else 0.0 for g in groups]
    elif k == "shape": v = np.concatenate([O.shape_weights(x, y, z, m if a[1] else None, g, oc) for g in a[0]])
    elif k == "ctx":
        op, local, firsts = a
        fn = {"distance": O.distance_args, "angle": O.angle_args, "dihedral": O.dihedral_args}[op]
        v = [fn(x, y, z, m, *[np.asarray(l[c], np.int32) if isinstance(l, list) else int(firsts[c]) + int(l) for l in local], oc) for c in range(len(firsts))]
    else: raise ValueError(k)
    return np.asarray(v, np.float32).ravel()


# ----------------------------------------------------------------------------------------------------------------------------- density
def density_params(cell):
    """k_density's constants from the initial cell, in float32 as the reference computes them (_internal_density): rc = A (0.5, 0.5, 0.5),
    re = diag(A), inv_ext = 1 / re (0 for re == 0), min_point = rc - re / 2"""
    f = np.float32; A = basis(cell).astype(np.float32); h = f(0.5)
    rc = np.array([(A[0, r] * h + A[1, r] * h) + A[2, r] * h for r in range(3)], np.float32)
    re = np.array([A[r, r] for r in range(3)], np.float32)
    inv = np.array([f(1) / e if e > 0 else f(0) for e in re], np.float32)
    return rc, re, inv, (rc - re * h).astype(np.float32)


def density_bins(coord, cell, axis):
    """the raw bin (before the clamp) and the clamped bin of every coordinate, k_density's float32 operations in order"""
    rc, re, inv, mn = (v[axis] for v in density_params(cell))
    x = np.asarray(coord, np.float32)
    with np.errstate(all="ignore"):
        if re != 0:
            d = (x - rc) * (np.float32(1) / re)
            x = rc + (d - np.rint(d)) * re                      # deperiodize1: rintf rounds a tie to even, as np.rint
        fc = ((x - mn) * inv) * np.float32(BINS)
        raw = np.trunc(fc.astype(np.float64))
    return raw, np.clip(raw, 0, BINS - 1).astype(np.int64)


def fixed_mass(mass):
    """round(mass * 2^24) as k_density accumulates it (the float product is exact)"""
    return np.rint(np.asarray(mass, np.float32).astype(np.float64) * 16777216.0).astype(np.uint64)


def density_counts(case, p, f):
    x, y, z = case.frames[f]
    idx = _pos_arg(p.args[1], x, y, z, O.UnitCell(*case.cells[f]))
    _, b = density_bins(case.frames[f][p.args[0]][idx], case.cells[0], p.args[0])
    out = np.zeros(BINS, np.uint64)
    np.add.at(out, b, fixed_mass(case.mass[idx]))
    return out, idx, b


def density_scale(cell):
    """the reference's normalisation of a bin: (float)(sum * (1660.5390666 / ((re0 * re1 * re2) / 1024)))"""
    _, re, _, _ = density_params(cell)
    slice_vol = np.float64(np.float32(np.float32(re[0] * re[1]) * re[2]) / np.float32(BINS))
    with np.errstate(divide="ignore"):
        return np.float64(1660.5390666) / slice_vol


def check_density_restatement(case, p, f):
    """the restatement's bins equal the oracle's (unit masses: the oracle counts atoms), and with integer masses the exact sums equal the
    oracle's float sums; -> the restated fixed-point counts of the frame"""
    counts, idx, b = density_counts(case, p, f)
    x, y, z = case.frames[f]
    ones, _ = O.density_frame(x, y, z, np.ones_like(case.mass), idx, O.UnitCell(*case.cells[0]), p.args[0])
    per_bin = np.bincount(b, minlength=BINS).astype(np.float64)
    with np.errstate(all="ignore"):
        want = (per_bin * density_scale(case.cells[0])).astype(np.float32)
    assert same(ones, want).all(), f"{case.name} {p.name} frame {f}: restated bins differ from the oracle's in {np.nonzero(~same(ones, want))[0][:8]}"
    m = case.mass[idx]
    if len(m) and (m == np.round(m)).all() and counts.max() < (1 << 48):
        got, _ = O.density_frame(x, y, z, case.mass, idx, O.UnitCell(*case.cells[0]), p.args[0])
        with np.errstate(all="ignore"):
            exact = ((counts.astype(np.float64) / 16777216.0).astype(np.float32).astype(np.float64) * density_scale(case.cells[0])).astype(np.float32)
        assert same(got, exact).all(), f"{case.name} {p.name} frame {f}: integer-mass sums differ from the oracle's"
    return counts


# ----------------------------------------------------------------------------------------------------------------------------- case table
class Case:
    def __init__(self, name, frames, cells, props, mass=None, bonds=(), require=None):
        self.name = name
        self.frames = np.ascontiguousarray(frames, np.float32)                                # [F, 3, N]
        F, _, N = self.frames.shape
        self.cells = cells if isinstance(cells, list) else [cells] * F
        self.props = props
        self.mass = np.full(N, 12.0, np.float32) if mass is None else np.asarray(mass, np.float32)
        self.conn_off, self.conn_idx = csr(N, bonds)
        self.require = require


CELLS3 = lambda L: [NO_CELL, ortho(L, L, L), tric(L, 0.5, -0.5, 0.45)]


def case_simd_split():
    N, L = 400, 21.0
    cells = CELLS3(L); rng = np.random.default_rng(101)
    fr = np.stack([in_cell(rng, N, c) for c in cells])
    mass = np.round(rng.uniform(1.0, 16.0, N), 3)
    sel = {n: (np.arange(n) * 3 + n) for n in SIMD_SIZES}
    props = []
    for j, n in enumerate(SIMD_SIZES):
        s = sel[n]
        props += [P(f"d{n}", "distance", s, 399), P(f"a{n}", "angle", 398, s, 397) if j % 2 else P(f"a{n}", "angle", s, 398, 397),
                  P(f"t{n}", "dihedral", *([396, 395, 394][:j % 4] + [s] + [396, 395, 394][j % 4:])[:4]), P(f"c{n}", "com", s)]

    def require():
        assert [c[6] for c in cells] == [0, ORTHO | PBC_ALL, TRICLINIC | PBC_ALL]
        assert min(SIMD_SIZES) < 8 and {n for n in SIMD_SIZES if n >= 8 and n % 8 == 0} and {n for n in SIMD_SIZES if n > 8 and n % 8}
        assert all(len(np.unique(sel[n])) == n and sel[n].max() < 394 for n in SIMD_SIZES)
    return Case("simd_split", fr, cells, props, mass=mass, require=require)


def case_masses():
    N, L = 300, 19.0
    cells = CELLS3(L); rng = np.random.default_rng(102)
    fr = np.stack([in_cell(rng, N, c) for c in cells])
    mass = np.full(N, 12.0, np.float32)
    zero, zero7, mixed, light, heavy = np.arange(0, 16), np.arange(16, 23), np.arange(30, 56), np.arange(60, 80), np.arange(80, 100)
    mass[zero] = 0.0; mass[zero7] = 0.0; mass[mixed[::2]] = 0.0
    mass[light] = rng.uniform(0.01, 0.99, len(light)).astype(np.float32)
    mass[heavy] = np.concatenate([[256.0, 257.0, 4096.0], rng.integers(256, 2000, len(heavy) - 3)])
    props = [P("c_zero", "com", zero), P("c_zero7", "com", zero7), P("c_mixed", "com", mixed), P("c_light", "com", light), P("c_heavy", "com", heavy),
             P("c_arr", "com", [zero, heavy]), P("d_zero", "distance", zero, 200), P("a_mix", "angle", mixed, 201, heavy),
             P("t_light", "dihedral", light, 202, 203, zero7), P("r_mixed", "rmsd", mixed), P("s_all", "shape", [zero, mixed, light, heavy], True),
             P("s_nomass", "shape", [zero, light], False), P("dx_all", "density", 0, np.arange(N)), P("dy_int", "density", 1, np.concatenate([zero, heavy, np.arange(150, 300)]))]

    def require():
        assert not mass[zero].any() and not mass[zero7].any() and len(zero) >= 8 > len(zero7)
        assert (mass[mixed] == 0).any() and (mass[mixed] > 0).any() and ((mass[light] > 0) & (mass[light] < 1)).all()
        assert (mass[heavy] >= 256).all() and (fixed_mass(mass[heavy]) >> np.uint64(32)).all()
    return Case("masses", fr, cells, props, mass=mass, require=require)


def case_nonperiodic():
    """frames 0-2: one axis non-periodic each (ORTHO flags); frame 3 fully periodic; 15 % of the atoms outside the box on each side"""
    N, Ls = 240, (17.0, 19.0, 23.0)
    rng = np.random.default_rng(103)
    cells = [ortho(*Ls, ORTHO | (PBC_ALL & ~(PBC_X << k))) for k in range(3)] + [ortho(*Ls)]
    fr = (rng.random((4, 3, N)) * 1.3 - 0.15) * np.asarray(Ls)[None, :, None]
    a, b = np.arange(0, 20), np.arange(20, 52)
    props = [P("d", "distance", 100, 101), P("d2", "distance", 102, 103), P("d_sel", "distance", a, b), P("a", "angle", 104, 105, 106),
             P("a_sel", "angle", a, 107, b), P("t", "dihedral", 108, 109, 110, 111), P("t_sel", "dihedral", a, 112, 113, b), P("c", "com", b),
             P("dmin", "dmin", a, b), P("dmax", "dmax", np.arange(60, 90), np.arange(120, 140)), P("dp", "dpair", np.arange(0, 12), np.arange(150, 170)),
             P("dx", "density", 0, np.arange(N)), P("dy", "density", 1, np.arange(N)), P("dz", "density", 2, np.arange(N))]

    def require():
        for k in range(3): assert not cells[k][6] & (PBC_X << k) and cells[k][6] & ORTHO
        out = (fr < 0) | (fr > np.asarray(Ls)[None, :, None])
        assert out[:, :, 100:112].any() and out.any(axis=2).all()
    return Case("nonperiodic", fr, cells, props, require=require)


def case_shear_npt():
    """a triclinic cell whose shear (up to L/2 on every off-diagonal) and box change every frame of one batch; 4-atom molecules with bonds"""
    F, n_mol = 4, 40
    cells = [tric(18.0 + 0.9 * f, 0.5 - 0.2 * f, -0.5 + 0.15 * f, 0.45 - 0.25 * f, 19.0 + 0.5 * f, 20.0 - 0.6 * f) for f in range(F)]
    rng = np.random.default_rng(104)
    t = np.array([[0, 0, 0], [1.5, 0, 0], [2.0, 1.4, 0], [3.4, 1.5, 0.6]])
    frac = rng.random((n_mol, 3)); frac[0] = (0.0, 0.0, 0.0)
    fr = []
    for f, c in enumerate(cells):
        A = basis(c); pts = np.concatenate([t + (frac[m] + 0.01 * f) @ A + rng.normal(scale=0.05, size=t.shape) for m in range(n_mol)])
        fr.append(pts.T)
    fr = np.stack(fr)
    bonds = [(4 * m + i, 4 * m + i + 1) for m in range(n_mol) for i in range(3)]
    a, b = np.arange(0, 16), np.arange(40, 64)
    props = [P("d", "distance", 0, 90), P("d_sel", "distance", a, b), P("a", "angle", 1, 2, 3), P("a_sel", "angle", a, 50, b),
             P("t", "dihedral", 0, 1, 2, 3), P("t2", "dihedral", 4, 5, 6, 7), P("t_sel", "dihedral", a, 81, 82, b), P("c", "com", b),
             P("c_arr", "com", [a, b, np.arange(100, 120)]), P("dmin", "dmin", a, b), P("dp", "dpair", np.arange(0, 10), np.arange(100, 113)),
             P("pl", "plane", np.arange(0, 4)), P("pl_sel", "plane", np.arange(0, 40)), P("r", "rmsd", np.arange(0, 40)),
             P("s", "shape", [np.arange(0, 4), np.arange(4, 8), np.arange(0, 40)], True), P("cx", "coord", 0, np.arange(0, 8)),
             P("dx", "density", 0, np.arange(4 * n_mol)), P("dy", "density", 1, np.arange(4 * n_mol)), P("dz", "density", 2, np.arange(4 * n_mol))]

    def require():
        assert len({c[1] for c in cells}) == F and len({c[0] for c in cells}) == F
        assert max(max(abs(c[1]), abs(c[2]), abs(c[4])) / c[0] for c in cells) == pytest.approx(0.5)
        assert all(c[6] == TRICLINIC | PBC_ALL for c in cells)
    return Case("shear_npt", fr, cells, props, bonds=bonds, require=require)


def far_geometry():
    """frame 0 orthorhombic, frame 1 triclinic; for every k in FAR and axis, a dihedral whose bond (k + axis) % 3 spans k box rows along
    the axis (alternating sign), the others 1.5 A; -> (frames, cells, [(k, axis, bond, atoms)])"""
    cells = [ortho(17.0, 19.0, 23.0), tric(20.0, 0.4, -0.3, 0.25)]
    rng = np.random.default_rng(105)
    combos = [(k, ax) for k in FAR for ax in range(3)]
    N = 4 * len(combos) + 40
    fr = np.empty((2, 3, N))
    base = rng.random((len(combos), 3)) * 10 + 3
    bonds = rng.normal(size=(len(combos), 3, 3)); bonds *= 1.5 / np.linalg.norm(bonds, axis=2, keepdims=True)
    meta = []
    for f, c in enumerate(cells):
        A = basis(c)
        for j, (k, ax) in enumerate(combos):
            p = [base[j]]; far = (k + ax) % 3; sign = 1 if j % 2 else -1
            for i in range(3): p.append(p[-1] + bonds[j, i] + (sign * k * A[ax] if i == far else 0.0))
            fr[f, :, 4 * j:4 * j + 4] = np.array(p).T
            if f == 0: meta.append((k, ax, far, np.arange(4 * j, 4 * j + 4)))
        fr[f, :, 4 * len(combos):] = in_cell(rng, 40, c)
    return fr, cells, meta


def case_far_images():
    fr, cells, meta = far_geometry()
    N = fr.shape[2]; n = 4 * len(meta)
    props = [P(f"t{k}_{ax}", "dihedral", *[int(i) for i in at]) for k, ax, _, at in meta]
    props += [P(f"d{k}_{ax}", "distance", int(at[far]), int(at[far + 1])) for k, ax, far, at in meta]
    props += [P("dp", "dpair", np.arange(0, n, 4), np.arange(n, N, 3)), P("dmin", "dmin", np.arange(0, n), np.arange(n, N)),
              P("dx", "density", 0, np.arange(N)), P("dy", "density", 1, np.arange(N)), P("dz", "density", 2, np.arange(N))]

    def require():
        for f, c in enumerate(cells):
            Ai = np.linalg.inv(basis(c)); spans = {}
            for k, ax, far, at in meta:
                d = (fr[f][:, at[far + 1]] - fr[f][:, at[far]]) @ Ai
                spans[(k, ax)] = abs(d[ax])
                assert abs(abs(d[ax]) - k) < 0.2, (f, k, ax, d)
            assert max(spans.values()) > 128 > 65 > 64   # past both caps of the old loop (64 subtractions, 128 steps in all)
        assert {k for k, _, _, _ in meta} == set(FAR) and {ax for _, ax, _, _ in meta} == {0, 1, 2} and cells[1][6] & TRICLINIC
    return Case("far_images", fr, cells, props, require=require)


def case_faces_ties():
    """x extent 16 (a power of two: rc +- ext/2 and the bin edges k * ext / 1024 are exact floats), y 18, z 20. Atoms on every cell face,
    at rc +- ext/2 + m ext (the deperiodisation's rintf ties: 0.5, 1.5, 2.5 round to even), on bin edges and one ulp either side, and
    pairs at exactly half a box (distance's tie) and on a 2 A lattice (equal minimum distances)"""
    Ls = (16.0, 18.0, 20.0); F = 2
    cells = [ortho(*Ls), ortho(*Ls)]
    rng = np.random.default_rng(106)
    pts = []
    for ax in range(3):   # on the faces 0 and L of each axis
        q = rng.random((12, 3)) * Ls; q[:6, ax] = 0.0; q[6:, ax] = Ls[ax]; pts.append(q)
    ties = np.array([8.0 + s * 8.0 + 16.0 * m for s in (-1, 1) for m in (-2, -1, 0, 1, 2)])
    q = rng.random((len(ties), 3)) * Ls; q[:, 0] = ties; pts.append(q)
    edges = [np.float32(k) * np.float32(16.0 / BINS) for k in (1, 2, 511, 512, 513, 1000, 1022, 1023)]
    ex = np.array([v for e in edges for v in (np.nextafter(e, np.float32(-1)), e, np.nextafter(e, np.float32(99)))], np.float32)
    q = rng.random((len(ex), 3)) * Ls; q[:, 0] = ex; pts.append(q)
    half = rng.integers(16, 32, (6, 3)) / 4.0; pts += [half, half + np.array([8.0, 0, 0]), half + np.array([0, 9.0, 0]), half + np.array([0, 0, -10.0])]
    lat = np.array([[i, j, k] for i in range(3) for j in range(3) for k in range(2)], float) * 2.0 + 3.0; pts.append(lat)
    P0 = np.concatenate(pts); N0 = len(P0)
    fr = np.stack([P0.T, (P0 + np.array([16.0, -18.0, 40.0])).T])   # frame 1: the same atoms one or two boxes away
    i_half = N0 - len(lat) - 24
    lat_i = np.arange(N0 - len(lat), N0)
    props = [P("d_face_x", "distance", 0, 6), P("d_face_y", "distance", 12, 18), P("d_face_z", "distance", 24, 30)]
    props += [P(f"d_half{a}", "distance", i_half + j, i_half + 6 * a + j) for a in (1, 2, 3) for j in (0, 3)]
    props += [P("dmin_lat", "dmin", lat_i[::2], lat_i[1::2]), P("dmax_lat", "dmax", lat_i[:9], lat_i[9:]), P("dp_lat", "dpair", lat_i[:6], lat_i[6:]),
              P("dmin_face", "dmin", np.arange(0, 18), np.arange(18, 36)), P("dx", "density", 0, np.arange(N0)), P("dy", "density", 1, np.arange(N0)),
              P("cx", "coord", 0, np.arange(0, 36))]

    def require():
        raw, b = density_bins(fr[0][0], cells[0], 0)
        assert (raw >= BINS).any() and (b == 0).any() and (b == BINS - 1).any()
        e0 = 36 + len(ties); eb = b[e0:e0 + len(ex)].reshape(-1, 3)
        ks = np.array([1, 2, 511, 512, 513, 1000, 1022, 1023])
        assert (eb[:, 1] == ks).all() and (eb[:, 2] == ks).all() and (eb[:, 0] <= ks).all()
        assert (eb[ks >= 256, 0] == ks[ks >= 256] - 1).all()   # the ulp below an edge lands in the bin below where x - rc is exact (x >= 4)
        d = (fr[0][0, 36:36 + len(ties)] - 8.0) / 16.0
        assert set(np.round(d, 6)) >= {-2.5, -1.5, -0.5, 0.5, 1.5, 2.5}
        assert (fr[0][0, :6] == 0).all() and (fr[0][0, 6:12] == 16.0).all()
        dl = [O.min_distance(*fr[0], lat_i[::2], lat_i[1::2], O.UnitCell(*cells[0]))]
        assert dl[0] == np.float32(2.0)
    return Case("faces_ties", fr, cells, props, require=require)


def collinear_angles(rng, want):
    """(a, b, c) float32 triples on one line whose normalised dot product rounds past +-1 (acosf -> NaN): `want` of each sign"""
    def dot(a, b, c):
        v = []
        for q in (a - b, c - b):
            l = np.sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]); v.append(q / l)
        return (v[0][0] * v[1][0] + v[0][1] * v[1][1]) + v[0][2] * v[1][2]
    got = {1: [], -1: []}
    while min(len(g) for g in got.values()) < want:
        p = (rng.random(3) * 10 + 2).astype(np.float32); u = rng.normal(size=3); u /= np.linalg.norm(u)
        t1, t2 = rng.uniform(1, 3, 2) * (1 if rng.random() < 0.5 else -1)
        b = (p + t1 * u).astype(np.float32); c = (p + t2 * u).astype(np.float32)
        dt = dot(p, b, c)
        s = 1 if dt > 1 else (-1 if dt < -1 else 0)
        if s and len(got[s]) < want: got[s].append(np.stack([p, b, c]))
    return got[1] + got[-1]


def case_degenerate():
    L, F = 20.0, 3
    cells = [NO_CELL, ortho(L, L, L), ortho(L, L, L)]
    rng = np.random.default_rng(107)
    base = rng.random((3, 200)) * L
    pts = list(base.T)
    def add(q):
        pts.extend(np.asarray(q)); return np.arange(len(pts) - len(q), len(pts))
    coin = add([[5, 5, 5], [5, 5, 5], [7, 5, 5], [7 + 4e-6, 5, 5], [5, 8, 5]])
    col = [add(t) for t in collinear_angles(rng, 3)]
    line = [add([[2, 3, 4], [2 + 1.5 * s1, 3, 4], [2 + 1.5 * (s1 + s2), 3, 4], [2 + 1.5 * (s1 + s2 + s3), 3, 4]]) for s1, s2, s3 in ((1, 1, 1), (1, -1, 1), (-1, 1, -1))]
    line.append(add([[4, 4, 4], [5.5, 5.5, 4], [7, 7, 4], [8.5, 8.5, 4]]))
    plan4 = add([[10, 10, 10], [11.6, 10, 10], [11.6, 11.6, 10], [10, 11.6, 10]])
    chain = add([[19.2, 5, 5], [0.6, 5.4, 5.2], [1.9, 6.2, 5.1], [3.3, 6.0, 5.6], [18.4, 4.1, 5.3]])   # across the face x = 0 / L
    one = add([[6, 6, 6]])
    P0 = np.array(pts).T; N = P0.shape[1]
    fr = np.stack([P0] * F)                                                  # the constructed atoms are the same in every frame
    fr[1][:, 0:200] += rng.normal(scale=0.3, size=(3, 200))                  # frame 2 is frame 0 again: rmsd of an identical structure
    fr[1][:, chain] += np.array([[0.05], [-0.03], [0.02]])
    bonds = [(chain[i], chain[i + 1]) for i in range(3)] + [(chain[0], chain[4])] + [(plan4[i], plan4[(i + 1) % 4]) for i in range(4)]
    props = [P("d_coin", "distance", int(coin[0]), int(coin[1])), P("a_coin", "angle", int(coin[0]), int(coin[1]), int(coin[4])),
             P("a_tiny", "angle", int(coin[2]), int(coin[3]), int(coin[4])), P("t_coin", "dihedral", *[int(i) for i in coin[:4]]),
             P("c_coin", "com", coin[:2])]
    props += [P(f"a_col{j}", "angle", *[int(i) for i in c]) for j, c in enumerate(col)]
    props += [P(f"t_line{j}", "dihedral", *[int(i) for i in l]) for j, l in enumerate(line)]
    props += [P("pl4", "plane", plan4), P("pl_line", "plane", line[0]), P("pl_chain", "plane", chain), P("s", "shape", [plan4, one, coin[:2], chain, coin[2:4]], True),
              P("r_same", "rmsd", np.arange(0, 200)), P("r_chain", "rmsd", chain), P("r_plan", "rmsd", plan4)]

    def require():
        assert (P0[:, coin[0]] == P0[:, coin[1]]).all() and 0 < np.linalg.norm(P0[:, coin[3]] - P0[:, coin[2]]) < 1e-5
        assert len(col) == 6
        for l in line:   # w = 0 exactly (the cross products of parallel, exactly representable bond vectors vanish)
            d = np.diff(fr[0][:, l].T.astype(np.float32), axis=0)
            assert not np.cross(np.cross(d[0], d[1]), np.cross(d[1], d[2])).any()
        assert np.ptp(fr[0][0, chain]) > L / 2 and (fr[2][:, 0:200] == fr[0][:, 0:200]).all()
    return Case("degenerate", fr, cells, props, bonds=bonds, require=require)


def case_arg_forms():
    N, L = 240, 20.0
    cells = CELLS3(L); rng = np.random.default_rng(108)
    fr = np.stack([in_cell(rng, N, c) for c in cells])
    S = 230                                                                  # the within() selection: one atom
    fr[:, :, S] = np.array([10.0, 10.0, 10.0])
    for f, c in enumerate(cells):   # frame 0: three atoms within 1.2 A of S; frames 1, 2: none within 2 A
        oc = O.UnitCell(*c)
        for _ in range(20):
            near = O.within(*fr[f].astype(np.float32), np.array([S]), 2.0, oc)
            if not len(near): break
            fr[f][:, near] = fr[f][:, near] + 4.0
        if f == 0: fr[0][:, 231:234] = np.array([10.0, 10.0, 10.0])[:, None] + np.array([[0.7, 0, 0], [0, -0.8, 0], [0, 0, 0.9]]).T
    w = Within(1.2, [S])
    s1, s2, s3 = np.arange(0, 5), np.arange(10, 30), np.arange(40, 49)
    firsts = np.arange(0, 96, 4)                                               # 24 contexts of 4 atoms
    ctx_sel = [np.arange(c, c + 4)[rng.random(4) < 0.5] for c in firsts]; ctx_sel[3] = ctx_sel[7] = np.zeros(0, np.int32)
    rmsd_groups = [np.arange(100 + 10 * g, 100 + 10 * g + (0 if g in (1, 4) else 3 + g)) for g in range(6)]
    props = [P("d_atoms", "distance", 50, 51), P("d_sel", "distance", s2, 52), P("d_arr", "distance", [s1, s2, s3], 53),
             P("a_arr", "angle", [s1, s3], 54, s2), P("t_arr", "dihedral", 55, [s1, s2], s3, 56), P("c_arr", "com", [s1, s2, s3]),
             P("c_arr2", "com", [s1, np.arange(60, 62)]), P("dc", "ctx", "distance", (0, 2), firsts), P("ac", "ctx", "angle", (0, 1, 2), firsts),
             P("tc", "ctx", "dihedral", (0, 1, 2, 3), firsts), P("dc_sel", "ctx", "distance", (ctx_sel, 1), firsts),
             P("tc_sel", "ctx", "dihedral", (0, ctx_sel, 2, 3), firsts), P("rc", "rmsd", rmsd_groups),
             P("d_dyn", "distance", w, 60), P("c_dyn", "com", w), P("a_dyn", "angle", w, 61, 62), P("dmin_dyn", "dmin", w, np.arange(100, 140)),
             P("dx_dyn", "density", 0, w)]

    def require():
        counts = [len(w.oracle(*fr[f].astype(np.float32), O.UnitCell(*cells[f]))) for f in range(3)]
        assert counts[0] == 3 and counts[1] == counts[2] == 0, counts
        assert any(len(g) == 0 for g in ctx_sel) and any(len(g) == 0 for g in rmsd_groups)
    return Case("arg_forms", fr, cells, props, require=require)


def case_pairs():
    N, L = 700, 24.0
    cells = [ortho(L, L, L), tric(L, 0.3, -0.2, 0.1)]
    rng = np.random.default_rng(109)
    fr = np.stack([in_cell(rng, N, c) for c in cells])
    lat = np.array([[i, j, k] for i in range(4) for j in range(4) for k in range(2)], float) * 2.5 + 1.0
    fr[:, :, 650:682] = lat.T
    fr[:, :, 699] = np.array([12.0, 12.0, 12.0])
    for f, c in enumerate(cells):
        near = O.within(*fr[f].astype(np.float32), np.array([699]), 1.0, O.UnitCell(*c)); fr[f][:, near] += 3.0
    empty = Within(0.5, [699])
    sizes = {"200": (np.arange(0, 10), np.arange(10, 30)), "256": (np.arange(30, 46), np.arange(46, 62)), "260": (np.arange(62, 82), np.arange(82, 95)),
             "75k": (np.arange(100, 400), np.arange(400, 650))}
    props = []
    for k, (a, b) in sizes.items():
        props += [P(f"dmin{k}", "dmin", a, b), P(f"dmax{k}", "dmax", b, a), P(f"dp{k}", "dpair", a, b)]
    props += [P("dmin_empty", "dmin", empty, np.arange(0, 50)), P("dmax_empty", "dmax", empty, np.arange(0, 50)),
              P("dmin_lat", "dmin", np.arange(650, 666), np.arange(666, 682)), P("dp_lat", "dpair", np.arange(650, 658), np.arange(658, 682)),
              P("dp_arr", "dpair", [np.arange(0, 5), np.arange(5, 12), np.arange(12, 14)], [np.arange(20, 23), np.arange(23, 40)]),
              P("dp_arr1", "dpair", np.arange(0, 6), [np.arange(20, 23), np.arange(23, 40), np.arange(40, 41)])]

    def require():
        n = {k: len(a) * len(b) for k, (a, b) in sizes.items()}
        assert n["200"] < 256 == n["256"] < n["260"] and n["75k"] > 1 << 16
        assert all(len(empty.oracle(*fr[f].astype(np.float32), O.UnitCell(*cells[f]))) == 0 for f in range(2))
        assert O.min_distance(*fr[0], np.arange(650, 666), np.arange(666, 682), O.UnitCell(*cells[0])) == np.float32(2.5)
    return Case("pairs", fr, cells, props, require=require)


HEAVY_BIN = (100, 140)   # 40 atoms of 16 u in one bin, all handled by CTA 0 (atom i goes to CTA (i // 256) % blocks)


def case_density_big():
    N, L = 5000, 30.0
    init = (L, 0.0, 0.0, L, 0.0, 0.0, ORTHO | PBC_X | PBC_Y)                  # z extent 0: inv_ext = 0, every atom in bin 0 of density_z
    cells = [init, ortho(L, L, L)]
    rng = np.random.default_rng(110)
    fr = rng.random((2, 3, N)) * L
    fr[:, 2] = fr[:, 2] * 3 - L                                                  # z spread over three boxes
    a, b = HEAVY_BIN
    fr[:, 0, a:b] = 7.05 + rng.random((2, b - a)) * 0.005                       # one x bin (30 / 1024 = 0.029 A wide)
    mass = rng.integers(1, 20, N).astype(np.float32)
    mass[a:b] = 16.0
    heavy = np.arange(3000, 3010); mass[heavy] = [256, 257, 300, 1000, 4096, 65536, 256, 512, 999, 2048]
    props = [P("dx", "density", 0, np.arange(N)), P("dy", "density", 1, np.arange(N)), P("dz", "density", 2, np.arange(N)),
             P("dx_heavy", "density", 0, np.concatenate([np.arange(a, b), heavy]))]

    def require():
        case = Case("x", fr, cells, [], mass=mass)
        blocks = min((N + 2047) // 2048, 64)
        assert N > 2048 and blocks == 3 and len({(i // 256) % blocks for i in range(a, b)}) == 1
        counts, _, bins = density_counts(case, props[0], 0)
        hb = bins[a:b]
        assert len(set(hb.tolist())) == 1 and counts[hb[0]] >= (1 << 32) and (b - a) * 16 * (1 << 24) >= 1 << 32
        assert not np.isin(bins[heavy], hb[0]).any()                          # the carry comes from the 16 u atoms alone
        assert (fixed_mass(mass[heavy]) >> np.uint64(32)).all()
        _, bz = density_bins(fr[0][2], init, 2)
        assert (bz == 0).all() and density_params(init)[2][2] == 0
    return Case("density_big", fr, cells, props, mass=mass, require=require)


def density_tric_geometry():
    init = tric(20.0, 0.5, -0.35, 0.4)
    rc, re, inv, mn = density_params(init)
    rng = np.random.default_rng(111)
    N0 = 600
    P0 = in_cell(rng, N0, init)
    extra = []
    for ax in range(3):
        step = np.float32(re[ax] / np.float32(BINS))
        for k in (0, 1, 300, 777, 1023, 1024):
            e = np.float32(mn[ax] + np.float32(k) * step)
            for v in (np.nextafter(e, np.float32(-1e9)), e, np.nextafter(e, np.float32(1e9))):
                q = rng.random(3) * 10; q[ax] = v; extra.append(q)
        for s in (-1, 1):
            for m in (-1, 0, 2):
                q = rng.random(3) * 10; q[ax] = rc[ax] + s * re[ax] * np.float32(0.5) + m * re[ax]; extra.append(q)
    Pt = np.concatenate([P0.T, np.array(extra)]).T
    frames = np.stack([Pt, Pt + rng.normal(scale=0.3, size=Pt.shape)])
    frames[1][:, N0:] = Pt[:, N0:]
    return frames, [init, tric(21.0, 0.45, -0.3, 0.35)]


def case_density_tric():
    fr, cells = density_tric_geometry()
    N = fr.shape[2]
    rng = np.random.default_rng(112)
    mass = np.round(rng.uniform(0.5, 40.0, N), 4).astype(np.float32)
    props = [P("dx", "density", 0, np.arange(N)), P("dy", "density", 1, np.arange(N)), P("dz", "density", 2, np.arange(N)),
             P("dz_dyn", "density", 2, Within(4.0, np.arange(0, 20)))]

    def require():
        rc, re, _, _ = density_params(cells[0])
        assert rc[0] != re[0] * np.float32(0.5) and rc[1] != re[1] * np.float32(0.5)   # the shear moves the centre
        for ax in range(3):
            raw, b = density_bins(fr[0][ax, 600:], cells[0], ax)
            assert (b == 0).any() and (b == BINS - 1).any() and (raw >= BINS).any()
        assert (mass != np.round(mass)).any()
        assert len(Within(4.0, np.arange(0, 20)).oracle(*fr[0].astype(np.float32), O.UnitCell(*cells[0]))) > 20
    return Case("density_tric", fr, cells, props, mass=mass, require=require)


CASES = [case_simd_split, case_masses, case_nonperiodic, case_shear_npt, case_far_images, case_faces_ties, case_degenerate, case_arg_forms,
         case_pairs, case_density_big, case_density_tric]
CASE_IDS = [c.__name__[5:] for c in CASES]
RUNS = ((1, 1), (1, 2), (0, 1), (0, 2))   # (batch_frames, num_streams) of the whole runs


# ----------------------------------------------------------------------------------------------------------------------------- evaluation
def same(a, b):
    """bit-equal float32 values; NaN equals NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def close(a, b):
    """the device bar for values through libm: 1e-5 (relative above 1), NaN equals NaN, +-pi equal"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    with np.errstate(invalid="ignore"):
        pi = (np.abs(np.abs(a) - np.pi) < TOL) & (np.abs(np.abs(b) - np.pi) < TOL)
        return (np.isnan(a) & np.isnan(b)) | pi | (np.abs(a - b) <= TOL * np.maximum(1.0, np.abs(b)))


def oracle_case(case):
    """per property: [F] arrays (temporal values) or [F] fixed-point count rows (density)"""
    F = case.frames.shape[0]
    return {p.name: [check_density_restatement(case, p, f) if p.kind == "density" else oracle_values(case, p, f) for f in range(F)] for p in case.props}


class Tally:
    def __init__(self): self.exact = self.bit_equal = self.total = 0


def compare(case, p, f, got, want, device, tally, tag):
    if p.kind == "density":
        if np.array_equal(got, want): return []
        d = np.nonzero(got != want)[0]
        return [f"{tag} frame {f} {p.name}: {len(d)} bins differ, first {d[:4].tolist()} got {got[d[:4]].tolist()} want {want[d[:4]].tolist()}"]
    if got.shape != want.shape: return [f"{tag} frame {f} {p.name}: {got.shape} values, oracle {want.shape}"]
    eq = same(got, want)
    strict = not device or p.exact(case.cells[f][6])
    if not strict:
        tally.total += len(eq); tally.bit_equal += int(eq.sum())
    ok = eq if strict else close(got, want)
    if ok.all(): return []
    i = np.nonzero(~ok)[0][:4]
    return [f"{tag} frame {f} {p.name} ({'bit-equal' if strict else 'within 1e-5'}): at {i.tolist()} got {got[i].tolist()} oracle {want[i].tolist()}"]


def _plan(case, **kw):
    import viamd_b200 as vb
    F, _, N = case.frames.shape
    plan = vb.Plan(vb.System(N, case.mass, conn_offset=case.conn_off, conn_idx=case.conn_idx), [p.prop() for p in case.props], F, **kw)
    plan.set_initial_frame(*case.frames[0], vb.UnitCell(*case.cells[0]))
    return plan


def read(plan, p, F):
    if p.kind == "density": return plan.counts(p.name)
    return plan.property_data(p.name).values.reshape(F, -1)


def cell_kind_runs(case):
    """[beg, end) runs of consecutive frames whose cells are all triclinic or all not"""
    tri = [bool(c[6] & TRICLINIC) for c in case.cells]
    cut = [0] + [f for f in range(1, len(tri)) if tri[f] != tri[f - 1]] + [len(tri)]
    return list(zip(cut[:-1], cut[1:]))


def check_case(case, device=False):
    import viamd_b200 as vb
    if case.require: case.require()
    want = oracle_case(case)
    F = case.frames.shape[0]
    tally = Tally(); bad = []
    plan = _plan(case, batch_frames=1)
    try:
        for f in range(F):
            plan.clear()
            plan.eval_host_frames(case.frames[f:f + 1], [vb.UnitCell(*case.cells[f])], f)
            plan.sync()
            for p in case.props:
                got = read(plan, p, F)
                bad += compare(case, p, f, got if p.kind == "density" else got[f], want[p.name][f], device, tally, "frame by frame")
    finally:
        plan.close()
    for bf, ns in RUNS:
        plan = _plan(case, batch_frames=bf, num_streams=ns)
        tag = f"batch_frames {bf} streams {ns}"
        try:
            for beg, end in cell_kind_runs(case):   # one batch holds either triclinic or other cells: one call per run of frames
                plan.eval_host_frames(case.frames[beg:end], [vb.UnitCell(*c) for c in case.cells[beg:end]], beg)
            plan.sync()
            assert plan.frame_mask().all()
            for p in case.props:
                got = read(plan, p, F)
                if p.kind == "density": bad += compare(case, p, 0, got, np.sum(want[p.name], axis=0, dtype=np.uint64), device, tally, tag)
                else:
                    for f in range(F): bad += compare(case, p, f, got[f], want[p.name][f], device, tally, tag)
        finally:
            plan.close()
    if device: print(f"{case.name}: {tally.bit_equal} of {tally.total} values through libm bit-equal to the oracle")
    assert not bad, f"{case.name}: {len(bad)} mismatches\n" + "\n".join(bad[:30])


@pytest.fixture
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "emul"))
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def check_nonterminating_loop():
    """inputs on which the reference's minimum-image loop never ends: the frame's dihedral is NaN, the others are unaffected"""
    import viamd_b200 as vb
    L = 20.0
    cells = [ortho(L, L, L)] * 3 + [tric(L, 0.3, -0.2, 0.1)] * 2
    base = np.array([[1.0, 2.0, 3.0], [2.5, 2.0, 3.0], [3.0, 3.4, 3.0], [4.2, 3.6, 4.0]]).T
    fr = np.stack([base] * len(cells)).astype(np.float32)
    fr[0][0, 1] = 3e9; fr[1][2, 3] = np.inf; fr[3][1, 2] = -3e9; fr[4][0, 3] = -np.inf   # x - box == x at 3e9 (ulp 256); frame 2: finite
    plan = vb.Plan(vb.System(4, np.ones(4, np.float32)), [vb.dihedral("t", 0, 1, 2, 3)], len(cells))
    try:
        plan.set_initial_frame(*fr[2], vb.UnitCell(*cells[2]))
        for beg, end in ((0, 3), (3, 5)): plan.eval_host_frames(fr[beg:end], [vb.UnitCell(*c) for c in cells[beg:end]], beg)
        plan.sync()
        t = plan.property_data("t").values
        assert np.isnan(t[[0, 1, 3, 4]]).all() and not np.isnan(t[2]), t
        assert close(t[2], O.dihedral(*fr[2], 0, 1, 2, 3, O.UnitCell(*cells[2])))
    finally:
        plan.close()


# ----------------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_under_emulation(emulated_library, make):
    check_case(make())


def test_dihedral_minimum_image_loop_stops_with_nan(emulated_library):
    check_nonterminating_loop()


def test_oracle_equals_the_reference_on_the_edge_geometries(golden_dir):
    """tests/golden/props_edges.npz: the unmodified reference's values of distance / angle / dihedral / com and density_x/_y/_z
    (make_golden_props_edges.py) on the far-image dihedrals, the per-axis non-periodic cells, the triclinic distance, the zero-mass centres,
    the SIMD split sizes, the collinear angles and dihedrals and the bin edges of a triclinic initial cell; the oracle gives every value"""
    import json
    g = np.load(os.path.join(golden_dir, "props_edges.npz"))
    names = sorted({k.split("/")[0] for k in g.files})
    checked = 0
    for name in names:
        frames, cells, flags, mass = g[f"{name}/frames"], g[f"{name}/cells"], g[f"{name}/flags"], g[f"{name}/mass"]
        for st in json.loads(str(g[f"{name}/stmts"])):
            sname, kind, args = st
            ref = g[f"{name}/{sname}"]
            for f in range(len(frames)):
                x, y, z = frames[f]; oc = O.UnitCell.from_params(*cells[f], flags[f])
                a = [np.arange(v[0], v[1], dtype=np.int32) if isinstance(v, list) else v for v in args]
                if kind == "distance": v = [O.distance_args(x, y, z, mass, *a, oc)]
                elif kind == "angle": v = [O.angle_args(x, y, z, mass, *a, oc)]
                elif kind == "dihedral": v = [O.dihedral_args(x, y, z, mass, *a, oc)]
                elif kind == "com": v = O.arg_position(x, y, z, mass, a[0], oc)
                else: v = O.density_frame(x, y, z, mass, a[1], O.UnitCell.from_params(*cells[0], flags[0]), a[0])[0]
                v = np.asarray(v, np.float32).ravel()
                assert same(v, ref[f]).all(), (name, sname, f, v[~same(v, ref[f])][:4], ref[f][~same(v, ref[f])][:4])
                checked += 1
    assert names == ["collinear", "density_tric", "far_images", "masses", "nonperiodic", "shear_npt", "simd_split"] and checked == 143, (names, checked)


@pytest.mark.gpu
@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_on_the_device(make):
    check_case(make(), device=True)


@pytest.mark.gpu
def test_dihedral_minimum_image_loop_stops_with_nan_on_the_device():
    check_nonterminating_loop()
