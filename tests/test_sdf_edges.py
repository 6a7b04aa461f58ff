"""sdf() against the plain-C oracle on adversarial structures and geometries.

An sdf runs three kernels per batch (sdf.cu): k_sdf_ref0 fits structure 0 of the initial frame (unwrapped along the bonds with the CURRENT
frame's cell), k_sdf_fit fits every structure of the frame and its cell range, and k_sdf_scatter walks the targets of the cells of
AABB(com, cutoff) on the grid with cell extent = cutoff (plan.cu), excludes the structure's own atoms and counts voxels. The case table
below drives the paths where these go wrong:
  exclusion    a contiguous run (one compare), non-contiguous rows that fit the 64-entry shared cache (SDF_EXCL_CACHE) and rows that reach
               the global tail loop, structures that are targets of one another, targets that are exactly the structures' union
  bond walk    unwrap_bonds walks the bonds of atoms 0 .. structure_size - 1 of the SYSTEM (the reference's local-index-as-atom quirk): a
               12-atom ring, a branched tree, two disconnected pieces (two BFS seeds), bonds to atoms at or beyond structure_size; each laid
               across a periodic face, in an orthorhombic and a triclinic cell
  fits         single atoms and atom pairs (degenerate covariances), planar structures (the sign-of-determinant branch of
               extract_rotation), a structure identical to structure 0, zero-mass atoms, and a massless structure 0 whose matrices are
               NaN: every hit then lands in voxel 0 on both sides (x86 (int)NaN is INT_MIN, clamped to 0; CUDA __float2int_rz(NaN) is 0)
  cells        each axis non-periodic in turn, frames without a cell, a structure whose centre lies outside the targets' bounding box on a
               non-periodic axis (the clamped or empty range of k_sdf_fit), a triclinic shear and a cubic box that change every frame
               inside one batch (so the initial frame is unwrapped with a different cell each frame)
  scatter      targets exactly on the faces com +- cutoff of the box test and on voxel faces (the clamp to voxel 127), one cell with more than
               200 targets (a half-warp runs many rounds), empty cells between full ones, a cutoff past half the box
  plumbing     compact host ingest of a sparse system against whole frames, a within() target, two devices against one

Every case is compared with oracle_lib.sdf_frame exactly, in two ways: frame by frame (plan.clear(), one frame, every voxel and the
frame's hit total), and as whole runs at batch_frames 1 and the default with one and two stream slots. Each case's `require` asserts that
it reaches the path it names: the geometry through mdgpu_debug_frame_geom at the sdf grid, the rest from the rows.

With cell extent = cutoff a structure's cell range spans at most ceil(2 * cutoff * cells / extent) + 1 cells per axis, a few cells, so
the SDF_MAXSEG (128-cell) chunk loop of k_sdf_scatter runs once: test_cell_ranges_stay_below_one_chunk bounds what the table reaches.

Geometries on which the reference itself faults have no defined answer and are left out (see make_golden_sdf_edges.py). Frames without a
cell stay under 1 000 atoms for that reason. tests/golden/sdf_edges.npz pins the oracle to the unmodified reference on the ring, tree,
non-periodic, cell-less, changing-cell and large-cutoff geometries.

The table runs on the CPU emulation of the library (tests/emul) and, with -m gpu, on the device.
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
VOL = 128 ** 3
EXCL_CACHE = 64     # SDF_EXCL_CACHE of sdf.cu
MAXSEG = 128        # SDF_MAXSEG of sdf.cu


def ortho(x, y, z, flags=ORTHO | PBC_ALL):
    return (float(x), 0.0, 0.0, float(y), 0.0, float(z), flags)


def csr(N, bonds):
    """undirected bond list -> (conn_offset [N + 1], conn_idx), neighbours ascending"""
    nb = [[] for _ in range(N)]
    for a, b in bonds: nb[a].append(b); nb[b].append(a)
    off = np.zeros(N + 1, np.uint32); off[1:] = np.cumsum([len(n) for n in nb])
    idx = np.array([j for n in nb for j in sorted(n)], np.int32)
    return off, (idx if len(idx) else np.zeros(1, np.int32))


def is_contiguous(row):
    return int(row[-1]) - int(row[0]) + 1 == len(row)


# ----------------------------------------------------------------------------------------------------------------------------- properties
class Sdf:
    """sdf(structures, targets, cutoff); targets: an index array or a Within"""
    def __init__(self, name, structs, trg, cutoff):
        self.name, self.structs, self.trg, self.cutoff = name, np.ascontiguousarray(structs, np.int32), trg, float(cutoff)
        assert self.structs.ndim == 2

    def prop(self):
        import viamd_b200 as vb
        return vb.sdf(self.name, self.structs, self.trg.vb() if isinstance(self.trg, Within) else np.asarray(self.trg, np.int32), self.cutoff)

    def targets(self, x, y, z, cell):
        return self.trg.oracle(x, y, z, cell) if isinstance(self.trg, Within) else np.asarray(self.trg, np.int32)


class Within:
    def __init__(self, radius, sel):
        self.radius, self.sel = float(radius), np.asarray(sel, np.int32)

    def vb(self):
        import viamd_b200 as vb
        return vb.Within(self.radius, self.sel)

    def oracle(self, x, y, z, cell):
        return O.within(x, y, z, self.sel, self.radius, cell)


# ----------------------------------------------------------------------------------------------------------------------------- case table
class Case:
    def __init__(self, name, frames, cells, props, mass=None, bonds=(), require=None, runs=((1, 1), (1, 2), (0, 1))):
        self.name = name
        self.frames = np.ascontiguousarray(frames, np.float32)                                # [F, 3, N]
        F, _, N = self.frames.shape
        self.cells = cells if isinstance(cells, list) else [cells] * F                       # per frame (x, xy, xz, y, yz, z, flags)
        self.props = props
        self.mass = np.ones(N, np.float32) if mass is None else np.asarray(mass, np.float32)
        self.conn_off, self.conn_idx = csr(N, bonds)
        self.require = require                                                                # require(geom): asserts the path
        self.runs = runs                                                                      # (batch_frames, num_streams) of the whole runs


def rotations(rng, n):
    """n random proper rotations (QR of Gaussian matrices)"""
    out = []
    for _ in range(n):
        q, r = np.linalg.qr(rng.normal(size=(3, 3)))
        q = q * np.sign(np.diag(r)); out.append(q if np.linalg.det(q) > 0 else -q)
    return out


def wrap(p, cell):
    """[3, N] cartesian -> the same points wrapped into the cell on its periodic axes"""
    x, xy, xz, y, yz, z, flags = cell
    A = np.array([[x, 0, 0], [xy, y, 0], [xz, yz, z]], np.float64)
    s = p.T @ np.linalg.inv(A)
    for k in range(3):
        if flags & (PBC_X << k): s[:, k] -= np.floor(s[:, k])
    return (s @ A).T


def molecules(seed, template, n_mol, n_solvent, cells, jitter=0.05, straddle=True):
    """n_mol copies of `template` ([n, 3], whole) at random positions and orientations, then n_solvent single atoms, wrapped into each
    frame's cell. Molecule 0 (and 1) sit on the corner of the cell, across its periodic faces, so the bond walk has to make them whole."""
    rng = np.random.default_rng(seed)
    n = len(template); t = template - template.mean(axis=0)
    F = len(cells); N = n_mol * n + n_solvent
    fr = np.empty((F, 3, N))
    cen0 = rng.random((n_mol, 3)); rot = rotations(rng, n_mol); sol = rng.random((3, n_solvent))
    for f, cell in enumerate(cells):
        x, xy, xz, y, yz, z, _ = cell
        A = np.array([[x, 0, 0], [xy, y, 0], [xz, yz, z]], np.float64)
        cen = (cen0 + 0.02 * f) % 1.0
        if straddle: cen[0] = (0.0, 0.0, 0.0); cen[min(1, n_mol - 1)] = (1.0, 0.5, 0.0)
        pts = [(t @ R.T + c @ A + rng.normal(scale=jitter, size=t.shape)) for c, R in zip(cen, rot)]
        fr[f, :, :n_mol * n] = np.concatenate(pts).T
        fr[f, :, n_mol * n:] = (sol.T @ A).T
        fr[f] = wrap(fr[f], cell)
    return fr


def ring(n=12, bond=1.4):
    a = 2 * np.pi * np.arange(n) / n; R = bond / (2 * np.sin(np.pi / n))
    return np.stack([R * np.cos(a), R * np.sin(a), 0.3 * (-1.0) ** np.arange(n)], axis=1), [(i, (i + 1) % n) for i in range(n)]


def tree():
    """10 atoms, 1.5 A bonds: 0-1, 1-2, 1-3, 3-4, 3-5, 0-6, 6-7, 6-8, 8-9"""
    bonds = [(0, 1), (1, 2), (1, 3), (3, 4), (3, 5), (0, 6), (6, 7), (6, 8), (8, 9)]
    d = {1: (1.5, 0, 0), 2: (0.5, 1.41, 0), 3: (0.5, -0.71, 1.22), 4: (1.5, 0, 0), 5: (-0.5, -1.41, 0), 6: (-1.5, 0, 0),
         7: (-0.5, 1.41, 0), 8: (-0.5, -0.71, -1.22), 9: (-1.5, 0, 0)}   # atoms that share no bond stay 2.4 A apart or more
    p = np.zeros((10, 3))
    for a, b in bonds: p[b] = p[a] + np.asarray(d[b])
    return p, bonds


def split_pieces():
    """8 atoms in two chains 0-1-2-3 and 4-5-6-7 with no bond between them (two BFS seeds)"""
    p = np.array([[0, 0, 0], [1.5, 0, 0], [3, 0.3, 0], [4.5, 0, 0.2], [0, 3, 0], [1.5, 3.2, 0], [3, 3, 0.4], [4.5, 3.1, 0]], float)
    return p, [(0, 1), (1, 2), (2, 3), (4, 5), (5, 6), (6, 7)]


def tile_bonds(bonds, n, n_mol):
    return [(a + m * n, b + m * n) for m in range(n_mol) for a, b in bonds]


def frames_triclinic(seed, N, L, F, shear=True):
    cells = [(L, (0.21 + 0.04 * f * shear) * L, -0.13 * L, L, 0.17 * L, L, TRICLINIC | PBC_ALL) for f in range(F)]
    rng = np.random.default_rng(seed)
    return np.stack([wrap((rng.random((3, N)).T * L).T, c) for c in cells]), cells


# --- exclusion
def case_exclusion():
    N, L, F = 700, 24.0, 2
    rng = np.random.default_rng(11)
    fr = rng.random((F, 3, N)) * L
    allv = np.arange(N)
    contig = np.arange(90).reshape(30, 3)
    nc = {k: np.stack([np.arange(b, b + 2 * k, 2) for b in (300, 301)]) for k in (30, 64, 65, 100)}
    nc[2] = np.stack([[k, k + 350] for k in range(0, 40, 2)])
    mutual = np.stack([np.arange(b, b + 60, 3) for b in range(0, 30)])   # 30 rows of 20 atoms, each row's atoms targets of the others
    union = np.unique(mutual)
    props = [Sdf("contig", contig, allv, 5.0)] + [Sdf(f"nc{k}", v, allv, 5.0) for k, v in sorted(nc.items())]
    props += [Sdf("mutual", mutual, union[::2], 4.0), Sdf("union", mutual, union, 4.0), Sdf("nc100u", nc[100], np.unique(nc[100]), 6.0)]

    def require(geom):
        assert all(is_contiguous(r) for r in contig)
        for k, v in nc.items():
            assert v.shape[1] == k and not any(is_contiguous(r) for r in v)
        assert max(k for k in nc if k <= EXCL_CACHE) == EXCL_CACHE and min(k for k in nc if k > EXCL_CACHE) == EXCL_CACHE + 1
        assert len(np.intersect1d(mutual[0], union[::2])) > 0
        assert all(geom(f, 5.0)[12] == 1 for f in range(F))
    return Case("exclusion", fr, ortho(L, L, L), props, require=require)


# --- bond walk
def _topology_case(name, template, tbonds, extra_bonds, tric, seed, n_mol=16, cutoff=6.0):
    L, F = 26.0, 3
    cells = frames_triclinic(0, 1, L, F)[1] if tric else [ortho(L, L, L)] * F
    n = len(template)
    fr = molecules(seed, template, n_mol, 500, cells)
    bonds = tile_bonds(tbonds, n, n_mol) + list(extra_bonds)
    structs = np.arange(n_mol * n).reshape(n_mol, n)
    N = fr.shape[2]
    props = [Sdf("all", structs, np.arange(N), cutoff), Sdf("solv", structs[::2], np.arange(n_mol * n, N), cutoff - 1.5)]

    def require(geom):
        assert all(geom(f, cutoff)[12] == 1 for f in range(F))
        assert all(bool(c[6] & TRICLINIC) == tric for c in cells)
        for f in range(F):   # molecule 0 is split across a periodic face in every frame: its raw extent spans most of the box
            assert np.ptp(fr[f, 0, :n]) > L / 2 or np.ptp(fr[f, 1, :n]) > L / 2 or np.ptp(fr[f, 2, :n]) > L / 2
    return Case(name, fr, cells, props, bonds=bonds, require=require)


def case_ring_ortho():
    t, b = ring(); return _topology_case("ring_ortho", t, b, (), False, 21)


def case_ring_triclinic():
    t, b = ring(); return _topology_case("ring_triclinic", t, b, (), True, 22)


def case_tree_ortho():
    t, b = tree(); return _topology_case("tree_ortho", t, b, (), False, 23)


def case_tree_triclinic():
    t, b = tree(); return _topology_case("tree_triclinic", t, b, (), True, 24)


def case_pieces_beyond():
    """two disconnected chains per structure, and bonds from molecule 0 to atom 8 (= structure_size) and 13 (beyond): the walk drops them"""
    t, b = split_pieces(); return _topology_case("pieces_beyond", t, b, [(3, 8), (7, 13)], False, 25)


def case_pieces_triclinic():
    t, b = split_pieces(); return _topology_case("pieces_triclinic", t, b, [(3, 8), (7, 13)], True, 26)


# --- degenerate fits
def case_fits():
    N, L, F = 600, 22.0, 3
    rng = np.random.default_rng(31)
    fr = rng.random((F, 3, N)) * L
    # atoms 0-3 of every 4 at 100..299 form a planar square (side 1.6) at a random place and orientation
    sq = np.array([[0, 0, 0], [1.6, 0, 0], [1.6, 1.6, 0], [0, 1.6, 0]], float)
    rot = rotations(rng, 50)
    for f in range(F):
        for m in range(50):
            fr[f, :, 100 + 4 * m: 104 + 4 * m] = (sq @ rot[(m + f) % 50].T + rng.random(3) * L).T
    mass = np.ones(N, np.float32)
    mass[300:400:3] = 0.0                                        # zero-mass atoms inside the "zmass" structures
    mass[500:503] = 0.0                                          # a massless structure 0 for "massless0"
    allv = np.arange(N)
    single = np.arange(0, 60, 3)[:, None]
    pairs = np.stack([np.arange(0, 80, 2), np.arange(1, 80, 2)], axis=1)
    planar = np.arange(100, 300).reshape(50, 4)
    same0 = np.concatenate([planar[:1], planar[:1], planar[1:20]])
    zmass = np.arange(300, 400).reshape(25, 4)
    massless0 = np.concatenate([np.arange(500, 503)[None], np.arange(510, 570).reshape(20, 3)])
    props = [Sdf("single", single, allv, 5.0), Sdf("pairs", pairs, allv, 5.0), Sdf("planar", planar, allv, 6.0), Sdf("same0", same0, allv, 6.0),
             Sdf("zmass", zmass, allv, 5.0), Sdf("massless0", massless0, allv, 5.0)]

    def require(geom):
        assert all(geom(f, 6.0)[12] == 1 for f in range(F))
        p = fr[:, :, planar[0]]
        for f in range(F):   # planar: the four points span a plane (smallest singular value ~0)
            s = np.linalg.svd((p[f] - p[f].mean(axis=1, keepdims=True)).T, compute_uv=False)
            assert s[2] < 1e-3 * s[0]
        assert (mass[zmass] == 0).any(axis=1).all() and (mass[zmass] > 0).any(axis=1).all()
        assert not mass[massless0[0]].any() and mass[massless0[1:]].all()
    return Case("fits", fr, ortho(L, L, L), props, mass=mass, require=require)


# --- cells
def case_nonperiodic():
    """frames 0-2: one axis non-periodic each; frame 3: no cell; 15 % of the atoms outside the box on each side"""
    N, L, F = 800, (24.0, 27.0, 21.0), 4
    rng = np.random.default_rng(41)
    fr = (rng.random((F, 3, N)) * 1.3 - 0.15) * np.asarray(L)[None, :, None]
    cells = [ortho(*L, ORTHO | (PBC_ALL & ~(PBC_X << k))) for k in range(3)] + [NO_CELL]
    res = np.arange(300).reshape(100, 3)
    props = [Sdf("res", res, np.arange(N), 5.0), Sdf("res7", res[::3], np.arange(0, N, 2), 7.0)]

    def require(geom):
        for f in range(3): assert not (cells[f][6] & (PBC_X << f)) and geom(f, 5.0)[12] == 1
        assert cells[3][6] == 0 and geom(3, 5.0)[12] == 1 and N < 1000
    return Case("nonperiodic", fr, cells, props, require=require)


def case_outside_aabb():
    """z non-periodic: targets in a slab z in [8, 14]; structures above it (z 14.5 .. 30: partly in reach), far above (z ~ 40) and below
    (z ~ -9): their cell ranges on z are clamped to the grid or empty"""
    N, L, F = 700, 24.0, 3
    rng = np.random.default_rng(42)
    fr = rng.random((F, 3, N)) * L
    fr[:, 2, 300:] = 8.0 + rng.random((F, N - 300)) * 6.0
    fr[:, 2, 0:90] = 14.5 + rng.random((F, 90)) * 15.0
    fr[:, 2, 90:150] = 40.0 + rng.random((F, 60))
    fr[:, 2, 150:210] = -9.0 - rng.random((F, 60))
    cells = [ortho(L, L, L, ORTHO | PBC_X | PBC_Y)] * F
    props = [Sdf("above", np.arange(90).reshape(30, 3), np.arange(300, N), 4.0), Sdf("far", np.arange(90, 210).reshape(40, 3), np.arange(300, N), 4.0),
             Sdf("mixed", np.arange(0, 210).reshape(70, 3), np.arange(300, N), 4.0)]

    def require(geom):
        for f in range(F):
            zmax = fr[f, 2, 300:].max()
            assert (fr[f, 2, 90:150] > zmax + 4.0).all() and (fr[f, 2, 150:210] < -4.0).all() and geom(f, 4.0)[12] == 1
    return Case("outside_aabb", fr, cells, props, require=require)


def case_shear():
    """a triclinic shear that changes every frame of one batch; 3-atom residues, bonded, split across faces"""
    L, F = 25.0, 4
    cells = frames_triclinic(0, 1, L, F)[1]
    t = np.array([[0, 0, 0], [0.96, 0, 0], [-0.24, 0.93, 0]])
    n_mol = 120
    fr = molecules(43, t, n_mol, 300, cells)
    N = fr.shape[2]
    props = [Sdf("w", np.arange(3 * n_mol).reshape(n_mol, 3), np.arange(0, N), 5.0), Sdf("w2", np.arange(90).reshape(30, 3), np.arange(3 * n_mol, N), 7.0)]

    def require(geom):
        assert len({c[1] for c in cells}) == F and all(geom(f, 5.0)[12] == 1 for f in range(F))
    return Case("shear", fr, cells, props, bonds=tile_bonds([(0, 1), (0, 2)], 3, n_mol), require=require)


def case_npt():
    """a cubic box of 22.0, 20.4, 23.6, 21.2 A inside one batch: k_sdf_ref0 unwraps the initial frame with each frame's own box"""
    boxes = [22.0, 20.4, 23.6, 21.2]
    t = np.array([[0, 0, 0], [0.96, 0, 0], [-0.24, 0.93, 0]])
    n_mol = 150
    base = molecules(44, t, n_mol, 200, [ortho(22.0, 22.0, 22.0)] * 4)
    fr = np.stack([wrap(base[f] * (b / 22.0), ortho(b, b, b)) for f, b in enumerate(boxes)])
    N = fr.shape[2]
    props = [Sdf("w", np.arange(3 * n_mol).reshape(n_mol, 3), np.arange(N), 5.0), Sdf("w8", np.arange(60).reshape(20, 3), np.arange(0, N, 3), 8.0)]

    def require(geom):
        assert len(set(boxes)) == 4 and all(geom(f, 5.0)[12] == 1 for f in range(4))
        x0 = fr[0, :, :3]
        assert np.ptp(x0, axis=1).max() > 11.0   # molecule 0 of the initial frame is split, so the unwrap's cell matters
    return Case("npt", fr, [ortho(b, b, b) for b in boxes], props, bonds=tile_bonds([(0, 1), (0, 2)], 3, n_mol), require=require)


# --- scatter
def case_faces():
    """tetrahedra centred exactly on lattice points (their centre of mass is exact); targets at com +- cutoff on every axis and corner (the
    <= / >= of the box test; voxel 128 clamps to 127), on voxel faces (multiples of 2 cutoff / 128 from the centre) and just inside"""
    L, r, F = 24.0, 4.0, 2
    tet = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], float) * 0.75
    cen = np.array([[6.0, 6.0, 6.0], [12.0, 18.0, 6.0], [18.0, 12.0, 18.0], [0.0, 12.0, 12.0]])
    pts = [c + tet for c in cen]
    vox = 2 * r / 128
    offs = [np.array(o, float) * r for o in np.ndindex(3, 3, 3)]
    offs = [o - r for o in offs]
    for c in cen:
        pts.append(c + np.array(offs))
        pts.append(c + np.array([[k * vox, (k % 7) * vox, -(k % 5) * vox] for k in range(-64, 65, 4)]))
        pts.append(c + np.array([[np.nextafter(np.float32(r), np.float32(0)), 0, 0], [0, -np.nextafter(np.float32(r), np.float32(0)), 0]]))
    P = np.concatenate(pts)
    N = len(P)
    fr = np.stack([P.T, P.T])
    structs = np.arange(16).reshape(4, 4)
    props = [Sdf("faces", structs, np.arange(16, N), r), Sdf("faces_all", structs, np.arange(N), r)]

    def require(geom):
        c0 = fr[0][:, structs[0]].astype(np.float32).astype(np.float64).mean(axis=1)
        assert np.array_equal(c0, cen[0]) and geom(0, r)[12] == 1
        assert ((fr[0].T[16:] - cen[0]) == r).any()
    return Case("faces", fr % L, ortho(L, L, L), props, require=require)


def case_crowded():
    """one cell with 300 targets (a half-warp runs ten rounds), cells alternately empty and full (targets only in slabs x in [0, 5) and
    [10, 15) of a 5 A grid), and 3-atom structures among them"""
    L, F, r = 20.0, 2, 5.0
    rng = np.random.default_rng(51)
    N = 900
    fr = np.empty((F, 3, N))
    fr[:, :, :300] = 11.0 + rng.random((F, 3, 300)) * 3.0
    fr[:, 0, 300:] = rng.random((F, N - 300)) * 5.0 + 10.0 * rng.integers(0, 2, (F, N - 300))
    fr[:, 1:, 300:] = rng.random((F, 2, N - 300)) * L
    props = [Sdf("crowd", np.arange(300, 420).reshape(40, 3), np.arange(N), r), Sdf("slabs", np.arange(420, 600).reshape(60, 3), np.arange(300, N), r)]

    def require(geom):
        g = geom(0, r)
        assert tuple(g[:3]) == (4, 4, 4)
        cell = (fr[0, :, :300] // 5.0).astype(int)
        assert (cell == 2).all()   # all 300 in cell (2, 2, 2)
        assert not ((fr[:, 0, 300:] % 10.0) >= 5.0).any()
    return Case("crowded", fr, ortho(L, L, L), props, require=require)


def case_large_cutoff():
    """cutoff 8 and 9.5 in a 14.4 A box (past half of it): a one-cell grid, images on both sides of every axis"""
    L, F = 14.4, 2
    t = np.array([[0, 0, 0], [0.96, 0, 0], [-0.24, 0.93, 0]])
    fr = molecules(52, t, 40, 200, [ortho(L, L, L)] * F)
    N = fr.shape[2]
    props = [Sdf("c8", np.arange(120).reshape(40, 3), np.arange(N), 8.0), Sdf("c95", np.arange(60).reshape(20, 3), np.arange(N), 9.5)]

    def require(geom):
        assert tuple(geom(0, 8.0)[:3]) == (1, 1, 1) and 2 * 8.0 > L
    return Case("large_cutoff", fr, ortho(L, L, L), props, bonds=tile_bonds([(0, 1), (0, 2)], 3, 40), require=require)


# --- plumbing
def case_within_target():
    N, L, F = 600, 22.0, 3
    fr = np.random.default_rng(61).random((F, 3, N)) * L
    props = [Sdf("w", np.arange(60).reshape(20, 3), Within(6.0, np.arange(60, 66)), 5.0)]

    def require(geom):
        assert all(len(Within(6.0, np.arange(60, 66)).oracle(*fr[f].astype(np.float32), O.UnitCell(*ortho(L, L, L)))) > 10 for f in range(F))
    return Case("within_target", fr, ortho(L, L, L), props, require=require)


CASES = [case_exclusion, case_ring_ortho, case_ring_triclinic, case_tree_ortho, case_tree_triclinic, case_pieces_beyond, case_pieces_triclinic,
         case_fits, case_nonperiodic, case_outside_aabb, case_shear, case_npt, case_faces, case_crowded, case_large_cutoff, case_within_target]
CASE_IDS = [c.__name__[5:] for c in CASES]


# ----------------------------------------------------------------------------------------------------------------------------- evaluation
def oracle_frames(case):
    """per property: [(voxel indices, counts, hit total)] per frame"""
    out = {p.name: [] for p in case.props}
    for f in range(case.frames.shape[0]):
        x, y, z = case.frames[f]; oc = O.UnitCell(*case.cells[f])
        for p in case.props:
            vol, total = O.sdf_frame(x, y, z, case.frames[0], case.mass, p.structs, p.targets(x, y, z, oc), case.conn_off, case.conn_idx, oc, p.cutoff)
            nz = np.nonzero(vol)[0]
            out[p.name].append((nz, vol[nz].astype(np.uint64), total))
    return out


def dense(sparse_rows):
    v = np.zeros(VOL, np.uint64)
    for nz, c, _ in sparse_rows: v[nz] += c
    return v


def target_aabb(case, p, f):
    x, y, z = case.frames[f]; t = p.targets(x, y, z, O.UnitCell(*case.cells[f]))
    pts = case.frames[f][:, t]
    return np.concatenate([np.minimum(pts.min(axis=1), 0.0), np.maximum(pts.max(axis=1), 0.0)]).astype(np.float32)


def frame_geom_of(case):
    """geom(frame, cutoff) -> mdgpu_debug_frame_geom at the sdf grid of that frame: cell extent = cutoff (plan.cu), grid fitted on
    non-periodic axes to the bounding box of the targets (of the first property with that cutoff) and the origin, as k_aabb builds it"""
    import ctypes as C
    import viamd_b200 as vb
    from viamd_b200 import api
    L = api.lib(); L.mdgpu_debug_frame_geom.argtypes = [C.POINTER(vb.UnitCell), C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]

    def geom(f, r, box=None):
        r = float(np.float32(r)); cell = vb.UnitCell(*case.cells[f])
        if box is None:
            p = next((p for p in case.props if p.cutoff == r), case.props[0])
            box = target_aabb(case, p, f)
        gi = np.zeros(13, np.int32); gf = np.zeros(7, np.float32)
        assert L.mdgpu_debug_frame_geom(C.byref(cell), r, r, box.ctypes.data, gi.ctypes.data, gf.ctypes.data) == 0
        return gi
    return geom


def cell_range_bound(case, geom, p, f):
    """an upper bound of the cells k_sdf_fit's range of any structure of p spans in frame f: per axis ceil(fractional extent of the box
    com +- cutoff * cells) + 1, at most the grid on a non-periodic axis"""
    box = target_aabb(case, p, f)
    cd = geom(f, p.cutoff, box)[:3]
    x, xy, xz, y, yz, z, flags = case.cells[f]
    A = np.array([[x, 0, 0], [xy, y, 0], [xz, yz, z]], np.float64)
    ce = max(p.cutoff, 3.0)
    for k in range(3):
        if (flags & PBC_ALL) != PBC_ALL and not flags & (PBC_X << k):
            ext = np.float32(np.ceil((box[3 + k] - box[k]) / np.float32(ce)) * np.float32(ce))
            A[k] = 0.0; A[k, k] = ext if ext > 0 else 1.0
    Iv = np.linalg.inv(A)
    n = 1
    for k in range(3):
        b = int(np.ceil(2 * p.cutoff * np.abs(Iv[:, k]).sum() * cd[k])) + 1
        if not flags & (PBC_X << k): b = min(b, int(cd[k]))
        n *= b
    return n


def _plan(case, **kw):
    import viamd_b200 as vb
    F, _, N = case.frames.shape
    plan = vb.Plan(vb.System(N, case.mass, conn_offset=case.conn_off, conn_idx=case.conn_idx), [p.prop() for p in case.props], F, **kw)
    plan.set_initial_frame(*case.frames[0], vb.UnitCell(*case.cells[0]))
    return plan


def run_whole(case, **kw):
    """-> ({name: counts uint64}, {name: [frame totals]})"""
    import viamd_b200 as vb
    F = case.frames.shape[0]
    plan = _plan(case, **kw)
    try:
        plan.eval_host_frames(case.frames, [vb.UnitCell(*c) for c in case.cells], 0)
        plan.sync()
        assert plan.frame_mask().all()
        return ({p.name: plan.counts(p.name) for p in case.props},
                {p.name: [plan.frame_counts(p.name, f, want_bins=False)[1] for f in range(F)] for p in case.props})
    finally:
        plan.close()


def compare_runs(case, want, got, tag):
    bad = []
    counts, totals = got
    for p in case.props:
        w = dense(want[p.name])
        if not np.array_equal(counts[p.name], w):
            d = np.nonzero(counts[p.name] != w)[0]
            bad.append(f"{tag} {p.name}: {len(d)} voxels differ, sum {int(counts[p.name].sum())} oracle {int(w.sum())}, first {d[:4].tolist()}")
        wt = [t for _, _, t in want[p.name]]
        if list(totals[p.name]) != wt: bad.append(f"{tag} {p.name}: frame totals {totals[p.name]} oracle {wt}")
    return bad


def check_frame_by_frame(case, want):
    import viamd_b200 as vb
    F = case.frames.shape[0]
    plan = _plan(case, batch_frames=1)
    bad = []
    try:
        for f in range(F):
            plan.clear()
            plan.eval_host_frames(case.frames[f:f + 1], [vb.UnitCell(*case.cells[f])], f)
            plan.sync()
            for p in case.props:
                nz, c, total = want[p.name][f]
                got = plan.counts(p.name)
                gnz = np.nonzero(got)[0]
                if not (np.array_equal(gnz, nz) and np.array_equal(got[gnz], c)):
                    bad.append(f"frame {f} {p.name}: {len(np.setxor1d(gnz, nz))} voxels set on one side only, sum {int(got.sum())} oracle {int(c.sum())}")
                gt = plan.frame_counts(p.name, f, want_bins=False)[1]
                if gt != total or int(got.sum()) != total: bad.append(f"frame {f} {p.name}: total {gt} (voxel sum {int(got.sum())}) oracle {total}")
    finally:
        plan.close()
    return bad


def check_case(case):
    if case.require: case.require(frame_geom_of(case))
    want = oracle_frames(case)
    assert sum(t for rows in want.values() for _, _, t in rows) > 0
    bad = check_frame_by_frame(case, want)
    for bf, ns in case.runs:
        bad += compare_runs(case, want, run_whole(case, batch_frames=bf, num_streams=ns), f"batch_frames {bf} streams {ns}")
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


# ----------------------------------------------------------------------------------------------------------------------------- tests
def test_case_table_reaches_its_edges():
    """what the docstrings promise on the oracle side, independent of any kernel"""
    fits = oracle_frames(case_fits())
    for nz, c, t in fits["massless0"]:
        assert t > 0 and nz.tolist() == [0] and int(c[0]) == t             # NaN matrices: every hit in voxel 0
    for name in ("single", "pairs", "planar", "same0", "zmass"): assert all(t > 0 for _, _, t in fits[name])
    faces = oracle_frames(case_faces())
    assert any(len(nz) and nz.max() >= 127 * 128 * 128 for nz, _, _ in faces["faces"])   # the clamp to voxel 127 is reached
    out = oracle_frames(case_outside_aabb())
    assert all(t > 0 for _, _, t in out["above"]) and all(t == 0 for _, _, t in out["far"])


def test_cell_ranges_stay_below_one_chunk():
    """Every structure's cell range spans fewer cells than SDF_MAXSEG, so k_sdf_scatter's chunk loop runs once throughout the table:
    with cell extent = cutoff the bound is 3-4 cells per axis in orthorhombic cells; the widest range of the table is the changing
    shear's, at most 60 cells, so the chunk loop stays unreachable from any of these geometries."""
    import viamd_b200  # noqa: F401   the product library provides mdgpu_debug_frame_geom
    worst = 0
    for make in CASES:
        case = make(); geom = frame_geom_of(case)
        for p in case.props:
            for f in range(case.frames.shape[0]):
                worst = max(worst, cell_range_bound(case, geom, p, f))
    assert worst == 60 and worst < MAXSEG, worst


def test_oracle_equals_the_reference_on_the_edge_geometries(golden_dir):
    """tests/golden/sdf_edges.npz: the reference's per-frame sdf(residue(a:b), targets, r) voxels on the ring, tree, non-periodic,
    cell-less, changing-cell and large-cutoff geometries (make_golden_sdf_edges.py), with the reference's masses and bonds; oracle_lib
    gives the same voxels in every frame"""
    g = np.load(os.path.join(golden_dir, "sdf_edges.npz"))
    names = sorted({k.split("/")[0] for k in g.files})
    checked = 0
    for name in names:
        frames, cells, flags = g[f"{name}/frames"], g[f"{name}/cells"], g[f"{name}/flags"]
        mass, co, ci = g[f"{name}/mass"], g[f"{name}/conn_off"], g[f"{name}/conn_idx"]
        for s, a, b, ta, tb, r in zip(g[f"{name}/stmts"], g[f"{name}/res_a"], g[f"{name}/res_b"], g[f"{name}/trg_a"], g[f"{name}/trg_b"], g[f"{name}/cutoff"]):
            comp = g[f"{name}/comp_off"]
            structs = np.stack([np.arange(comp[k], comp[k + 1]) for k in range(a - 1, b)]).astype(np.int32)
            trg = np.arange(ta - 1, tb, dtype=np.int32)
            for f in range(len(frames)):
                oc = O.UnitCell.from_params(*cells[f], flags[f])
                vol, total = O.sdf_frame(*frames[f], frames[0], mass, structs, trg, co, ci, oc, float(r))
                nz = np.nonzero(vol)[0]
                assert np.array_equal(nz, g[f"{name}/{s}/pf{f}_idx"]) and np.array_equal(vol[nz], g[f"{name}/{s}/pf{f}_val"]), (name, str(s), f)
                checked += 1
    assert names == ["cellless", "large_cutoff", "nonperiodic", "npt", "ring_ortho", "ring_triclinic", "shear", "tree_ortho"] and checked >= 40


def _bad_rows():
    return {"non-ascending": np.array([[0, 5, 2], [10, 15, 12], [20, 25, 22]], np.int32), "duplicates": np.array([[3, 3, 5], [7, 7, 9]], np.int32),
            "descending": np.array([[2, 1, 0], [5, 4, 3]], np.int32)}


def check_rows_rejected():
    import viamd_b200 as vb
    N = 400
    sysm = vb.System(N, np.ones(N, np.float32), conn_offset=np.zeros(N + 1, np.uint32), conn_idx=np.zeros(1, np.int32))
    for kind, rows in _bad_rows().items():
        with pytest.raises(vb.MdgpuError, match=r"sdf 'bad_v'.*not strictly ascending"):
            vb.Plan(sysm, [vb.sdf("bad_v", rows, np.arange(N), 5.0)], 2)
    ok = vb.Plan(sysm, [vb.sdf("ok", np.array([[0, 2, 5], [10, 12, 15]], np.int32), np.arange(N), 5.0)], 2)   # ascending, not contiguous
    ok.close()


@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_under_emulation(emulated_library, make):
    check_case(make())


def test_structure_rows_must_be_strictly_ascending(emulated_library):
    """rows that are not strictly ascending (first - last + 1 == size can hold for them, and k_sdf_scatter would exclude the wrong run) and
    rows with a repeated atom are rejected at plan creation with MDGPU_ERR_INVALID_ARG, naming the property"""
    check_rows_rejected()


def test_compact_ingest_equals_whole_frames(emulated_library):
    """a sparse sdf in a 6 000-atom system: host ingest copies only the atoms it reads (compact atom space, its own indices for structures,
    targets and the exclusion test); equal to whole frames and to the oracle"""
    check_compact_ingest()


def check_compact_ingest():
    N, L, F = 6000, 40.0, 3
    rng = np.random.default_rng(71)
    t = np.array([[0, 0, 0], [0.96, 0, 0], [-0.24, 0.93, 0]])
    fr = molecules(72, t, 1000, N - 3000, [ortho(L, L, L)] * F)
    structs = np.arange(1500, 1500 + 3 * 40).reshape(40, 3)                    # residues 500-539
    sparse_rows = np.stack([np.arange(b, b + 12, 4) for b in range(2000, 2400, 12)])  # non-contiguous rows: contiguous in the compact space
    trg = np.sort(rng.choice(np.arange(3000, N), 500, replace=False))
    case = Case("compact", fr, ortho(L, L, L), [Sdf("res", structs, trg, 6.0), Sdf("sp", sparse_rows, np.arange(2000, 2400, 2), 6.0)],
                bonds=tile_bonds([(0, 1), (0, 2)], 3, 1000))
    want = oracle_frames(case)
    out = {}
    for mode in (0, 1):
        plan = _plan(case, ingest_mode=mode, batch_frames=2)
        import viamd_b200 as vb
        plan.eval_host_frames(case.frames, [vb.UnitCell(*c) for c in case.cells], 0); plan.sync()
        out[mode] = (plan.ingest_info()[0], {p.name: plan.counts(p.name) for p in case.props},
                     {p.name: [plan.frame_counts(p.name, f, want_bins=False)[1] for f in range(F)] for p in case.props})
        plan.close()
    assert out[0][0] < N // 2 and out[1][0] == N, (out[0][0], out[1][0])
    for mode in (0, 1):
        bad = compare_runs(case, want, out[mode][1:], f"ingest_mode {mode}")
        assert not bad, "\n".join(bad)


def test_two_devices_give_the_single_device_volume(emulated_library, monkeypatch):
    """num_devices = 2 under the emulation (frame blocks per device, volumes and frame totals reduced onto devices[0] through the fake
    NCCL) equals one device and the oracle"""
    import build_emul
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    case = case_npt()
    want = oracle_frames(case)
    one = run_whole(case, batch_frames=1)
    two = run_whole(case, batch_frames=1, devices=[0, 1])
    for tag, got in (("one device", one), ("two devices", two)):
        bad = compare_runs(case, want, got, tag)
        assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_on_the_device(make):
    check_case(make())


@pytest.mark.gpu
def test_structure_rows_must_be_strictly_ascending_on_the_device():
    check_rows_rejected()


@pytest.mark.gpu
def test_compact_ingest_equals_whole_frames_on_the_device():
    check_compact_ingest()
