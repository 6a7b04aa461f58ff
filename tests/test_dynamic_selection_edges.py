"""within() and the coordinate ranges, the per-frame selections every dynamic consumer reads, against the plain-C oracle on adversarial geometries.

Every dynamic selection goes through one query (within.cu): a grid over all atoms with cell extent ceil(r / 6) * 6 (cells.cu), k_within_mark, then
k_within_count (count), k_group_count (count over residues / chains / structures) or k_within_compact (the per-frame index list an rdf,
distance_min, ... reads). k_range_mark feeds the same count and compaction kernels. The case table below drives them where cell-list code goes
wrong: pile-ups on cell faces, radii past half the box, neighbour reach 2 and reach > 2 (the reference returns no pairs), a triclinic shear that
changes inside a batch, non-periodic axes, frames without a cell (with more grid cells than the former fixed default capacity), empty and
complete selections, and more groups than k_group_count has threads. Geometries on which the reference itself faults (reach 2 on a one-cell
grid, unwrapped triclinic frames, frames without a cell beyond about 1 000 atoms; see make_golden_within_edges.py) have no defined answer and
are left out.

All properties of a case are evaluated in ONE plan (each holds its own within() scratch per stream slot, and the slots are reused across batches),
with batch_frames 1 and the default, and compared frame by frame and exactly with the oracle (oracle_lib.within = mdo_within_range):
  count_within             the number of oracle atoms, restricted to the static `and` side
  count_groups             the number of distinct groups among them (atoms in no group count for nothing)
  count_range / _groups    Range.mask
  rdf(Within(...), trg)    oracle_lib.rdf_frame on the oracle's list, bin for bin (the list of k_within_compact, read by a bit-exact consumer)
  distance_min(Within, b)  oracle_lib.min_distance on the oracle's list
Each case's `require` asserts, through mdgpu_debug_frame_geom at the within() grid, that the case reaches the path it names.
tests/golden/within_edges.npz (tests/golden/make_golden_within_edges.py) pins the oracle to the reference on these geometries.

The table runs on the CPU emulation of the library (tests/emul) and, with -m gpu, on the device. A last test drives a batch over its cell
capacity under the AddressSanitizer build of the emulation, in a child process; it never runs on the device.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PBC_X, PBC_Y, PBC_Z, ORTHO, TRICLINIC = 4, 8, 16, 1, 2
PBC_ALL = PBC_X | PBC_Y | PBC_Z
NO_CELL = (0.0,) * 6 + (0,)


# ----------------------------------------------------------------------------------------------------------------------------- properties
class Within:
    def __init__(self, radius, sel, radius_min=0.0, and_idx=None):
        self.radius, self.radius_min = float(radius), float(radius_min)
        self.sel = np.asarray(sel, np.int32); self.and_idx = None if and_idx is None else np.asarray(and_idx, np.int32)

    def vb(self):
        import viamd_b200 as vb
        return vb.Within(self.radius, self.sel, self.radius_min, self.and_idx)

    def oracle(self, x, y, z, cell):
        """the atoms of the frame's selection, ascending"""
        got = O.within(x, y, z, self.sel, self.radius, cell, self.radius_min)
        return got if self.and_idx is None else np.intersect1d(got, self.and_idx).astype(np.int32)


def _range_atoms(rng, x, y, z):
    return np.nonzero(rng.mask(x, y, z))[0].astype(np.int32)


class Count:
    """count(within(...)) or count(range)"""
    def __init__(self, name, sel):
        self.name, self.sel = name, sel

    def prop(self):
        import viamd_b200 as vb
        if isinstance(self.sel, Within):
            w = self.sel
            return vb.count_within(self.name, w.radius, w.sel, w.radius_min, w.and_idx)
        return vb.count_range(self.name, self.sel)

    def want(self, x, y, z, cell):
        a = self.sel.oracle(x, y, z, cell) if isinstance(self.sel, Within) else _range_atoms(self.sel, x, y, z)
        return np.float32(len(a))


class Groups(Count):
    """count(x, 'residue' | 'chain' | ...) over explicit groups"""
    def __init__(self, name, sel, groups):
        super().__init__(name, sel); self.groups = [np.asarray(g, np.int32) for g in groups]

    def prop(self):
        import viamd_b200 as vb
        return vb.count_groups(self.name, self.sel.vb() if isinstance(self.sel, Within) else self.sel, self.groups)

    def want(self, x, y, z, cell):
        a = self.sel.oracle(x, y, z, cell) if isinstance(self.sel, Within) else _range_atoms(self.sel, x, y, z)
        group_of = np.full(len(x), -1, np.int64)
        for k, g in enumerate(self.groups): group_of[g] = k
        hit = group_of[a]
        return np.float32(len(np.unique(hit[hit >= 0])))


class Rdf:
    """rdf(within(...), targets, cutoff): per-frame bins and pair total"""
    def __init__(self, name, ref, trg, cutoff):
        self.name, self.ref, self.trg, self.cutoff = name, ref, np.asarray(trg, np.int32), float(cutoff)

    def prop(self):
        import viamd_b200 as vb
        return vb.rdf(self.name, self.ref.vb() if isinstance(self.ref, Within) else self.ref, self.trg, self.cutoff)

    def want(self, x, y, z, cell):
        r = self.ref.oracle(x, y, z, cell) if isinstance(self.ref, Within) else self.ref
        bins, _, total = O.rdf_frame(x, y, z, r, self.trg, cell, 0.0, self.cutoff)
        return bins, total


class DistMin:
    """distance_min(within(...), b)"""
    def __init__(self, name, a, b):
        self.name, self.a, self.b = name, a, np.asarray(b, np.int32)

    def prop(self):
        import viamd_b200 as vb
        return vb.distance_min(self.name, self.a.vb(), self.b)

    def want(self, x, y, z, cell):
        return np.float32(O.min_distance(x, y, z, self.a.oracle(x, y, z, cell), self.b, cell))


# ----------------------------------------------------------------------------------------------------------------------------- case table
class Case:
    def __init__(self, name, frames, cells, props, batches=(1, 0), require=None):
        self.name = name
        self.frames = np.ascontiguousarray(frames, np.float32)                                # [F, 3, N]
        self.cells = cells if isinstance(cells, list) else [cells] * self.frames.shape[0]     # per frame (x, xy, xz, y, yz, z, flags)
        self.props = props
        self.batches = batches                                                                # batch_frames of the plans (0: the plan's default)
        self.require = require                                                                # geom(frame, radius) -> int32[13]; asserts the path


def ortho(x, y, z, flags=ORTHO | PBC_ALL):
    return (float(x), 0.0, 0.0, float(y), 0.0, float(z), flags)


def frames_pileup(seed, N=500, F=3, L=24.0):
    """coordinates drawn per axis from {0, -0, 3, 6, 12, 18, L, nextafter(L, 0)}: many atoms at one position, pairs at exactly 3 and 6 A, points on
    cell faces (6 A cells) and on both faces of the box"""
    L = np.float32(L)
    vals = np.array([0.0, -0.0, 3.0, 6.0, 12.0, 18.0, L, np.nextafter(L, np.float32(0.0))], np.float32)
    return vals[np.random.default_rng(seed).integers(0, len(vals), (F, 3, N))], float(L)


def frames_box(seed, N, boxes, margin=0.0):
    """uniform points in each frame's orthorhombic box, `margin` (a fraction of the box) outside it on both sides"""
    rng = np.random.default_rng(seed)
    return np.stack([(rng.random((3, N)) * (1 + 2 * margin) - margin) * np.asarray(b, np.float64)[:, None] for b in boxes])


def frames_triclinic(seed, N=900, L=25.0, F=4):
    """a triclinic cell whose shear xy changes every frame, the atoms wrapped into each frame's cell"""
    rng = np.random.default_rng(seed)
    cells = [(L, (0.21 + 0.04 * f) * L, -0.13 * L, L, 0.17 * L, L, TRICLINIC | PBC_ALL) for f in range(F)]
    s = rng.random((F, 3, N)) * L
    fr = np.empty((F, 3, N))
    for f, (_, xy, xz, _, yz, _, _) in enumerate(cells):
        X, Y, Z = s[f]
        fr[f, 0] = X + (xy / L) * Y + (xz / L) * Z; fr[f, 1] = Y + (yz / L) * Z; fr[f, 2] = Z
    return fr, cells


def frames_nonperiodic(seed, N=600, L=(26.0, 31.0, 22.0)):
    """frames 0-2: one axis non-periodic each; frame 3: no cell at all (a grid fitted to the atoms' bounding box); 30 % of the atoms outside"""
    cells = [ortho(*L, ORTHO | (PBC_ALL & ~(PBC_X << k))) for k in range(3)] + [NO_CELL]
    return frames_box(seed, N, [L] * 4, 0.15), cells


def frames_cellless_large(seed, N=1000, F=2, ext=320.0):
    """no cell: half the atoms in a 30 A blob near the lower corner, the rest over a 320 A cube around the origin"""
    rng = np.random.default_rng(seed)
    fr = rng.random((F, 3, N)) * ext - ext / 2
    fr[:, :, : N // 2] = -ext / 2 + 5.0 + rng.random((F, 3, N // 2)) * 30.0
    return fr


def case_pileup():
    fr, L = frames_pileup(101)
    N = fr.shape[2]; sel = np.arange(40); odd = np.arange(1, N, 2)
    res = np.split(np.arange(N), np.cumsum([1 + k % 5 for k in range(N)]))[:-1]
    res = [g for g in res if len(g)]
    props = [Count("c6", Within(6.0, sel)), Count("c599", Within(5.99, sel)), Count("c3", Within(3.0, sel)), Count("m36", Within(6.0, sel, 3.0)),
             Count("c6and", Within(6.0, sel, 0.0, odd)), Count("m36and", Within(6.0, sel, 3.0, odd)),
             Groups("g6", Within(6.0, sel), res), Rdf("rdf3", Within(3.0, sel), np.arange(N), 6.0), DistMin("dmin", Within(5.99, sel), np.arange(400, N)),
             Count("x3", _range(0, 3.0, 3.0)), Count("zero", _range3((-0.0,) * 3, (0.0,) * 3)), Count("y00", _range(1, 0.0, 0.0)),
             Count("zn00", _range(2, -0.0, -0.0)), Count("z612", _range(2, 6.0, 12.0)), Count("xL", _range(0, L, L)),
             Groups("gz", _range(2, 6.0, 12.0, odd), res)]

    def require(geom):
        g6, g3, g599 = geom(0, 6.0), geom(0, 3.0), geom(0, 5.99)
        assert tuple(g6[:3]) == (4, 4, 4) and g6[12] == 1 and max(g6[3:6]) <= 2
        assert tuple(g3[:6]) == (4, 4, 4, 1, 1, 1) and tuple(g599[:6]) == (4, 4, 4, 1, 1, 1)
    return Case("pileup", fr, ortho(L, L, L), props, require=require)


def _range(axis, lo, hi, and_idx=None):
    import viamd_b200 as vb
    return vb.Range.axis(axis, lo, hi, and_idx)


def _range3(lo, hi, and_idx=None):
    import viamd_b200 as vb
    return vb.Range(lo, hi, and_idx)


def case_large_radius():
    """an 18.6 A box (frames 0-1) and a 17.2 A box (frame 2), atoms up to 5 % outside; radii 9.4 / 12 / 17 (past half the box: one cell, reach 1)
    and 40 (reach 3: the reference yields nothing). Reach 2 on a one-cell grid is left out: the reference faults there (see
    make_golden_within_edges.py); the pile-up case has reach 2 on a 4-cell grid."""
    boxes = [(18.6,) * 3] * 2 + [(17.2,) * 3]
    fr = frames_box(102, 260, boxes, 0.05)
    N = fr.shape[2]; sel = np.array([3, 77, 150])
    props = [Count(f"c{r}", Within(r, sel)) for r in (9.4, 12.0, 17.0, 40.0)]
    props += [Count("m912", Within(12.0, sel, 9.0)), Count("m1217", Within(17.0, sel, 12.0)),
              Groups("g17", Within(17.0, sel), [np.arange(k, min(k + 7, N)) for k in range(0, N, 7)]),
              Rdf("rdf12", Within(12.0, sel[:1]), np.arange(N), 9.4), DistMin("dmin", Within(9.4, sel), np.arange(200, N))]

    def require(geom):
        for r in (9.4, 12.0, 17.0):
            for f in range(3): assert tuple(geom(f, r)[[0, 1, 2, 3, 4, 5, 12]]) == (1, 1, 1, 1, 1, 1, 1), (r, f)
        assert all(tuple(geom(f, 40.0)[3:6]) == (3, 3, 3) and geom(f, 40.0)[12] == 0 for f in range(3))
    return Case("large_radius", fr, [ortho(*b) for b in boxes], props, require=require)


def case_triclinic():
    fr, cells = frames_triclinic(103)
    N = fr.shape[2]; sel = np.arange(0, N, 45)
    props = [Count("c35", Within(3.5, sel)), Count("c7", Within(7.0, sel)), Count("m27", Within(7.0, sel, 2.0)),
             Count("c7and", Within(7.0, sel, 0.0, np.arange(0, N, 3))), Groups("g5", Within(5.0, sel), [np.arange(k, k + 3) for k in range(0, N, 3)]),
             Rdf("rdf35", Within(3.5, sel), np.arange(N), 6.0), DistMin("dmin", Within(3.5, sel), np.arange(N - 100, N))]

    def require(geom):
        assert all(geom(f, 3.5)[12] == 1 and geom(f, 7.0)[12] == 1 for f in range(4))
        assert len({c[1] for c in cells}) == 4   # the shear changes inside one default batch
    return Case("triclinic", fr, cells, props, require=require)


def case_nonperiodic():
    fr, cells = frames_nonperiodic(104)
    N = fr.shape[2]; sel = np.arange(0, N, 30)
    props = [Count("c4", Within(4.0, sel)), Count("c75", Within(7.5, sel)), Count("m2575", Within(7.5, sel, 2.5)),
             Count("c75and", Within(7.5, sel, 0.0, np.arange(N // 2))), Groups("g4", Within(4.0, sel), [np.arange(k, k + 4) for k in range(0, N - 50, 4)]),
             Rdf("rdf4", Within(4.0, sel), np.arange(N), 8.0), DistMin("dmin", Within(4.0, sel), np.arange(N - 60, N))]

    def require(geom):
        for f in range(3):
            g = geom(f, 7.5)
            assert g[12] == 1 and not (cells[f][6] & (PBC_X << f))
        assert cells[3][6] == 0 and geom(3, 4.0)[12] == 1
    return Case("nonperiodic", fr, cells, props, batches=(1, 4, 0), require=require)


def case_cellless_large():
    """1 000 atoms over 320 A without a cell: the within() grid at radius 2 and the rdf grid at cutoff 5 need more cells than the former fixed
    default capacity (2^16), so the plan sizes it from the frames (mdgpu_eval_host_frames). The reference evaluates such frames up to about
    1 000 atoms and faults beyond (see make_golden_within_edges.py)."""
    fr = frames_cellless_large(105)
    N = fr.shape[2]; sel = np.arange(50)
    props = [Count("c2", Within(2.0, sel)), Groups("g2", Within(2.0, sel), [np.arange(k, k + 2) for k in range(0, N, 2)]),
             Rdf("rdfw", Within(2.0, sel), np.arange(N), 5.0), Rdf("rdf", np.arange(N), np.arange(N), 5.0)]

    def require(geom):
        for f in range(fr.shape[0]):
            g = geom(f, 2.0)
            assert g[12] == 1 and int(np.prod(g[9:12].astype(np.int64))) + 1 > 1 << 16, g
    return Case("cellless_large", fr, NO_CELL, props, require=require)


def case_selections():
    """an empty selection, one atom, every atom (nothing left once the selection is removed), a selection whose result is empty in frame 1 only
    (atoms 0-1 sit 7 A above all others there), and static sides that remove everything"""
    L = 20.0; N = 400
    fr = frames_box(106, N, [(L, L, L)] * 3)
    fr[1, 2] = np.random.default_rng(7).random(N) * 8.0; fr[1, 2, :2] = 15.0
    two = np.array([0, 1]); allv = np.arange(N)
    props = [Count("empty", Within(3.0, [])), Count("one", Within(4.0, [7])), Count("all", Within(4.0, allv)), Count("two", Within(3.0, two)),
             Count("and_sel", Within(5.0, two, 0.0, two)), Count("and_none", Within(5.0, two, 0.0, [])),
             Groups("gtwo", Within(3.0, two), [np.arange(k, k + 5) for k in range(0, N, 5)]), Groups("gempty", Within(3.0, []), [np.arange(5)]),
             Groups("gnone", Within(3.0, two), []), Rdf("rdf2", Within(3.0, two), allv, 6.0), DistMin("dmin", Within(3.0, two), np.arange(300, N))]

    def require(geom):
        assert all(geom(f, 3.0)[12] == 1 for f in range(3))
    return Case("selections", fr, ortho(L, L, L), props, require=require)


def case_groups():
    """1 500 residues of 1-3 atoms (more groups than the 1 024 threads of k_group_count) and a chain map with atoms in no chain"""
    L = 36.0; N = 3000
    fr = frames_box(107, N, [(L, L, L)] * 2)
    sizes = [1 + (k * 7) % 3 for k in range(N)]
    res = [g for g in np.split(np.arange(N), np.cumsum(sizes))[:-1] if len(g)]
    chains = [np.arange(b, b + 90) for b in range(0, N, 200)]   # atoms 90-199 of every 200 belong to no chain
    sel = np.arange(0, N, 97)
    props = [Groups("res", Within(4.0, sel), res), Groups("res_m", Within(4.0, sel, 2.0), res), Groups("chain", Within(6.0, sel), chains),
             Groups("chain_and", Within(6.0, sel, 0.0, np.arange(0, N, 2)), chains), Groups("res_rng", _range(0, 5.0, 9.0), res),
             Groups("chain_rng", _range3((0.0, 0.0, 0.0), (18.0, 18.0, 36.0), np.arange(N // 2)), chains), Count("atoms", Within(4.0, sel))]

    def require(geom):
        assert len(res) > 1024
    return Case("groups", fr, ortho(L, L, L), props, require=require)


CASES = [case_pileup, case_large_radius, case_triclinic, case_nonperiodic, case_cellless_large, case_selections, case_groups]
CASE_IDS = [c.__name__[5:] for c in CASES]


# ----------------------------------------------------------------------------------------------------------------------------- evaluation
_ORACLE = {}


def oracle(case):
    """per property: the oracle's value of every frame"""
    if case.name not in _ORACLE:
        rows = {p.name: [] for p in case.props}
        for f in range(case.frames.shape[0]):
            x, y, z = case.frames[f]; oc = O.UnitCell(*case.cells[f])
            for p in case.props: rows[p.name].append(p.want(x, y, z, oc))
        _ORACLE[case.name] = rows
    return _ORACLE[case.name]


def frame_geom_of(case):
    """geom(frame, radius) -> mdgpu_debug_frame_geom at the within() grid of that frame: cell extent ceil(r / 6) * 6, cutoff r (as float), grid
    fitted to the bounding box of all atoms and the origin on non-periodic axes, as k_aabb builds it"""
    import ctypes as C
    import viamd_b200 as vb
    from viamd_b200 import api
    L = api.lib(); L.mdgpu_debug_frame_geom.argtypes = [C.POINTER(vb.UnitCell), C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]

    def geom(f, r):
        r = float(np.float32(r)); cell = vb.UnitCell(*case.cells[f])
        p = case.frames[f]
        box = np.concatenate([np.minimum(p.min(axis=1), 0.0), np.maximum(p.max(axis=1), 0.0)]).astype(np.float32)
        gi = np.zeros(13, np.int32); gf = np.zeros(7, np.float32)
        assert L.mdgpu_debug_frame_geom(C.byref(cell), np.ceil(r / 6.0) * 6.0, r, box.ctypes.data, gi.ctypes.data, gf.ctypes.data) == 0
        return gi
    return geom


def evaluate(case, batch_frames):
    """every property of the case in one plan -> {name: per-frame values}; rdf: [(bins float32, total)]"""
    import viamd_b200 as vb
    F, _, N = case.frames.shape
    plan = vb.Plan(vb.System(N, np.ones(N, np.float32)), [p.prop() for p in case.props], F, keep_frame_results=True, batch_frames=batch_frames)
    try:
        plan.eval_host_frames(case.frames, [vb.UnitCell(*c) for c in case.cells], 0)
        plan.sync()
        assert plan.frame_mask().all()
        out = {}
        for p in case.props:
            if isinstance(p, Rdf):
                out[p.name] = [(b.astype(np.float32), t) for b, t in (plan.frame_counts(p.name, f) for f in range(F))]
            else:
                out[p.name] = np.asarray(plan.property_data(p.name).values, np.float32).reshape(F, -1)[:, 0]
        return out
    finally:
        plan.close()


def compare(case, got, tag):
    bad = []
    for p in case.props:
        for f, want in enumerate(oracle(case)[p.name]):
            if isinstance(p, Rdf):
                (gb, gt), (wb, wt) = got[p.name][f], want
                if gt != wt or not np.array_equal(gb, wb):
                    bad.append(f"{tag} {p.name} frame {f}: total {gt} oracle {wt}, {int((gb != wb).sum())} bins differ")
            elif got[p.name][f].tobytes() != np.float32(want).tobytes():
                bad.append(f"{tag} {p.name} frame {f}: {got[p.name][f]!r} oracle {want!r}")
    return bad


def check_case(case):
    if case.require: case.require(frame_geom_of(case))
    bad = []
    for b in case.batches: bad += compare(case, evaluate(case, b), f"batch_frames {b}")
    assert not bad, f"{case.name}: {len(bad)} mismatches\n" + "\n".join(bad[:30])


def _check_case_table():
    """what the docstrings promise about the oracle side, independent of any kernel"""
    o = {c.__name__: oracle(c()) for c in (case_large_radius, case_selections, case_pileup)}
    lr = o["case_large_radius"]
    assert all(v == 0 for v in lr["c40.0"]) and min(lr["c9.4"]) > 0 and min(lr["m1217"]) > 0
    sel = o["case_selections"]
    assert [v > 0 for v in sel["two"]] == [True, False, True] and all(v == 0 for k in ("empty", "all", "and_sel", "and_none") for v in sel[k])
    assert min(sel["one"]) > 0
    pu = o["case_pileup"]
    assert min(pu["m36"]) > 0 and min(pu["x3"]) > 0 and min(pu["zero"]) > 0 and min(pu["xL"]) > 0


@pytest.fixture
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "emul"))
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def test_case_table_reaches_its_edges():
    _check_case_table()


def test_oracle_equals_the_reference_on_the_edge_geometries(golden_dir):
    """tests/golden/within_edges.npz: the reference's count(within([rmin:]r, atom(1:k))) per frame on the pile-up, large-radius (reach 3
    included), triclinic, non-periodic and cell-less geometries; oracle_lib.within gives the same count on every frame"""
    g = np.load(os.path.join(golden_dir, "within_edges.npz"))
    names = sorted({k.split("/")[0] for k in g.files})
    assert names == ["cellless", "large_radius", "nonperiodic", "pileup", "triclinic"]
    checked = 0
    for name in names:
        frames, cells, flags = g[f"{name}/frames"], g[f"{name}/cells"], g[f"{name}/flags"]
        for s, k, rmin, rmax in zip(g[f"{name}/stmts"], g[f"{name}/k"], g[f"{name}/rmin"], g[f"{name}/rmax"]):
            want = g[f"{name}/{s}"]
            for f in range(len(frames)):
                oc = O.UnitCell.from_params(*cells[f], flags[f])
                got = len(O.within(*frames[f], np.arange(k), float(rmax), oc, float(rmin)))
                assert got == want[f], (name, str(s), f, got, want[f])
                checked += 1
    assert checked > 50 and g["large_radius/c40"].sum() == 0 and g["pileup/m36"].min() > 0


@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_under_emulation(emulated_library, make):
    check_case(make())


@pytest.mark.gpu
@pytest.mark.parametrize("make", CASES, ids=CASE_IDS)
def test_case_on_the_device(make):
    check_case(make())


# ----------------------------------------------------------------------------------------------------------------------------- cell capacity
def _wide_cellless(seed, N, ext):
    return frames_box(seed, N, [(ext,) * 3], 0.0) - ext / 2


def test_default_capacity_follows_the_host_frames(emulated_library):
    """Without cell_capacity, host frames without a cell size the grid reservation from their bounding box: 320 A evaluates. A later frame
    that needs more cells fails its batch with MDGPU_ERR_CAPACITY, stays out of the frame mask, and the next evaluation is correct."""
    import viamd_b200 as vb
    N = 1200; sel = np.arange(40)
    big = _wide_cellless(201, N, 320.0)[0]
    huge = _wide_cellless(202, N, 3000.0)[0]
    frames = np.stack([big, huge, big * 0.5, big]).astype(np.float32)
    plan = vb.Plan(vb.System(N, np.ones(N, np.float32)), [vb.count_within("c", 6.0, sel)], 4, batch_frames=1)
    try:
        cell = vb.UnitCell(*NO_CELL)
        plan.eval_host_frames(frames[:1], [cell], 0); plan.sync()
        with pytest.raises(vb.MdgpuError, match="cell capacity"):
            plan.eval_host_frames(frames[1:2], [cell], 1); plan.sync()
        plan.eval_host_frames(frames[2:], [cell] * 2, 2); plan.sync()
        assert list(plan.frame_mask()) == [True, False, True, True]
        vals = np.asarray(plan.property_data("c").values, np.float32).reshape(4, -1)[:, 0]
        oc = O.UnitCell(*NO_CELL)
        for f in (0, 2, 3):
            assert vals[f] == len(O.within(*frames[f], sel, 6.0, oc)), f
    finally:
        plan.close()


_ASAN_CHILD = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import viamd_b200.api as api
api.LIB_PATH = sys.argv[2]; api._lib = None
import viamd_b200 as vb
import oracle_lib as O
from test_dynamic_selection_edges import NO_CELL, ortho, _wide_cellless, frames_box
N = 1000; sel = np.arange(30)
wide = _wide_cellless(301, N, 200.0)[0]                     # radius 2: 34^3 grid cells, over twice the capacity of the batch's two frames
small = frames_box(302, N, [(20.0,) * 3] * 3)
cells = [vb.UnitCell(*NO_CELL), vb.UnitCell(*ortho(20, 20, 20))]
plan = vb.Plan(vb.System(N, np.ones(N, np.float32)), [vb.count_within("c", 2.0, sel), vb.rdf("r", vb.Within(2.0, sel), np.arange(N), 5.0)], 4,
               batch_frames=2, cell_capacity=4096, keep_frame_results=True)
try:
    plan.eval_host_frames(np.stack([wide, small[0]]).astype(np.float32), cells, 0); plan.sync()
    raise SystemExit("no error for a frame over the cell capacity")
except vb.MdgpuError as e:
    assert "cell capacity" in str(e), str(e)
assert not plan.frame_mask().any()
fit = small[1:].astype(np.float32); oc = O.UnitCell(*ortho(20, 20, 20))
plan.eval_host_frames(fit, [cells[1]] * 2, 2); plan.sync()
assert list(plan.frame_mask()) == [False, False, True, True]
vals = np.asarray(plan.property_data("c").values, np.float32).reshape(4, -1)[:, 0]
for f in (2, 3):
    w = O.within(*fit[f - 2], sel, 2.0, oc)
    assert vals[f] == len(w), (f, vals[f], len(w))
    bins, tot = plan.frame_counts("r", f); ob, _, ot = O.rdf_frame(*fit[f - 2], w, np.arange(N), oc, 0.0, 5.0)
    assert tot == ot and np.array_equal(bins.astype(np.float32), ob), f
plan.close()
print("OK")
"""


def test_capacity_overflow_stays_inside_its_buffers_under_asan(monkeypatch):
    """A two-frame batch whose frame 0 needs more than twice the explicit cell_capacity: the batch fails with MDGPU_ERR_CAPACITY, its frames
    stay out of the mask, AddressSanitizer sees no access outside the cell-list buffers (k_scan_cells scans nothing for such a frame), and the
    same plan then evaluates frames that fit equal to the oracle. CPU only: the emulated library built with -fsanitize=address, in a child
    process with libasan preloaded."""
    sys.path.insert(0, os.path.join(HERE, "emul"))
    import build_emul
    monkeypatch.setenv("MDGPU_EMUL_ASAN", "1")
    lib_path = build_emul.build_library()
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan): pytest.skip("gcc has no libasan")
    env = {k: v for k, v in os.environ.items() if not k.startswith("MDGPU_EMUL")}
    env.update(LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _ASAN_CHILD, ROOT, lib_path]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert "AddressSanitizer" not in r.stderr, r.stderr[-6000:]
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), (r.returncode, r.stdout[-2000:], r.stderr[-4000:])
