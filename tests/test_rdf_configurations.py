"""Every rdf candidate-cull configuration and pair-kernel variant against the plain-C oracle, bin for bin, each in a process of its own.

launch_rdf chooses its cull kernel from MDGPU_CULL / MDGPU_CULL_OCC, read once per process (rdf_cull_config in rdf.cu), so setting them inside
the pytest process does nothing once any rdf has run there. Instead a worker (this file run as a script) evaluates the case table below in a
fresh child process whose environment is set before the library loads. It reports the cull it runs (mdgpu_debug_rdf_config) and writes
per-frame bins and pair totals to an .npz file. The parent compares them with the oracle (oracle_lib.rdf_frame; oracle_lib.within for
dynamic selections) and, as raw 32-bit counts, with the list-free scalar kernel (rdf_variant 1), so all configurations equal each other too.

With a GPU (-m gpu) every configuration runs rdf_variant 0, 2 and 4 on the device. Without one, the CPU emulation of the library
(tests/emul) runs every configuration at rdf_variant 0, and variants 2 and 4 under the default cull, the children in parallel.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PBC_X, PBC_Y, PBC_Z, ORTHO, TRICLINIC = 4, 8, 16, 1, 2
PBC_ALL = PBC_X | PBC_Y | PBC_Z

# configuration name (as mdgpu_debug_rdf_config reports it) -> environment of the child
CONFIGS = {
    "full8": {},
    "full6": {"MDGPU_CULL_OCC": "6"},
    "full4": {"MDGPU_CULL_OCC": "4"},
    "half": {"MDGPU_CULL": "half"},
    "flat6": {"MDGPU_CULL": "flat"},
    "flat8": {"MDGPU_CULL": "flat", "MDGPU_CULL_OCC": "8"},
    "flat4": {"MDGPU_CULL": "flat", "MDGPU_CULL_OCC": "4"},
}
EMUL_TIMEOUT, DEVICE_TIMEOUT = 900, 300   # seconds per child


# ----------------------------------------------------------------------------------------------------------------------------- case table
class Dyn:
    """within(radius, sel) as an rdf argument: evaluated per frame"""
    def __init__(self, radius, sel):
        self.radius, self.sel = float(radius), np.asarray(sel, np.int32)


class Case:
    def __init__(self, name, frames, cells, props, batches=(0,), require=None):
        self.name = name
        self.frames = np.ascontiguousarray(frames, np.float32)                    # [F, 3, N]
        self.cells = cells if isinstance(cells, list) else [cells] * self.frames.shape[0]   # per frame (x, xy, xz, y, yz, z, flags)
        self.props = props                                                        # [(name, ref, trg, cutoff_min, cutoff_max)]
        self.batches = batches                                                    # batch_frames of the plans (0: the plan's default)
        self.require = require                                                    # geometry -> None; asserts the case reaches its path


def ortho(x, y, z, flags=ORTHO | PBC_ALL):
    return (float(x), 0.0, 0.0, float(y), 0.0, float(z), flags)


def _sym_ok(g, flags):
    """k_rdf_cull's symmetric mode needs cdim >= 2 ncell + 1 on every periodic axis (cells.cu)"""
    return all(g[k] >= 2 * g[3 + k] + 1 for k in range(3) if flags & (PBC_X << k))


def _cell_counts(p, L, cd):
    """points per cell of an orthorhombic grid, positions wrapped into the box"""
    c = [np.floor(np.mod(p[k], L[k]) / L[k] * cd[k]).astype(np.int64).clip(0, cd[k] - 1) for k in range(3)]
    return np.bincount((c[2] * cd[1] + c[1]) * cd[0] + c[0], minlength=cd[0] * cd[1] * cd[2]).reshape(cd[2], cd[1], cd[0])


def case_slab():
    """Slab: 1 500 atoms in a 3 A layer of a 30 x 30 x 60 A box, cutoff 9 A (3 x 3 x 6 cells). Each of the layer's 9 cells holds more than
    128 targets, so the culls walk a neighbour cell in several 64-wide steps and end on a 1-63-target tail, and the pair kernel runs full
    128-target chunks and 64-target tails. Once for half the atoms against all, once symmetric (the same selection on both sides)."""
    rng = np.random.default_rng(11); N, F, L = 1500, 2, (30.0, 30.0, 60.0)
    p = rng.random((F, 3, N)) * np.array(L)[None, :, None]
    p[:, 2] = 31.0 + 3.0 * rng.random((F, N))
    for f in range(F):
        n = _cell_counts(p[f], L, (3, 3, 6)); n = n[n > 0]
        assert len(n) == 9 and n.min() > 128 and (n % 64).min() > 0
    def require(G):
        assert all(tuple(G[k][f][:3]) == (3, 3, 6) for k in G for f in range(F))
    return Case("slab", p, ortho(*L), [("half", np.arange(0, N, 2), np.arange(N), 0.0, 9.0), ("sym", np.arange(N), np.arange(N), 0.0, 9.0)],
                require=require)


def case_pileup():
    """Pile-up: 500 atoms whose coordinates are drawn from {0, -0.0, 3, 6, 12, 18, L, nextafter(L, 0)} per axis in a 24 A box, 4 cells of 6 A per
    axis: many atoms at identical positions (d2 = 0, below the minimum distance), pairs at exactly 3 and 6 A, targets at a zero gap from the
    reference box in the cull bound, and coordinates on cell boundaries and on both faces of the box. Cutoff 6 A (float rounding of 1 / L
    makes the reach 2, so symmetric mode is off) and 5.99 A (reach 1, symmetric mode on), symmetric and for 100 reference atoms."""
    rng = np.random.default_rng(12); N, F, L = 500, 2, np.float32(24.0)
    vals = np.array([0.0, -0.0, 3.0, 6.0, 12.0, 18.0, L, np.nextafter(L, np.float32(0.0))], np.float32)
    p = vals[rng.integers(0, len(vals), (F, 3, N))]
    def require(G):
        assert tuple(G["sym6"][0][:6]) == (4, 4, 4, 2, 2, 2) and not _sym_ok(G["sym6"][0], PBC_ALL)
        assert tuple(G["sym599"][0][:6]) == (4, 4, 4, 1, 1, 1) and _sym_ok(G["sym599"][0], PBC_ALL)
    return Case("pileup", p, ortho(L, L, L),
                [("sym6", np.arange(N), np.arange(N), 0.0, 6.0), ("sym599", np.arange(N), np.arange(N), 0.0, 5.99), ("part", np.arange(100), np.arange(N), 0.0, 6.0)],
                require=require)


def case_symmetric_cutoffs():
    """Identical reference and target selections (symmetric mode) in an 18.6 A box, atoms up to 5 % outside the cell: cutoff 6.1 A
    (3 cells per axis, reach 1: cdim == 2n+1, symmetric mode on), 9.4 A (past half the box: one cell, cdim < 2n+1, symmetric mode off),
    12 A and 17 A (just under the box length). Reach 2 with symmetric mode off is in case_pileup and case_cell_per_frame."""
    rng = np.random.default_rng(13); N, F, L = 260, 2, 18.6
    p = rng.random((F, 3, N)) * (1.1 * L) - 0.05 * L
    cuts = (6.1, 9.4, 12.0, 17.0)
    def require(G):
        g = {c: G[f"c{c}"][0] for c in cuts}
        assert tuple(g[6.1][:6]) == (3, 3, 3, 1, 1, 1) and _sym_ok(g[6.1], PBC_ALL)
        assert all(tuple(g[c][:3]) == (1, 1, 1) and not _sym_ok(g[c], PBC_ALL) for c in cuts[1:])
    return Case("symmetric_cutoffs", p, ortho(L, L, L), [(f"c{c}", np.arange(N), np.arange(N), 0.0, c) for c in cuts],
                require=require)


def case_selections():
    """Reference and target differ, so symmetric mode must stay off: partial overlap, reference a subset of the target, a single
    reference point, a single target; 700 atoms in a 26 x 31 x 22 A box."""
    rng = np.random.default_rng(14); N, F, L = 700, 2, (26.0, 31.0, 22.0)
    p = rng.random((F, 3, N)) * np.array(L)[None, :, None]
    return Case("selections", p, ortho(*L),
                [("overlap", np.arange(0, 400), np.arange(200, 700), 0.0, 7.0), ("subset", np.arange(0, N, 3), np.arange(N), 0.0, 7.0),
                 ("one_ref", np.array([5]), np.arange(N), 0.0, 10.0), ("one_trg", np.arange(N), np.array([17]), 0.0, 10.0)])


def case_nonperiodic():
    """Each single axis non-periodic (frames 0-2) and no cell at all (frame 3: the grid is fitted to the atoms' bounding box), with 30 % of
    the atoms outside the cell: the enumeration skips wraps across non-periodic axes, and the candidate lists are sized for 125 neighbours."""
    rng = np.random.default_rng(15); N, F, L = 600, 4, (26.0, 31.0, 22.0)
    p = rng.random((F, 3, N)) * (1.3 * np.array(L))[None, :, None] - (0.15 * np.array(L))[None, :, None]
    cells = [ortho(*L, ORTHO | (PBC_ALL & ~(PBC_X << k))) for k in range(3)] + [(0.0,) * 6 + (0,)]
    return Case("nonperiodic", p, cells,
                [("part", np.arange(0, N, 3), np.arange(N), 2.5, 8.0), ("sym", np.arange(N), np.arange(N), 0.0, 7.0)])


def case_triclinic():
    """Triclinic cell (xy = 0.21 L, xz = -0.13 L, yz = 0.17 L), frames 0-1 wrapped into the cell, frames 2-3 unwrapped: 20 % of the atoms
    moved by +a, half of those by -b as well (the construction of test_rdf_triclinic_unwrapped_coordinates_overflow_pass). Reference points
    outside the unit cell populate home cells beyond the grid, the candidate lists outgrow their buffer and the overflow pass
    (k_rdf_pairs<TRI, false, OVF>) evaluates the home cells that did not fit, under every cull."""
    rng = np.random.default_rng(16); N, L = 1500, 25.0
    xy, xz, yz = 0.21 * L, -0.13 * L, 0.17 * L
    s = rng.random((2, 3, N)) * L
    fr = np.empty((4, 3, N))
    for f in range(4):
        X, Y, Z = s[f % 2]
        fr[f, 0] = X + (xy / L) * Y + (xz / L) * Z; fr[f, 1] = Y + (yz / L) * Z; fr[f, 2] = Z
    sh = rng.random(N) < 0.2; half = sh & (np.arange(N) % 2 == 0)
    fr[2:, 0, sh] += L; fr[2:, 0, half] -= xy; fr[2:, 1, half] -= L
    cell = (L, xy, xz, L, yz, L, TRICLINIC | PBC_ALL)
    o = np.arange(0, N, 3); h = np.setdiff1d(np.arange(N), o)
    return Case("triclinic", fr, cell, [("diff", o, h, 0.0, 7.0), ("sym", o, o, 0.0, 7.5)])


OVF_N, OVF_L, OVF_CUT = 4800, 37.0, 6.0


def case_ortho_overflow():
    """Orthorhombic overflow: 4 800 atoms in a 37 A box, references every third atom, targets within(30, atoms 0-9) (nearly the whole
    system), cutoff 6 A: 6 x 6 x 6 cells, 27 neighbour offsets. A dynamic target set gets a list buffer of
    min(27, 125) * max(N / 4, 1024) + 1024 = 27 * 1200 + 1024 = 33 424 entries per frame. Each home cell with reference points advances the
    frame's list cursor by all the targets of its 27 neighbour cells before culling them (the survivors are written compacted inside that
    reservation), and every cell holds reference points, so the reservations add up to 27 * |targets| > 120 000 entries (computed in
    _check_case_table from the cell counts): most home cells do not fit and the overflow pass evaluates them."""
    rng = np.random.default_rng(17); N, F, L = OVF_N, 2, OVF_L
    p = rng.random((F, 3, N)) * L
    ref = np.arange(0, N, 3)
    def require(G):
        assert all(tuple(g[:6]) == (6, 6, 6, 1, 1, 1) for g in G["dyn"])
    return Case("ortho_overflow", p, ortho(L, L, L), [("dyn", ref, Dyn(30.0, np.arange(10)), 0.0, OVF_CUT)], require=require)


def case_empty_reference():
    """A dynamic reference set, within(3, atoms 0-1), that is empty in frame 1 (the two atoms sit 7 A above all others): a frame without
    reference points between frames with some."""
    rng = np.random.default_rng(18); N, F, L = 500, 3, 20.0
    p = rng.random((F, 3, N)) * L
    p[1, 2] = rng.random(N) * 8.0; p[1, 2, :2] = 15.0
    return Case("empty_reference", p, ortho(L, L, L), [("dyn", Dyn(3.0, [0, 1]), np.arange(N), 0.0, 6.0)])


def case_narrow_window():
    """min:max with a narrow window: 4.9:5.0 A for half the atoms against all, 2.0:2.05 A symmetric; 1024 bins over 0.1 A put hits in
    the first and last few bins, and pairs placed at exactly 4.9 / 5.0 / 2.0 / 2.05 A apart (up to float rounding) test both window edges."""
    rng = np.random.default_rng(19); N, F, L = 2000, 2, 20.0
    p = rng.random((F, 3, N)) * L
    for f in range(F):   # atom 2i+1 sits at a window edge from atom 2i, along x
        for i, d in enumerate((4.9, 5.0, 2.0, 2.05, 4.9, 5.0)):
            p[f, :, 2 * i] = (1.0 + 3.0 * i, 1.0 + f, 2.0 + 3.0 * i); p[f, :, 2 * i + 1] = (1.0 + 3.0 * i + d, 1.0 + f, 2.0 + 3.0 * i)
    return Case("narrow_window", p, ortho(L, L, L),
                [("part", np.arange(0, N, 2), np.arange(N), 4.9, 5.0), ("sym", np.arange(N), np.arange(N), 2.0, 2.05)])


def case_cell_per_frame():
    """A cell that changes from frame to frame, fractional positions fixed: 20^3 (reach 1, symmetric mode on), 20 x 20 x 5.5 (one cell
    along z, reach 2: 45 neighbour offsets instead of 27, symmetric mode off), 24 x 20 x 11, 13^3 (2 cells per axis, symmetric mode off).
    Evaluated with batch_frames 1 (one frame per batch: the list buffer grows between batches) and 8 (one batch: per-frame geometry inside it)."""
    rng = np.random.default_rng(20); N = 400
    boxes = [(20.0, 20.0, 20.0), (20.0, 20.0, 5.5), (24.0, 20.0, 11.0), (13.0, 13.0, 13.0)]
    s = rng.random((3, N))
    p = np.stack([s * np.array(b)[:, None] for b in boxes])
    def require(G):
        g = G["sym"]
        assert tuple(g[0][3:6]) == (1, 1, 1) and _sym_ok(g[0], PBC_ALL)
        assert tuple(g[1][3:6]) == (1, 1, 2) and not _sym_ok(g[1], PBC_ALL)
        assert not _sym_ok(g[3], PBC_ALL)
    return Case("cell_per_frame", p, [ortho(*b) for b in boxes],
                [("sym", np.arange(N), np.arange(N), 0.0, 6.0), ("part", np.arange(0, N, 2), np.arange(N), 0.0, 6.0)], batches=(1, 8), require=require)


CASES = [case_slab, case_pileup, case_symmetric_cutoffs, case_selections, case_nonperiodic, case_triclinic, case_ortho_overflow,
         case_empty_reference, case_narrow_window, case_cell_per_frame]


def build_cases():
    return [c() for c in CASES]


# ----------------------------------------------------------------------------------------------------------------------------- worker
def _worker(argv):
    """child process: --lib-path <libmdgpu> --variants 0,2,4 --out <file.npz> [--report-only]"""
    import argparse
    import ctypes as C
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-path", required=True); ap.add_argument("--variants", default="0"); ap.add_argument("--out"); ap.add_argument("--report-only", action="store_true")
    args = ap.parse_args(argv)
    sys.path[:0] = [ROOT, HERE]
    import viamd_b200.api as api
    api.LIB_PATH = args.lib_path; api._lib = None
    import viamd_b200 as vb
    config = api.debug_rdf_config()
    if args.report_only:   # the switches are latched: changing them now must not change the answer
        os.environ["MDGPU_CULL"] = "half" if config != "half" else "flat"; os.environ["MDGPU_CULL_OCC"] = "4"
        print(config, api.debug_rdf_config())
        return 0
    L = api.lib(); L.mdgpu_debug_frame_geom.argtypes = [C.POINTER(vb.UnitCell), C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    out = {"config": np.array(config)}
    for case in build_cases():
        F, _, N = case.frames.shape
        cells = [vb.UnitCell(*c) for c in case.cells]
        props = []
        for name, ref, trg, lo, hi in case.props:
            if isinstance(ref, Dyn): props.append(vb.rdf_within(name, ref.radius, ref.sel, trg, hi, lo))
            else: props.append(vb.rdf(name, ref, vb.Within(trg.radius, trg.sel) if isinstance(trg, Dyn) else trg, hi, lo))
            geom = np.zeros((F, 13), np.int32); gf = np.zeros(7, np.float32)
            cut = float(np.float32(hi))   # the plan keeps cutoff_max as a float and derives the frame's grid from that value
            for f in range(F):
                assert L.mdgpu_debug_frame_geom(C.byref(cells[f]), cut, cut, None, geom[f].ctypes.data, gf.ctypes.data) == 0
            out[f"{case.name}/{name}/geom"] = geom
        for b in case.batches:
            for v in (int(x) for x in args.variants.split(",")):
                plan = vb.Plan(vb.System(N, np.ones(N, np.float32)), props, F, keep_frame_results=True, rdf_variant=v, batch_frames=b)
                plan.eval_host_frames(case.frames, cells, 0)
                for name, *_ in case.props:
                    rows = [plan.frame_counts(name, f) for f in range(F)]
                    out[f"{case.name}/{name}/b{b}/v{v}/bins"] = np.stack([r[0] for r in rows])
                    out[f"{case.name}/{name}/b{b}/v{v}/total"] = np.array([r[1] for r in rows], np.uint64)
                plan.close()
    np.savez(args.out, **out)
    return 0


def _child(env_extra, lib_path, args, timeout):
    env = {k: v for k, v in os.environ.items() if not k.startswith("MDGPU_CULL")}
    env.update(env_extra)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--worker", "--lib-path", lib_path, *args]
    return subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)


def _run(config, lib_path, variants, out_dir, timeout):
    out = os.path.join(out_dir, f"{config}_v{'_'.join(map(str, variants))}.npz")
    r = _child(CONFIGS[config], lib_path, ["--variants", ",".join(map(str, variants)), "--out", out], timeout)
    assert r.returncode == 0, f"worker {config} {variants} failed:\n{r.stdout}\n{r.stderr[-4000:]}"
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


# ----------------------------------------------------------------------------------------------------------------------------- parent
_ORACLE = {}


def _oracle(case):
    """per property and frame: (bins float32 [1024], total) of oracle_lib.rdf_frame, with within() selections from oracle_lib.within"""
    if case.name not in _ORACLE:
        import oracle_lib as O
        res = {}
        for name, ref, trg, lo, hi in case.props:
            rows = []
            for f in range(case.frames.shape[0]):
                x, y, z = case.frames[f]; oc = O.UnitCell(*case.cells[f])
                r = O.within(x, y, z, ref.sel, ref.radius, oc) if isinstance(ref, Dyn) else ref
                t = O.within(x, y, z, trg.sel, trg.radius, oc) if isinstance(trg, Dyn) else trg
                ob, _, ot = O.rdf_frame(x, y, z, r, t, oc, lo, hi)
                rows.append((ob, ot, len(r), len(t)))
            res[name] = rows
        _ORACLE[case.name] = res
    return _ORACLE[case.name]


def _check_case_table(cases):
    """what the docstrings promise about the oracle side of the cases (independent of any kernel)"""
    import oracle_lib as O
    for case in cases:
        for name, rows in _oracle(case).items():
            assert sum(r[1] for r in rows) > 0, (case.name, name, "no pairs at all")
    emp = _oracle(next(c for c in cases if c.name == "empty_reference"))["dyn"]
    assert [r[2] == 0 for r in emp] == [False, True, False]
    ovf = next(c for c in cases if c.name == "ortho_overflow")
    for f, (ob, ot, nr, nt) in enumerate(_oracle(ovf)["dyn"]):
        stride = 27 * max(OVF_N // 4, 1024) + 1024
        ref_cells = _cell_counts(ovf.frames[f][:, ::3], (OVF_L,) * 3, (6, 6, 6))
        t = O.within(*ovf.frames[f], np.arange(10), 30.0, O.UnitCell(*ovf.cells[f]))
        trg_cells = _cell_counts(ovf.frames[f][:, t], (OVF_L,) * 3, (6, 6, 6))
        reach = sum(np.roll(trg_cells, (dz, dy, dx), (0, 1, 2)) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1))
        reserved = int(reach[ref_cells > 0].sum())
        assert nt > OVF_N // 4 and reserved > 3 * stride, (nt, reserved, stride)
    win = _oracle(next(c for c in cases if c.name == "narrow_window"))
    for name in ("part", "sym"):
        acc = sum(r[0] for r in win[name])
        assert acc[:8].sum() > 0 and acc[-8:].sum() > 0, name


def _compare(res, cases, variants, control=None):
    """-> list of mismatches (config's bins and totals against the oracle, and against the scalar kernel's raw counts)"""
    bad = []
    for case in cases:
        orc = _oracle(case)
        if case.require:
            case.require({name: res[f"{case.name}/{name}/geom"] for name, *_ in case.props})
        for name, *_ in case.props:
            for b in case.batches:
                for v in variants:
                    bins, tot = res[f"{case.name}/{name}/b{b}/v{v}/bins"], res[f"{case.name}/{name}/b{b}/v{v}/total"]
                    for f, (ob, ot, _, _) in enumerate(orc[name]):
                        if not np.array_equal(bins[f].astype(np.float32), ob) or int(tot[f]) != ot:
                            bad.append(f"{case.name}/{name} batch {b} variant {v} frame {f}: total {int(tot[f])} oracle {ot}, "
                                       f"{int((bins[f].astype(np.float32) != ob).sum())} bins differ")
                    if control is not None:
                        cb = control[f"{case.name}/{name}/b{b}/v1/bins"]
                        if not np.array_equal(bins, cb):
                            bad.append(f"{case.name}/{name} batch {b} variant {v}: raw counts differ from the scalar kernel's")
    return bad


@pytest.fixture(scope="module")
def cases():
    c = build_cases()
    _check_case_table(c)
    return c


def _launch_all(jobs, lib_path, out_dir, timeout):
    """all children at once (bounded by the cores), each under a timeout; the pool is joined before the module ends"""
    ex = ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1)))
    return ex, {job: ex.submit(_run, job[0], lib_path, job[1], out_dir, timeout) for job in jobs}


EMUL_JOBS = [(c, (0,)) for c in CONFIGS] + [("full8", (2,)), ("full8", (4,)), ("full8", (1,))]
DEVICE_JOBS = [(c, (0, 2, 4)) for c in CONFIGS] + [("full8", (1,))]


@pytest.fixture(scope="module")
def emulated_library():
    """tests/emul/build/libmdgpu_emul.so: the library's sources compiled by g++, built once before any child starts"""
    sys.path.insert(0, os.path.join(HERE, "emul"))
    import build_emul
    return build_emul.build_library()


@pytest.fixture(scope="module")
def emulated_runs(emulated_library, tmp_path_factory):
    ex, futs = _launch_all(EMUL_JOBS, emulated_library, str(tmp_path_factory.mktemp("rdf_cfg_emul")), EMUL_TIMEOUT)
    yield futs
    ex.shutdown(wait=True)


@pytest.fixture(scope="module")
def device_runs(tmp_path_factory):
    from viamd_b200 import api
    ex, futs = _launch_all(DEVICE_JOBS, api.LIB_PATH, str(tmp_path_factory.mktemp("rdf_cfg_device")), DEVICE_TIMEOUT)
    yield futs
    ex.shutdown(wait=True)


def _assert_run(runs, cases, config, variants):
    res = runs[(config, variants)].result()
    assert str(res["config"]) == config
    control = runs[("full8", (1,))].result()
    bad = _compare(res, cases, variants, control)
    assert not bad, f"{config}: {len(bad)} mismatches\n" + "\n".join(bad[:20])


@pytest.mark.parametrize("config,variant", [(c, 0) for c in CONFIGS] + [("full8", 2), ("full8", 4)], ids=lambda x: f"v{x}" if isinstance(x, int) else x)
def test_configuration_under_emulation(emulated_runs, cases, config, variant):
    _assert_run(emulated_runs, cases, config, (variant,))


def test_scalar_kernel_under_emulation(emulated_runs, cases):
    """rdf_variant 1: no cull, no candidate lists: the control every configuration is compared with"""
    res = emulated_runs[("full8", (1,))].result()
    bad = _compare(res, cases, (1,))
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_configuration_on_the_device(device_runs, cases, config):
    _assert_run(device_runs, cases, config, (0, 2, 4))


@pytest.mark.gpu
def test_scalar_kernel_on_the_device(device_runs, cases):
    res = device_runs[("full8", (1,))].result()
    bad = _compare(res, cases, (1,))
    assert not bad, "\n".join(bad[:20])


@pytest.mark.parametrize("env,expect", [
    ({}, "full8"), ({"MDGPU_CULL_OCC": "6"}, "full6"), ({"MDGPU_CULL_OCC": "7"}, "full6"), ({"MDGPU_CULL_OCC": "12"}, "full8"),
    ({"MDGPU_CULL_OCC": "5"}, "full4"), ({"MDGPU_CULL_OCC": "abc"}, "full4"), ({"MDGPU_CULL_OCC": ""}, "full4"),
    ({"MDGPU_CULL": "flat"}, "flat6"), ({"MDGPU_CULL": "flat", "MDGPU_CULL_OCC": "9"}, "flat8"), ({"MDGPU_CULL": "flat", "MDGPU_CULL_OCC": "x"}, "flat4"),
    ({"MDGPU_CULL": "half", "MDGPU_CULL_OCC": "4"}, "half"), ({"MDGPU_CULL": "FLAT"}, "full8"), ({"MDGPU_CULL": "quarter"}, "full8"),
], ids=lambda x: ",".join(f"{k[6:]}={v}" for k, v in x.items()) or "unset" if isinstance(x, dict) else x)
def test_cull_switches_are_read_once(emulated_library, env, expect):
    """mdgpu_debug_rdf_config of a fresh process: MDGPU_CULL = half | flat (exact, anything else: full), MDGPU_CULL_OCC rounded down to 8 / 6 / 4
    (not a number: 4), default 8 for the full-warp cull and 6 for the flattened one; changing the environment afterwards changes nothing.
    Host code only, so the emulated library (the same rdf.cu and plan.cu) answers without a GPU or an nvcc build."""
    r = _child(env, emulated_library, ["--report-only"], 60)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == [expect, expect]


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "--worker":
    sys.exit(_worker(sys.argv[2:]))
