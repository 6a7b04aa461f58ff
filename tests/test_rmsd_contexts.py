"""rmsd() inside `in` contexts (_rmsd md_script_functions.inl:4287-4345 under evaluate_context md_script.c:3418-3500): one fit per context and
frame, k_rmsd_groups on the device, a [F, n] temporal with the per-frame aggregates.

CPU: the plain-C oracle over each context's group and the emulated library (tests/emul: libmdgpu's own sources on host threads) against the
reference's results in tests/golden/rmsdctx.npz (tests/golden/make_golden_rmsdctx.py); the shim's lowering against the Python mirror's, the
shim-only forms on the emulated library, the forms that are reported instead of lowered, invalid groups and a two-device plan.
GPU: rmsdctx.npz on the device, and a column-by-column equivalence with separate rmsd() properties at a realistic size."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
from helpers import load_golden, golden_system, cell_from_row, vb_cell

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
TOOL = os.path.join(ROOT, "oracle", "build", "synth_tool")
PDB = "/root/reference/datasets/1ALA-500.pdb"
SETS = {"a": ("ala50.npz", "ALA"), "w": ("water6.npz", "SOL"), "t": ("tric6.npz", "SOL")}
MIRROR = ("r", "ro", "rh", "r7", "rn")   # what the Python mirror lowers; rr / ra are context-relative and re takes an identifier: shim only


@pytest.fixture
def emulated_library():
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def _same(a, b):
    """a fit: bit-equal on the CPU build, within 1e-5 relative on the device (DESIGN.md section 2)"""
    import viamd_b200.api as api
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    if "emul" in os.path.basename(api.LIB_PATH): return bool(np.array_equal(a, b))
    return bool(np.allclose(a, b, rtol=1e-5, atol=1e-7))


def _set(tag):
    """(golden, frame set, system dict, viamd_b200.System with the set's residue name, frames, cells)"""
    import viamd_b200 as vb
    name, resname = SETS[tag]
    g = load_golden("rmsdctx.npz"); src = load_golden(name); s = golden_system(src)
    sym = {1: "H", 6: "C", 7: "N", 8: "O"}
    vs = vb.System(len(s["mass"]), s["mass"], s["conn_off"], s["conn_idx"], element=[sym.get(int(z), "X") for z in s["z"]], name=s["names"],
                   resname=[resname] * (len(s["comp_off"]) - 1), res_atom_offset=s["comp_off"])
    cells = [vb_cell(src["cells"][f], src["cell_flags"][f]) for f in range(src["frames"].shape[0])]
    return g, src, s, vs, src["frames"], cells


def _statements(g, tag, names):
    return " ".join(st.strip() + ";" for st in str(g[f"{tag}_script"]).split(";") if st.strip() and st.split("=")[0].strip() in names)


def _groups(s, stmt):
    """the reference's groups of each statement: per context the atoms of (argument AND context); residue() and atom() count from the
    context's first residue / atom, so residue(1:3) in a one-residue context is that residue"""
    co = s["comp_off"]; nres = len(co) - 1; z = np.asarray(s["z"]); names = np.asarray(s["names"])
    res = [np.arange(co[r], co[r + 1]) for r in range(nres)]
    pick = {"r": lambda a: a, "rr": lambda a: a, "rn": lambda a: a, "ro": lambda a: a[z[a] == 8], "rh": lambda a: a[z[a] == 1], "ra": lambda a: a[:2],
            "re": lambda a: a[np.isin(names[a], ["H1", "H2", "H3"])]}
    if stmt == "r7": return [res[6].astype(np.int32)]
    return [pick[stmt](a).astype(np.int32) for a in res]


def _check(tag, name, plan, g, exact=False):
    k = f"{tag}_{name}"; d = plan.property_data(name)
    assert tuple(d.dim[:2]) == tuple(g[k + "__dim"][:2]), k
    same = (lambda a, b: np.array_equal(a, b)) if exact else _same
    assert same(d.values, g[k + "__full"]), (k, np.abs(d.values - g[k + "__full"]).max())
    if k + "__mean" in g:
        agg = plan.aggregate(name)
        for a in ("mean", "var", "ext"): assert same(np.asarray(agg[a]).reshape(-1), g[f"{k}__{a}"].reshape(-1)), (k, a)


@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_oracle_per_context_equals_the_reference(tag):
    """mdo_rmsd_frame over each context's group (0 for an empty group) equals the reference bit for bit, every statement and frame"""
    g, src, s, _, frames, _ = _set(tag)
    F = frames.shape[0]
    for st in str(g[f"{tag}_script"]).split(";"):
        if "rmsd" not in st: continue
        name = st.split("=")[0].strip(); groups = _groups(s, name)
        want = g[f"{tag}_{name}__full"].reshape(F, len(groups))
        for f in range(F):
            cell = cell_from_row(src["cells"][f], src["cell_flags"][f])
            got = [O.rmsd_frame(*frames[f], frames[0], s["mass"], grp, s["conn_off"], s["conn_idx"], cell) if len(grp) else np.float32(0) for grp in groups]
            assert np.array_equal(np.asarray(got, np.float32), want[f]), (tag, name, f)


def run_golden(tag, props=None, names=MIRROR, **plan_kw):
    """the mirror's lowering of the statements `names` of set `tag` (or the given properties), evaluated by the library, against the reference"""
    import viamd_b200 as vb
    g, src, s, vs, frames, cells = _set(tag)
    F = frames.shape[0]
    if props is None: props = vb.compile_script(_statements(g, tag, names), vs)
    assert all(p.op == vb.OP_RMSD and p.num_structures > 0 for p in props)
    plan = vb.Plan(vs, props, F, batch_frames=7, **plan_kw)
    plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
    for p in props: _check(tag, p.name, plan, g)
    plan.close()


@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_rmsd_contexts_against_the_reference_emulated(emulated_library, tag):
    run_golden(tag)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_rmsd_contexts_against_the_reference_on_the_device(tag):
    run_golden(tag)


def test_groups_may_be_empty_and_share_atoms(emulated_library):
    """groups given through the ABI: empty ones evaluate to 0, an atom may be in several groups, groups of equal size share their unwrap pairs;
    every value equals the oracle's fit of that group"""
    import viamd_b200 as vb
    g, src, s, vs, frames, cells = _set("w")
    groups = [np.arange(0, 6), np.zeros(0, np.int64), np.arange(3, 9), np.array([5]), np.arange(0, 6), np.zeros(0, np.int64), np.arange(30, 42)]
    plan = vb.Plan(vs, [vb.rmsd("g", [x.astype(np.int32) for x in groups])], 4)
    plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
    got = plan.property_data("g").values.reshape(4, len(groups))
    for f in range(4):
        cell = cell_from_row(src["cells"][f], src["cell_flags"][f])
        want = [O.rmsd_frame(*frames[f], frames[0], s["mass"], x.astype(np.int32), s["conn_off"], s["conn_idx"], cell) if len(x) else 0.0 for x in groups]
        assert np.array_equal(got[f], np.asarray(want, np.float32)), f
    assert got[1:, 0].min() > 0 and not got[:, 1].any() and np.array_equal(got[:, 0], got[:, 4])
    plan.close()


def test_invalid_groups_are_rejected(emulated_library):
    """structure offsets that do not cover idx[0] or decrease, or neither offsets nor a structure size -> MDGPU_ERR_INVALID_ARG"""
    import viamd_b200 as vb
    _, _, _, vs, _, _ = _set("w")
    idx = np.arange(0, 12, dtype=np.int32)
    for off, size in (([0, 3, 6, 11], 0), ([0, 3, 6, 13], 0), ([1, 3, 6, 12], 0), ([0, 6, 3, 12], 0), (None, 0), (None, 5)):
        p = vb.Property("bad", vb.OP_RMSD, [idx], num_structures=3, structure_size=size,
                        structure_offsets=None if off is None else np.asarray(off, np.uint32))
        with pytest.raises(vb.MdgpuError, match="rmsd 'bad'"):
            vb.Plan(vs, [p], 4)
    assert vb.lib().mdgpu_last_error is not None
    ok = vb.Plan(vs, [vb.Property("ok", vb.OP_RMSD, [idx], num_structures=4, structure_size=3)], 4)   # runs of structure_size atoms
    assert tuple(ok.property_data("ok").dim[:2]) == (4, 4)
    ok.close()


def test_two_devices_give_the_single_device_results(emulated_library, monkeypatch):
    """mdgpu_plan_options_t.num_devices = 2 under the emulation (frame blocks per device, reduced onto devices[0] through the fake NCCL):
    values and aggregates equal the single-device plan"""
    import build_emul
    import viamd_b200 as vb
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    g, src, s, vs, frames, cells = _set("a")
    F = frames.shape[0]; props = vb.compile_script(_statements(g, "a", ("r", "rh")), vs)
    out = []
    for devices in (None, [0, 1]):
        plan = vb.Plan(vs, props, F, batch_frames=8, devices=devices)
        plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
        out.append([plan.property_data(n).values.copy() for n in ("r", "rh")] + [np.asarray(plan.aggregate("r")[a]).copy() for a in ("mean", "var", "ext")])
        if devices: assert plan.exchange_stats()[1] == 1
        plan.close()
    for a, b in zip(*out): assert np.array_equal(a, b)
    assert out[0][0].max() > 0


# ---------------------------------------------------------------------------------------------------------------------------------------------
# the md_script shim
# ---------------------------------------------------------------------------------------------------------------------------------------------
REPORTED = ["r = rmsd(within(3.0, residue(1))) in residue(:);", "r = rmsd(within_x(1:3)) in residue(1:4);", "x = distance_max(element('O'), element('H')) in residue(:);",
            "m = distance_min(1, 2) in residue(:);", "p = porosity(all) in residue(1:4);"]
DISTANCE_FORMS = ("d = distance(1,3) in residue(:); dc = distance(element('O'), element('H')) in residue(1:10); "
                  "ac = angle(atom(2), element('O'), 3) in residue(1:5);")


def _shim_lowerer(tmp_path):
    """tests/rmsdctx_lower.c compiled as tests/test_range_selections.py compiles tests/range_lower.c"""
    ref = "/root/reference/ext/mdlib"   # REF of oracle/Makefile
    objs = os.path.join(ROOT, "oracle", "_ref", "obj_strict")
    if not (os.path.isdir(os.path.join(ref, "src")) and os.path.isdir(objs)):
        pytest.skip("needs the reference sources and oracle/_ref (make -C oracle ref)")
    inc = [f"-I{ref}/{d}" for d in ("src", "ext/simde", "ext/xxhash", "ext/svd3", "ext/fastlz", "ext/xtc", "ext/stb", "ext/libdivide", "ext/hy36")]
    defs = ["-D__FMA__", "-D__LITTLE_ENDIAN__", "-D__FORCE_ASSERTIONS__=0", "-DMD_GL_SPLINE_SUBDIVISION_COUNT=8", "-D_GNU_SOURCE", "-DNDEBUG"]
    exe = str(tmp_path / "rmsdctx_lower")
    o = sorted(os.path.join(objs, f) for f in os.listdir(objs) if f.endswith(".o") and f != "md_script.o")
    subprocess.check_call(["gcc", "-std=gnu2x", "-w", "-mavx2", "-mfma", *defs, *inc, "-O2", "-fno-fast-math", "-ffp-contract=off", "-fno-strict-aliasing",
                           f"-I{ROOT}/include", os.path.join(ROOT, "tests", "rmsdctx_lower.c"), *o, "-o", exe, f"-L{ROOT}/viamd_b200", "-lmdgpu",
                           f"-Wl,-rpath,{ROOT}/viamd_b200", "-lm", "-lpthread"])
    systems = {"a": PDB}
    for tag, seed in (("w", "77"), ("t", "91")):
        gro = str(tmp_path / f"{tag}.gro"); subprocess.check_call([TOOL, "water-gro", "6", seed, gro]); systems[tag] = gro
    return lambda tag, script: subprocess.run([exe, "lower", "--sys", systems[tag], "--script", script], capture_output=True, text=True)


def _lowered(p):
    assert p.returncode == 0, p.stderr[-2000:]
    return {a["name"]: a for a in (json.loads(l) for l in p.stdout.splitlines() if l.startswith("{"))}


@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_shim_lowering_matches_the_mirror_and_the_reference(emulated_library, tmp_path, tag):
    """integration/md_script_mdgpu.inl lowers every statement the mirror lowers exactly as viamd_b200.script does (op, groups, offsets); the
    statements only it lowers (context-relative arguments, an identifier) evaluate to the reference's values on the emulated library"""
    import viamd_b200 as vb
    lower = _shim_lowerer(tmp_path)
    g, _, _, vs, _, _ = _set(tag)
    low = _lowered(lower(tag, str(g[f"{tag}_script"])))
    for p in vb.compile_script(_statements(g, tag, MIRROR), vs):
        a = low[p.name]
        assert a["op"] == vb.OP_RMSD and a["num_structures"] == p.num_structures, p.name
        assert np.array_equal(np.asarray(a["structure_offsets"], np.uint32), p.structure_offsets), p.name
        assert np.array_equal(np.asarray(a["idx"][0], np.int32), p.idx[0]), p.name
    shim_only = [vb.Property(n, a["op"], [np.asarray(a["idx"][0], np.int32)], num_structures=a["num_structures"],
                             structure_offsets=np.asarray(a["structure_offsets"], np.uint32)) for n, a in low.items() if n not in MIRROR]
    assert sorted(p.name for p in shim_only) == (["ra", "re", "rr"] if tag == "a" else ["ra", "rr"])
    run_golden(tag, shim_only)


def test_shim_reports_what_it_does_not_lower_and_keeps_distance_in_contexts(tmp_path):
    """dynamic arguments inside contexts and every procedure but distance / angle / dihedral / rmsd are reported, by the shim and by the mirror;
    distance / angle in contexts lower as the mirror lowers them"""
    import viamd_b200 as vb
    lower = _shim_lowerer(tmp_path)
    vs = vb.water_system(6)
    for s in REPORTED:
        p = lower("w", s)
        assert p.returncode == 3 and "mdgpu" in (p.stdout + p.stderr), (s, p.returncode, p.stderr[-300:])
        with pytest.raises(vb.ScriptError):
            vb.compile_script(s, vs)
    # non-static contexts: the mirror reports them (the reference's own compiler crashes on `rmsd(all) in within(3.0, residue(1))`, so the shim
    # never sees one; its check on the contexts' data stays)
    with pytest.raises(vb.ScriptError, match="context expression"):
        vb.compile_script("r = rmsd(all) in within(3.0, residue(1));", vs)
    for s in ("r = rmsd(atom(1:2)) in residue(:);", "r = rmsd(residue(1:3)) in residue(:);"):   # context-relative: the shim only
        with pytest.raises(vb.ScriptError, match="shim only"):
            vb.compile_script(s, vs)
    low = _lowered(lower("w", DISTANCE_FORMS))
    for p in vb.compile_script(DISTANCE_FORMS, vs):
        a = low[p.name]
        assert a["op"] == p.op and a["num_structures"] == p.num_structures and a["com_args"] == p.com_args, p.name
        for k in range(len(p.idx)):
            assert np.array_equal(np.asarray(a["idx"][k], np.int32), p.idx[k]), (p.name, k)
            want = p.arg_offsets.get(k) if p.arg_offsets else None
            assert (a["arg_offsets"][k] is None) == (want is None) and (want is None or np.array_equal(np.asarray(a["arg_offsets"][k], np.uint32), want)), (p.name, k)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GPU: a realistic size, column by column against separate rmsd() properties
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _water_frames(n, seed, Fn, tric):
    """water_system(n) frames [Fn, 3, N] and their cells; tric: sheared into a triclinic cell that changes every frame"""
    import viamd_b200 as vb
    base, L = vb.synth_water_base(n, seed)
    fr = vb.synth_water_frames_host(n, seed, base, 0, Fn).astype(np.float64)
    if not tric: return fr.astype(np.float32), [vb.UnitCell.from_basis(L, L, L)] * Fn
    cells = []
    for f in range(Fn):
        xy, xz, yz = 3.0 + 0.05 * f, -2.0 - 0.03 * f, 4.0 - 0.04 * f
        fr[f, 0] += (xy / L) * fr[f, 1] + (xz / L) * fr[f, 2]; fr[f, 1] += (yz / L) * fr[f, 2]
        cells.append(vb.UnitCell(L, xy, xz, L, yz, L, vb.CELL_TRICLINIC | vb.CELL_PBC_ALL))
    return fr.astype(np.float32), cells


@pytest.mark.gpu
@pytest.mark.parametrize("tric", [False, True], ids=["ortho", "triclinic"])
def test_contexts_equal_separate_rmsd_properties(tric):
    """water_system(16) (12 288 atoms), 48 frames in batches of 16: `rmsd(all) in residue(1:K)` (k_rmsd_groups, one thread per group) equals,
    column for column, K separate `rmsd(residue(k))` properties of the same plan (k_rmsd, one warp per frame). Both run the same wrap, unwrap
    pairs (they depend on the group's size only) and fit in the same order, so the values are bit-equal — through host ingest in both modes
    and through mdgpu_eval_device_frames."""
    import viamd_b200 as vb
    n, seed, Fn, K = 16, 2024, 48, 40
    s = vb.water_system(n); fr, cells = _water_frames(n, seed, Fn, tric)
    src = f"c = rmsd(all) in residue(1:{K}); " + " ".join(f"s{k} = rmsd(residue({k}));" for k in range(1, K + 1))
    props = vb.compile_script(src, s)
    assert props[0].num_structures == K and all(p.num_structures == 0 for p in props[1:])
    d_fr = vb.device_alloc(0, fr.nbytes)
    try:
        vb.memcpy_h2d(0, d_fr, fr.ctypes.data, fr.nbytes)
        for how in ("host0", "host1", "device"):
            plan = vb.Plan(s, props, Fn, batch_frames=16, ingest_mode=1 if how == "host1" else 0)
            plan.set_initial_frame(*fr[0], cells[0])
            if how == "device": plan.eval_device_frames(d_fr, 3 * fr.shape[2], fr.shape[2], cells, 0, Fn)
            else: plan.eval_host_frames(fr, cells, 0)
            got = plan.property_data("c").values.reshape(Fn, K)
            want = np.stack([plan.property_data(f"s{k}").values for k in range(1, K + 1)], axis=1)
            assert np.array_equal(got, want), (how, np.abs(got - want).max())
            assert want[1:].min() > 0, how
            plan.close()
    finally:
        vb.device_free(0, d_fr)
