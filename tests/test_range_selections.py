"""Coordinate-range selections within_x / within_y / within_z / within_xyz (md_script_functions.inl:668-671, coordinate_range :2394-2476),
evaluated per frame on the device, as the argument of every consumer of dynamic selections.

CPU: the emulated library (tests/emul: libmdgpu's own sources on host threads) against the reference's results in tests/golden/range6.npz
(tests/golden/make_golden_range.py), the shim's lowering against the Python mirror's, the compositions that are reported instead of lowered,
the ABI's invalid arguments, NaN / infinite coordinates, and a two-device plan. GPU: range6.npz on the device, and a frame-by-frame equivalence
with static selections at a realistic size."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import load_golden, golden_system, vb_system, vb_cell, dense_from_sparse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
TOOL = os.path.join(ROOT, "oracle", "build", "synth_tool")
F = 4


@pytest.fixture
def emulated_library():
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def _same(a, b):
    """temporals through double sin / cos / atan2 or a fit: bit-equal on the CPU build, within 1e-5 on the device (DESIGN.md section 2)"""
    import viamd_b200.api as api
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    if "emul" in os.path.basename(api.LIB_PATH): return bool(np.array_equal(a, b))
    return bool(np.allclose(a, b, rtol=1e-5, atol=1e-6))


def _golden_set(tag):
    g = load_golden("range6.npz"); src = load_golden("water6.npz" if tag == "w" else "tric6.npz")
    sysm = vb_system(golden_system(src))
    frames = g[f"{tag}_frames"]; cells = [vb_cell(g[f"{tag}_cells"][f], g[f"{tag}_cell_flags"][f]) for f in range(F)]
    return g, sysm, frames, cells


def run_range_golden(tag, **plan_kw):
    """The script of set `tag` lowered by the Python mirror, evaluated by the library, against the reference: rdf per-frame bins, pair totals and
    weights, sdf voxels and counts exactly; densities, distances, angles and centres of mass as the static forms of the same procedures."""
    import viamd_b200 as vb
    g, sysm, frames, cells = _golden_set(tag)
    props = vb.compile_script(str(g[f"{tag}_script"]), sysm)
    assert all(p.ranges for p in props)
    plan = vb.Plan(sysm, props, F, keep_frame_results=True, batch_frames=3, **plan_kw)
    plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
    for p in props:
        k = f"{tag}_{p.name}"
        if p.op == vb.OP_RDF:
            for f in range(F):
                bins, tot = plan.frame_counts(p.name, f); ref = g[k + "__pf"][f, :1024]
                assert np.array_equal(bins.astype(np.float32), ref) and tot == int(ref.sum()), (k, f)
            assert np.array_equal(plan.property_data(p.name).weights, g[k + "__pf"][F - 1, 1024:]), k
        elif p.op == vb.OP_SDF:
            vol = np.zeros(128 ** 3, np.float32)
            for f in range(F): vol += dense_from_sparse(g[f"{k}__pf{f}_idx"], g[f"{k}__pf{f}_val"])
            assert np.array_equal(plan.counts(p.name).astype(np.float32), vol) and vol.sum() > 0, k
        elif p.op in (vb.OP_DENSITY_X, vb.OP_DENSITY_Z):
            np.testing.assert_allclose(plan.property_data(p.name).values[:1024], g[k + "__full"][:1024], rtol=1e-5, atol=1e-3, err_msg=k)
        elif p.op == vb.OP_WITHIN_COUNT:
            got = plan.property_data(p.name).values
            assert np.array_equal(got, g[k + "__full"]), (k, got, g[k + "__full"])
            r = p.ranges[0]   # the Python mirror's own reading of the statement selects the same atoms
            assert [int(r.mask(*frames[f]).sum()) for f in range(F)] == [int(v) for v in got], k
        elif p.op == vb.OP_ANGLE:
            np.testing.assert_allclose(plan.property_data(p.name).values, g[k + "__full"], rtol=1e-5, atol=1e-6, err_msg=k)
        else:
            assert _same(plan.property_data(p.name).values, g[k + "__full"]), k
    plan.close()
    return props


@pytest.mark.parametrize("tag", ["w", "t", "u"])
def test_range_selections_against_the_reference_emulated(emulated_library, tag):
    """w: orthorhombic, t: changing triclinic cell, u: triclinic with atoms outside the cell (no rdf there: the reference faults on such frames)"""
    props = run_range_golden(tag)
    forms = {p.name: p for p in props}
    assert forms["c4"].ranges[0].and_idx is not None and forms["c4"].ranges[0].and_idx.size == 0   # `nothing and within_z(:)`: an empty static side
    assert forms["c3"].ranges[0].and_idx.size > 0 and forms["c2"].ranges[0].and_idx.size > 0        # static side after / before the range


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["w", "t", "u"])
def test_range_selections_against_the_reference_on_the_device(tag):
    run_range_golden(tag)


def test_range_counts_skip_nan_and_infinite_coordinates(emulated_library):
    """An axis the call does not constrain is [-FLT_MAX, FLT_MAX] and is still compared: an atom with a NaN or +-inf coordinate on ANY axis is
    never selected, also when that axis is not the range's; finite atoms on the bounds are (both ends inclusive)."""
    import viamd_b200 as vb
    g, sysm, frames, cells = _golden_set("w")
    fr = frames[:2].copy()
    fr[0, 0, 0] = np.nan; fr[0, 1, 3] = np.inf; fr[0, 2, 6] = -np.inf; fr[1, 0, 9] = np.inf; fr[1, 1, 12] = np.nan
    z_lo, z_hi = float(fr[1, 2, 20]), float(fr[1, 2, 40])
    lo, hi = min(z_lo, z_hi), max(z_lo, z_hi)
    props = [vb.count_range("all", vb.Range.axis(2, -vb.api.FLT_MAX, vb.api.FLT_MAX)), vb.count_range("slab", vb.Range.axis(2, lo, hi)),
             vb.count_range("xyz", vb.Range([-vb.api.FLT_MAX] * 3, [vb.api.FLT_MAX] * 3, np.arange(0, 30, dtype=np.int32)))]
    plan = vb.Plan(sysm, props, 2); plan.eval_host_frames(fr, cells[:2], 0)
    assert list(plan.property_data("all").values) == [645.0, 646.0]
    assert list(plan.property_data("xyz").values) == [27.0, 28.0]
    x, y, z = fr[1]; finite = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
    want = int((finite & (lo <= z) & (z <= hi)).sum())
    assert plan.property_data("slab").values[1] == want and want >= 2
    plan.close()


def test_invalid_range_arguments_are_rejected(emulated_library):
    """mdgpu_plan_create: an argument with both a radius and a range, a range with lo > hi, a NaN bound -> MDGPU_ERR_INVALID_ARG"""
    import viamd_b200 as vb
    g, sysm, frames, cells = _golden_set("w")
    o = np.arange(0, 648, 3, dtype=np.int32)
    both = vb.density("b", 2, vb.Range.axis(2, 1.0, 5.0)); both.dyn[0] = (0.0, 3.0, None)
    both_count = vb.count_range("bc", vb.Range.axis(2, 1.0, 5.0)); both_count.cutoff_max = 2.0
    for p in (both, both_count, vb.count_range("inv", vb.Range.axis(0, 5.0, 4.0)), vb.rdf("nan", vb.Range.axis(1, np.nan, 4.0), o, 5.0),
              vb.distance("nan2", vb.Range([0, 0, 0], [1, np.nan, 1]), 3)):
        with pytest.raises(vb.MdgpuError, match="both a radius and a coordinate range|invalid coordinate range"):
            vb.Plan(sysm, [p], F)
    with pytest.raises(vb.MdgpuError, match="not lowered as argument"):   # a range where no dynamic selection is consumed
        p = vb.distance_pair("dp", o[:3], o[3:6]); p.ranges[0] = vb.Range.axis(0, 1.0, 2.0); vb.Plan(sysm, [p], F)
    # mdgpu_range_arg_t entries that name no argument of the plan, or one argument twice
    L = vb.lib(); create = L.mdgpu_plan_create_with_ranges
    for bad, msg in (([(1, 0)], "out of range"), ([(0, 4)], "out of range"), ([(0, 0), (0, 0)], "two ranges")):
        arr = (vb.api._RangeArg * len(bad))()
        for j, (pi, k) in enumerate(bad): arr[j].prop = pi; arr[j].arg = k; arr[j].hi[0] = arr[j].hi[1] = arr[j].hi[2] = 1.0
        L.mdgpu_plan_create_with_ranges = lambda sd, d, n, f, opt, r, nr, arr=arr: create(sd, d, n, f, opt, arr, len(arr))
        try:
            with pytest.raises(vb.MdgpuError, match=msg):
                vb.Plan(sysm, [vb.count_range("c", vb.Range.axis(2, 1.0, 5.0))], F)
        finally:
            L.mdgpu_plan_create_with_ranges = create


def test_property_descriptor_layout_is_that_of_hosts_built_before_ranges(tmp_path):
    """Coordinate ranges travel beside the property descriptors (mdgpu_plan_create_with_ranges), so a host compiled against the header of the
    previous release — which passes arrays of mdgpu_property_desc_t to mdgpu_plan_create — keeps working: the sizes and offsets are unchanged."""
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <mdgpu.h>\nint main(void) { printf("%zu %zu %zu %zu %zu", sizeof(mdgpu_dynamic_arg_t), sizeof(mdgpu_property_desc_t), '
                   'offsetof(mdgpu_property_desc_t, dyn), offsetof(mdgpu_property_desc_t, arg_offsets), offsetof(mdgpu_property_desc_t, arg_parts)); return 0; }\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-std=c11", f"-I{ROOT}/include", str(src), "-o", exe])
    assert subprocess.check_output([exe]).decode().split() == ["32", "320", "144", "272", "304"]


def test_unsupported_range_compositions_are_reported():
    """Everything but `range` and `static and range` (either order) is an error of the Python mirror — and of the shim, where it is built."""
    import viamd_b200 as vb
    sysm = vb.water_system(6)
    for s in UNSUPPORTED:
        with pytest.raises(vb.ScriptError):
            vb.compile_script(s, sysm)


UNSUPPORTED = ["n = count(not within_z(1:2));", "n = count(within(3.0, residue(1)) and within_z(1:2));", "n = count(within_z(1:2) or element('O'));",
               "d = distance(within_z(1:5), 3) in residue(1:4);", "d = distance(element('O') and within_z(1:5), 3) in residue(1:4);",
               "r = rmsd(within_x(1:3));", "p = porosity(within_y(0:9));", "n = count(within_x(1:2) and within_y(1:2));"]

SHIM_FORMS = ("sa = count(within_z(10:)); sb = count(within_xyz(1:2, 3.5:4, :5) and atom(1:4)); sc = count(element('H') and within_x(1.5:7.25)); "
              "sr = rdf(element('O') and within_z(4:12), element('O'), 6.0); srt = rdf(element('O'), within_x(2.5:9.5) and element('H'), 5.0); "
              "srb = rdf(within_z(0:9), within_z(9:19), 4.0); srw = rdf(within(4.0, residue(1)), within_y(3:7), 5.0); sv = sdf(residue(1:20), within_y(3:14) and element('O'), 5.0); "
              "sdz = density_z(element('O') and within_x(0:9)); sdx = density_x(within_xyz(0:10, 2:16, 5:15)); sdy = density_y(within_y(:)); "
              "sd = distance(within_z(2:6) and element('O'), 200); san = angle(within_x(1:5), 10, residue(7)); sh = dihedral(1, within_z(0:4), 100, within_x(10:12)); "
              "scm = com(within_y(5.5:7.25)); sdm = distance_min(within_z(0:3), residue(30)); sdn = distance_max(element('H') and within_y(10:12), within_x(:4)); "
              "se = count((atom(1:3) and residue(10)) and within_z(:)); si = count(within_y(3:7));")


def _shim_lowerer(tmp_path):
    """tests/range_lower.c compiled as oracle/Makefile compiles oracle/shim_harness (the reference's md_script.c + the shim in one unit)"""
    ref = "/root/reference/ext/mdlib"   # REF of oracle/Makefile
    objs = os.path.join(ROOT, "oracle", "_ref", "obj_strict")
    if not (os.path.isdir(os.path.join(ref, "src")) and os.path.isdir(objs)):
        pytest.skip("needs the reference sources and oracle/_ref (make -C oracle ref)")
    inc = [f"-I{ref}/{d}" for d in ("src", "ext/simde", "ext/xxhash", "ext/svd3", "ext/fastlz", "ext/xtc", "ext/stb", "ext/libdivide", "ext/hy36")]
    defs = ["-D__FMA__", "-D__LITTLE_ENDIAN__", "-D__FORCE_ASSERTIONS__=0", "-DMD_GL_SPLINE_SUBDIVISION_COUNT=8", "-D_GNU_SOURCE", "-DNDEBUG"]
    exe = str(tmp_path / "range_lower")
    o = sorted(os.path.join(objs, f) for f in os.listdir(objs) if f.endswith(".o") and f != "md_script.o")
    subprocess.check_call(["gcc", "-std=gnu2x", "-w", "-mavx2", "-mfma", *defs, *inc, "-O2", "-fno-fast-math", "-ffp-contract=off", "-fno-strict-aliasing",
                           f"-I{ROOT}/include", os.path.join(ROOT, "tests", "range_lower.c"), *o, "-o", exe, f"-L{ROOT}/viamd_b200", "-lmdgpu",
                           f"-Wl,-rpath,{ROOT}/viamd_b200", "-lm", "-lpthread"])
    gro = str(tmp_path / "w6.gro"); subprocess.check_call([TOOL, "water-gro", "6", "77", gro])
    return lambda script: subprocess.run([exe, "lower", "--sys", gro, "--script", script], capture_output=True, text=True)


def test_shim_lowering_of_range_forms_matches_python_lowering(tmp_path):
    """integration/md_script_mdgpu.inl lowers the compiled IR of every range form exactly as viamd_b200.script does (op, index lists, bounds,
    static side), and reports the compositions it does not lower."""
    import viamd_b200 as vb
    lower = _shim_lowerer(tmp_path)
    g = load_golden("range6.npz")
    script = SHIM_FORMS + " " + str(g["u_script"])
    p = lower(script); assert p.returncode == 0, p.stderr
    low = [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]
    props = vb.compile_script(script, vb.water_system(6))
    assert [a["name"] for a in low] == [b.name for b in props]
    for a, b in zip(low, props):
        assert a["op"] == b.op and np.float32(a["cutoff"][1]) == np.float32(b.cutoff_max) and a["com_args"] == b.com_args, a["name"]
        for k in range(4):
            want = np.asarray(b.idx[k], np.int32) if k < len(b.idx) else np.zeros(0, np.int32)
            if b.op == vb.OP_RDF and b.ref_within > 0 and k == 2: continue   # the round-1 spelling of a within() reference keeps its AND side in idx[2]
            assert np.array_equal(np.asarray(a["idx"][k], np.int32), want), (a["name"], k)
        for k in range(4):
            d = a["dyn"][k]
            if k in b.ranges:
                r = b.ranges[k]
                assert d["range"] == 1 and d["radius"] == [0, 0], (a["name"], k)
                assert np.array_equal(np.float32(d["lo"]), r.lo) and np.array_equal(np.float32(d["hi"]), r.hi), (a["name"], k, d, r.lo, r.hi)
                assert bool(d["has_and"]) == (r.and_idx is not None) and (r.and_idx is None or np.array_equal(np.asarray(d["and_idx"], np.int32), r.and_idx)), (a["name"], k)
            else:
                assert d["range"] == 0, (a["name"], k)
    for s in UNSUPPORTED:
        p = lower(s)
        assert p.returncode == 3 and "mdgpu" in (p.stdout + p.stderr), (s, p.returncode, p.stderr[-300:])


def test_two_devices_with_a_range_consumer_give_the_single_device_results(emulated_library, monkeypatch):
    """mdgpu_plan_options_t.num_devices = 2 under the emulation (frame blocks per device, accumulators reduced onto devices[0] through the fake
    NCCL of tests/emul): rdf, density and count of range selections equal the single-device evaluation."""
    import build_emul
    import viamd_b200 as vb
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    g, sysm, frames, cells = _golden_set("t")
    src = "r = rdf(element('O') and within_z(4:12), element('O'), 6.0); dz = density_z(within_x(0:9)); n = count(within_y(3:7) and element('H'));"
    out = []
    for devices in (None, [0, 1]):
        plan = vb.Plan(sysm, vb.compile_script(src, sysm), F, keep_frame_results=True, devices=devices)
        plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
        out.append(dict(r=plan.counts("r"), rw=plan.property_data("r").weights, dz=plan.counts("dz"), n=plan.property_data("n").values,
                        rf=np.stack([plan.frame_counts("r", f)[0] for f in range(F)]), mask=plan.frame_mask()))
        if devices: assert plan.exchange_stats()[1] == 1
        plan.close()
    for k in out[0]: assert np.array_equal(out[0][k], out[1][k]), k
    assert out[0]["r"].sum() > 0 and out[0]["mask"].all()


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GPU: a realistic size, frame by frame against static selections
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
def test_range_plans_equal_static_plans_frame_by_frame(tric):
    """water_system(16) (12 288 atoms), 48 frames in batches of 16. For every frame the selected atoms are computed in numpy and the same
    statements are evaluated with those STATIC selections: rdf bins per frame, the accumulated density bins (integer fixed-point sums) and the
    per-frame counts of the dynamic plan equal them exactly — through host ingest in both modes and through mdgpu_eval_device_frames."""
    import viamd_b200 as vb
    n, seed, Fn = 16, 2024, 48
    s = vb.water_system(n); fr, cells = _water_frames(n, seed, Fn, tric)
    L = float(cells[0].x)
    za, zb, xa, xb = 0.3 * L, 0.55 * L, 0.1 * L, 0.4 * L
    src = (f"r = rdf(element('O') and within_z({za:.3f}:{zb:.3f}), element('O'), 8.0); d = density_z(within_x({xa:.3f}:{xb:.3f})); "
           f"c = count(within_z({za:.3f}:{zb:.3f})); ch = count(within_y({xa:.3f}:{xb:.3f}) and element('H'));")
    props = vb.compile_script(src, s)
    rr, rd, rc, rh = (props[i].ranges[0] for i in range(4))
    O = np.nonzero(np.asarray(s.element) == "O")[0].astype(np.int32)
    want_bins, want_dens = [], np.zeros(1024, np.uint64)
    for f in range(Fn):   # static selections of frame f, one plan per frame
        sr = np.nonzero(rr.mask(*fr[f]))[0].astype(np.int32); sd = np.nonzero(rd.mask(*fr[f]))[0].astype(np.int32)
        st = vb.Plan(s, [vb.rdf("r", sr, O, 8.0), vb.density("d", 2, sd)], 1, keep_frame_results=True)
        st.set_initial_frame(*fr[0], cells[0]); st.eval_host_frames(fr[f:f + 1], cells[f:f + 1], 0)
        want_bins.append(st.frame_counts("r", 0)[0]); want_dens += st.counts("d"); st.close()
    want_c = np.array([rc.mask(*fr[f]).sum() for f in range(Fn)], np.float32); want_h = np.array([rh.mask(*fr[f]).sum() for f in range(Fn)], np.float32)
    assert want_c.min() > 0 and len(set(want_c.tolist())) > 1
    d_fr = vb.device_alloc(0, fr.nbytes)
    try:
        vb.memcpy_h2d(0, d_fr, fr.ctypes.data, fr.nbytes)
        for how in ("host0", "host1", "device"):
            plan = vb.Plan(s, props, Fn, keep_frame_results=True, batch_frames=16, ingest_mode=1 if how == "host1" else 0)
            plan.set_initial_frame(*fr[0], cells[0])
            if how == "device": plan.eval_device_frames(d_fr, 3 * fr.shape[2], fr.shape[2], cells, 0, Fn)
            else: plan.eval_host_frames(fr, cells, 0)
            for f in range(Fn): assert np.array_equal(plan.frame_counts("r", f)[0], want_bins[f]), (how, f)
            assert np.array_equal(plan.counts("d"), want_dens), how
            assert np.array_equal(plan.property_data("c").values, want_c) and np.array_equal(plan.property_data("ch").values, want_h), how
            plan.close()
    finally:
        vb.device_free(0, d_fr)
