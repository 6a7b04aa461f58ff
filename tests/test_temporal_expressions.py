"""Temporal expressions (MDGPU_OP_EXPRESSION): arithmetic and math functions over other temporal properties, evaluated per frame on the device
(operators md_script_functions.inl:505-571, functions :576-603).

CPU: the emulated library (tests/emul) fed from the Python mirror's lowering against the reference's results in tests/golden/expr6.npz
(tests/golden/make_golden_expr.py), the shim's lowering against the mirror's, the ABI's invalid arguments, a two-device plan and the forms that
stay reported. GPU: expr6.npz on the device, an expression against the host arithmetic of its operands at a realistic size, and the aggregates
of an array expression against numpy."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import load_golden, golden_system, vb_cell

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
TOOL = os.path.join(ROOT, "oracle", "build", "synth_tool")
SETS = {"a": "ala50.npz", "w": "water6.npz", "t": "tric6.npz"}
# evaluated in double and rounded to float on the device, glibc's float functions in the reference: within 2 ulp or 1e-5 relative
ROUNDED = {"f2", "f3", "f4", "f5", "f6", "f7", "f8", "f9", "f10", "f11", "f12", "g1", "g2", "g3", "g6", "z7"}


@pytest.fixture
def emulated_library():
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def _set(tag):
    import viamd_b200 as vb
    src = load_golden(SETS[tag]); s = golden_system(src)
    vs = vb.System(len(s["mass"]), s["mass"], s["conn_off"], s["conn_idx"], res_atom_offset=s["comp_off"])
    F = src["frames"].shape[0]
    return vs, src["frames"], [vb_cell(src["cells"][f], src["cell_flags"][f]) for f in range(F)]


def _close(got, want, exact):
    """bit for bit (NaN where the reference has NaN), or within 2 ulp / 1e-5 relative"""
    got = np.asarray(got, np.float32).reshape(-1); want = np.asarray(want, np.float32).reshape(-1)
    if exact: return bool(np.array_equal(got, want, equal_nan=True))
    if not np.array_equal(np.isnan(got), np.isnan(want)): return False
    ok = ~np.isnan(want)
    ulp = np.abs(got[ok].view(np.int32).astype(np.int64) - want[ok].view(np.int32).astype(np.int64))
    return bool(np.all((ulp <= 2) | np.isclose(got[ok], want[ok], rtol=1e-5, atol=0)))


def run_golden(tag, **plan_kw):
    """the golden script lowered by the Python mirror and evaluated by the library: values, per-frame aggregates and the reported min / max
    value and range of every statement against the reference"""
    import viamd_b200 as vb
    g = load_golden("expr6.npz"); vs, frames, cells = _set(tag)
    F = frames.shape[0]
    props = vb.compile_script(str(g["script"]), vs)
    assert sum(p.op == vb.OP_EXPRESSION for p in props) > 40 and [p.name for p in props if "#" in p.name] == ["x#0"]
    plan = vb.Plan(vs, props, F, batch_frames=7, **plan_kw)
    plan.set_initial_frame(*frames[0], cells[0]); plan.eval_host_frames(frames, cells, 0)
    on_device = "emul" not in os.path.basename(vb.api.LIB_PATH)
    # on the device the procedures' own values are within 1e-5 (DESIGN.md section 2), and a difference of nearly equal operands (a1 - 2, the
    # variance of equal angles) magnifies that: there every result is compared within 1e-4. That the operators themselves are exact on the
    # device is test_difference_equals_the_host_difference_of_its_operands.
    same = (lambda x, y: np.allclose(x, y, rtol=1e-4, atol=1e-4, equal_nan=True)) if on_device else None
    for p in props:
        if "#" in p.name: continue
        k = f"{tag}_{p.name}"; d = plan.property_data(p.name)
        exact = p.name not in ROUNDED   # the exact operators: bit for bit on the emulated build
        check = same or (lambda x, y: _close(x, y, exact))
        assert check(d.values, g[k + "__full"]), (k, d.values[:8], g[k + "__full"][:8])
        meta = np.array([d.min_value, d.max_value, d.min_range[0], d.max_range[0]], np.float32)
        assert check(meta, g[k + "__meta"]), (k, meta, g[k + "__meta"])
        if k + "__mean" in g:
            agg = plan.aggregate(p.name)
            for a in ("mean", "var", "ext"): assert check(agg[a], g[f"{k}__{a}"]), (k, a)
    plan.close()


@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_expressions_against_the_reference_emulated(emulated_library, tag):
    run_golden(tag)


def test_exact_operators_are_bit_exact_on_host_operands(emulated_library):
    """+ - * / neg abs floor ceil min max sqrt of the rows of d1 / d2 equal numpy's float32 arithmetic on the same rows, NaN and inf included"""
    import viamd_b200 as vb
    vs, frames, cells = _set("w")
    src = ("d1 = distance(1, 10); d2 = distance(4, 20); s = sqrt(d1 - d2); m = min(d1 / 0, d2); n = max(0 / (d1 - d1), d2); "
           "c = ceil(d1 * 3) - floor(d2 / 3); q = -(d1 * d2) / (d1 + 1);")
    plan = vb.Plan(vs, vb.compile_script(src, vs), 4); plan.eval_host_frames(frames, cells, 0)
    v = {k: plan.property_data(k).values for k in ("d1", "d2", "s", "m", "n", "c", "q")}
    d1, d2, f32 = v["d1"], v["d2"], np.float32
    with np.errstate(all="ignore"):
        want = dict(s=np.sqrt(d1 - d2), m=np.fmin(d1 / f32(0), d2), n=np.fmax(f32(0) / (d1 - d1), d2), c=np.ceil(d1 * f32(3)) - np.floor(d2 / f32(3)),
                    q=-(d1 * d2) / (d1 + f32(1)))
    for k, w in want.items(): assert np.array_equal(v[k], w.astype(np.float32), equal_nan=True), k
    plan.close()


def _shim_lowerer(tmp_path):
    """tests/expr_lower.c compiled as oracle/Makefile compiles oracle/shim_harness (the reference's md_script.c + the shim in one unit)"""
    ref = "/root/reference/ext/mdlib"   # REF of oracle/Makefile
    objs = os.path.join(ROOT, "oracle", "_ref", "obj_strict")
    if not (os.path.isdir(os.path.join(ref, "src")) and os.path.isdir(objs)):
        pytest.skip("needs the reference sources and oracle/_ref (make -C oracle ref)")
    inc = [f"-I{ref}/{d}" for d in ("src", "ext/simde", "ext/xxhash", "ext/svd3", "ext/fastlz", "ext/xtc", "ext/stb", "ext/libdivide", "ext/hy36")]
    defs = ["-D__FMA__", "-D__LITTLE_ENDIAN__", "-D__FORCE_ASSERTIONS__=0", "-DMD_GL_SPLINE_SUBDIVISION_COUNT=8", "-D_GNU_SOURCE", "-DNDEBUG"]
    exe = str(tmp_path / "expr_lower")
    o = sorted(os.path.join(objs, f) for f in os.listdir(objs) if f.endswith(".o") and f != "md_script.o")
    subprocess.check_call(["gcc", "-std=gnu2x", "-w", "-mavx2", "-mfma", *defs, *inc, "-O2", "-fno-fast-math", "-ffp-contract=off", "-fno-strict-aliasing",
                           f"-I{ROOT}/include", os.path.join(ROOT, "tests", "expr_lower.c"), *o, "-o", exe, f"-L{ROOT}/viamd_b200", "-lmdgpu",
                           f"-Wl,-rpath,{ROOT}/viamd_b200", "-lm", "-lpthread"])
    gro = str(tmp_path / "w6.gro"); subprocess.check_call([TOOL, "water-gro", "6", "77", gro])
    return lambda script: subprocess.run([exe, "lower", "--sys", gro, "--script", script], capture_output=True, text=True)


REPORTED = ["x = shape_weights(all);", "n = count(element('O'));", "r = rdf(element('O'), element('O'), 5.0) - rdf(element('O'), element('H'), 5.0);",
            "d = (distance(1, 2) * 2) in residue(:);", "b = distance(1, 2) > 2;", "{a, b, c} = com(residue(1));",
            "m = min(distance(1, 2) in residue(1:3));", "p = porosity(within_y(0:9)) * 2;"]


def test_shim_lowering_matches_python_lowering(tmp_path):
    """integration/md_script_mdgpu.inl lowers the compiled IR of the golden script exactly as viamd_b200.script does — the same properties, the
    hidden one of the inline call after the script's own, and the same postfix programs — and still reports every out-of-scope form"""
    import viamd_b200 as vb
    lower = _shim_lowerer(tmp_path)
    script = str(load_golden("expr6.npz")["script"])
    p = lower(script); assert p.returncode == 0, p.stderr
    low = [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]
    props = vb.compile_script(script, vb.water_system(6)); names = [b.name for b in props]
    assert [a["name"] for a in low] == names and [a["own"] for a in low] == [int("#" not in n) for n in names]
    for a, b in zip(low, props):
        assert a["op"] == b.op, a["name"]
        prog = [[vb.EXPR_KINDS[k], float(np.float32(v)), names.index(r) if k == "prop" else 0] for k, v, r in (b.program or [])]
        assert [[n[0], float(np.float32(n[1])), n[2]] for n in a["program"]] == prog, a["name"]
        if b.op != vb.OP_EXPRESSION:
            for k in range(len(b.idx)): assert np.array_equal(np.asarray(a["idx"][k], np.int32), np.asarray(b.idx[k], np.int32)), (a["name"], k)
    from test_range_selections import UNSUPPORTED
    from test_rmsd_contexts import REPORTED as CTX_REPORTED
    for s in REPORTED + UNSUPPORTED + CTX_REPORTED:
        p = lower(s)
        # 3: the shim reports it; 2: the front end rejects it; 0 without output: the reference makes no property of it (shape_weights)
        assert (p.returncode == 3 and "mdgpu" in p.stderr) or p.returncode == 2 or (p.returncode == 0 and not p.stdout.strip()), (s, p.returncode, p.stderr[-300:])


def test_out_of_scope_forms_are_reported():
    """arithmetic on distributions, expressions inside `in`, comparisons, destructuring and the forms reported before: ScriptError, never a value"""
    import viamd_b200 as vb
    from test_range_selections import UNSUPPORTED
    from test_rmsd_contexts import REPORTED as CTX_REPORTED
    sysm = vb.water_system(6)
    for s in REPORTED + UNSUPPORTED + CTX_REPORTED + ["d = distance(1, 2); a = angle(1, 2, 3) in residue(1:3); b = angle(1, 2, 3) in residue(1:4); c = a - b;",
                                                     "a = angle(1, 2, 3) in residue(1:3); s = sqrt(a);", "d = distance(1, 2); e = pow(d, 2, 3);", "e = q * 2;"]:
        with pytest.raises(vb.ScriptError):
            vb.compile_script(s, sysm)


def test_invalid_expressions_are_rejected(emulated_library):
    """mdgpu_plan_create_ex: every malformed program -> MDGPU_ERR_INVALID_ARG with its reason"""
    import viamd_b200 as vb
    vs, frames, cells = _set("w")
    base = [vb.distance("d", 0, 9), vb.angle("a", 0, 1, 2), vb.density("rho", 2, np.arange(0, 30, 3, dtype=np.int32)), vb.in_contexts("c3", vb.OP_ANGLE, [1, 0, 2], [0, 3, 6]),
            vb.in_contexts("c4", vb.OP_ANGLE, [1, 0, 2], [0, 3, 6, 9])]
    P, C = (lambda r: ("prop", r)), (lambda v: ("const", v))
    cases = [([P("rho"), C(1), ("add",)], "not a temporal"), ([P("e"), C(1), ("add",)], "cannot name itself"), ([P(99)], "out of range"),
             ([("add",)], "pops an empty stack"), ([P("d"), ("sub",)], "pops an empty stack"), ([C(1)] * 17 + [("add",)] * 16, "more than 16 operands"),
             ([P("d"), P("a")], "instead of one"), ([P("c3"), P("c4"), ("mul",)], "different lengths"), ([P("c3"), ("sqrt",)], "floats only"),
             ([P("c3"), P("d"), ("pow",)], "floats only"), ([P("d"), C(1.0), ("add",)], None)]
    for prog, msg in cases:
        props = base + [vb.expression("e", prog)]
        if msg is None: vb.Plan(vs, props, 4).close(); continue
        with pytest.raises(vb.MdgpuError, match=msg):
            vb.Plan(vs, props, 4)
    with pytest.raises(vb.MdgpuError, match="cycle"):
        vb.Plan(vs, base + [vb.expression("e", [P("f"), C(1), ("add",)]), vb.expression("f", [P("e"), C(2), ("mul",)])], 4)
    bad = vb.expression("e", [P("d")]); bad.program = [("bogus", 0.0, None)]
    with pytest.raises((vb.MdgpuError, KeyError)):
        vb.Plan(vs, base + [bad], 4)
    # an EXPRESSION property without a program, and a program for a property that is no expression (through the C ABI directly)
    L = vb.lib(); create = L.mdgpu_plan_create_ex
    for drop, msg in ((True, "has no program"), (False, "not an expression property")):
        def patched(sd, d, n, f, opt, r, nr, e, ne, drop=drop):
            if drop: return create(sd, d, n, f, opt, r, nr, None, 0)
            e[0].prop = 0; return create(sd, d, n, f, opt, r, nr, e, ne)
        L.mdgpu_plan_create_ex = patched
        try:
            with pytest.raises(vb.MdgpuError, match=msg):
                vb.Plan(vs, base + [vb.expression("e", [P("d")])], 4)
        finally:
            L.mdgpu_plan_create_ex = create


def test_two_devices_give_the_single_device_results(emulated_library, monkeypatch):
    """num_devices = 2 under the emulation (frame blocks per device, rows summed onto devices[0] through the fake NCCL of tests/emul): every
    expression, two levels deep and element-wise on arrays, equals the single-device evaluation"""
    import build_emul
    import viamd_b200 as vb
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    vs, frames, cells = _set("t")
    src = "d1 = distance(1, 10); d2 = distance(4, 20); dd = d1 - d2; e = dd * 2 + sqrt(d1); a = angle(2, 1, 3) in residue(1:5); b = abs(a - dd) / 2;"
    out = []
    for devices in (None, [0, 1]):
        props = vb.compile_script(src, vs)
        plan = vb.Plan(vs, props, 4, devices=devices); plan.eval_host_frames(frames, cells, 0)
        out.append({p.name: (plan.property_data(p.name).values, plan.property_data(p.name).min_value) for p in props})
        out[-1]["agg"] = (plan.aggregate("b")["mean"], 0)
        plan.close()
    for k in out[0]: assert np.array_equal(out[0][k][0], out[1][k][0]) and out[0][k][1] == out[1][k][1], k
    assert out[0]["e"][0].any()


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "w", "t"])
def test_expressions_against_the_reference_on_the_device(tag):
    run_golden(tag)


@pytest.mark.gpu
def test_difference_equals_the_host_difference_of_its_operands():
    """water_system(16) (12 288 atoms), 48 frames in batches of 16: `dd = d1 - d2` equals the host difference of the plan's own d1 and d2 rows bit
    for bit, and an expression of it two levels deep equals the host arithmetic — through host ingest in both modes and from device frames"""
    import viamd_b200 as vb
    n, seed, Fn = 16, 2024, 48
    s = vb.water_system(n); base, L = vb.synth_water_base(n, seed)
    fr = vb.synth_water_frames_host(n, seed, base, 0, Fn); cells = [vb.UnitCell.from_basis(L, L, L)] * Fn
    src = ("d1 = distance(element('O') and residue(1:40), 200); d2 = distance(3, residue(100:130)); dd = d1 - d2; "
           "e = abs(dd) * 2 + d1 / 3; a = angle(2, 1, 3) in residue(1:300); b = a * dd - a;")
    props = vb.compile_script(src, s)
    d_fr = vb.device_alloc(0, fr.nbytes)
    try:
        vb.memcpy_h2d(0, d_fr, fr.ctypes.data, fr.nbytes)
        for how in ("host0", "host1", "device"):
            plan = vb.Plan(s, props, Fn, batch_frames=16, ingest_mode=1 if how == "host1" else 0)
            plan.set_initial_frame(*fr[0], cells[0])
            if how == "device": plan.eval_device_frames(d_fr, 3 * fr.shape[2], fr.shape[2], cells, 0, Fn)
            else: plan.eval_host_frames(fr, cells, 0)
            v = {p.name: plan.property_data(p.name).values for p in props}
            f32 = np.float32
            assert np.array_equal(v["dd"], v["d1"] - v["d2"]) and v["dd"].any(), how
            assert np.array_equal(v["e"], np.abs(v["dd"]) * f32(2) + v["d1"] / f32(3)), how
            a = v["a"].reshape(Fn, 300)
            assert np.array_equal(v["b"].reshape(Fn, 300), a * v["dd"][:, None] - a), how
            plan.close()
    finally:
        vb.device_free(0, d_fr)


@pytest.mark.gpu
def test_array_expression_aggregates_and_histogram():
    """the per-frame mean / variance / extent, min / max and the device histogram of an array expression equal numpy's fold of its rows"""
    import viamd_b200 as vb
    n, seed, Fn = 16, 7, 40
    s = vb.water_system(n); base, L = vb.synth_water_base(n, seed)
    fr = vb.synth_water_frames_host(n, seed, base, 0, Fn); cells = [vb.UnitCell.from_basis(L, L, L)] * Fn
    plan = vb.Plan(s, vb.compile_script("a = angle(2, 1, 3) in residue(1:500); x = floor(a * 100) / 7 - a;", s), Fn)
    plan.eval_host_frames(fr, cells, 0)
    d = plan.property_data("x"); rows = d.values.reshape(Fn, 500); agg = plan.aggregate("x")
    assert tuple(d.dim[:2]) == (Fn, 500)
    for f in range(Fn):
        r = rows[f]; m = np.float32(0)
        for v in r: m += v
        m = m / np.float32(500)
        var = np.float32(0)
        for v in r: var += (v - m) * (v - m)
        assert agg["mean"][f] == m and agg["var"][f] == var / np.float32(500) and tuple(agg["ext"][f]) == (r.min(), r.max()), f
    assert d.min_value == rows.min() and d.max_value == rows.max() and d.min_range[0] == d.min_value and d.max_range[0] == d.max_value
    h, _ = plan.histogram("x", 64, float(rows.min()), float(rows.max()))
    assert h.shape == (500, 64) and np.all(h.sum(axis=1) > 0)
    plan.close()
