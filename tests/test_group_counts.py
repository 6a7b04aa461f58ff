"""count(x, 'atom' | 'residue' | 'chain' | 'structure') of a per-frame selection x (_count_with_arg md_script_functions.inl:5536 -> internal_count
:5465-5531), evaluated on the device: MDGPU_OP_WITHIN_COUNT with bit 1 of com_args and the groups in idx[1].

CPU: the emulated library (tests/emul) against the reference's values in tests/golden/count6.npz (tests/golden/make_golden_count.py), the
Python mirror's groups against the reference's, the shim's lowering against the mirror's, the forms both report, invalid group arguments and
a two-device plan. GPU: count6.npz on the device, and water_system(16) frame by frame against a numpy brute-force count."""
import os
import sys

import numpy as np
import pytest

from helpers import load_golden, vb_cell
import count_lower

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
TOOL = os.path.join(ROOT, "oracle", "build", "synth_tool")
SETS = ["w", "t", "d", "p"]
SYM = {1: "H", 6: "C", 7: "N", 8: "O", 15: "P", 16: "S"}


@pytest.fixture
def emulated_library():
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    yield api
    api.LIB_PATH, api._lib = saved


def golden_set(tag):
    """the system of set `tag` as the mirror needs it (names, elements, residues, bonds, chain ranges), its frames and cells"""
    import viamd_b200 as vb
    g = load_golden("count6.npz")
    z = g[f"{tag}_z"].astype(int); comp = g[f"{tag}_comp_off"].astype(np.int64)
    s = vb.System(len(z), g[f"{tag}_mass"], g[f"{tag}_conn_off"], g[f"{tag}_conn_idx"], element=[SYM.get(int(v), "X") for v in z],
                  name=[str(n) for n in g[f"{tag}_names"]], resname=["RES"] * (len(comp) - 1), res_atom_offset=comp, chain_atom_range=g[f"{tag}_chains"])
    frames = g[f"{tag}_frames"]
    cells = [vb_cell(g[f"{tag}_cells"][f], g[f"{tag}_cell_flags"][f]) for f in range(len(frames))]
    return g, s, frames, cells


def run_golden(tag, **plan_kw):
    """the script of set `tag` lowered by the Python mirror and evaluated by the library: every value equals the reference's"""
    import viamd_b200 as vb
    g, s, frames, cells = golden_set(tag)
    props = vb.compile_script(str(g[f"{tag}_script"]), s)
    plan = vb.Plan(s, props, len(frames), **plan_kw)
    plan.eval_host_frames(frames, cells, 0)
    got = {p.name: np.array(plan.property_data(p.name).values) for p in props}
    plan.close()
    for p in props:
        want = g[f"{tag}_{p.name}"]
        assert np.array_equal(got[p.name], want), (tag, p.name, got[p.name], want)
        assert p.op == vb.OP_WITHIN_COUNT and bool(p.com_args & 2) == (p.name[0] != "a" and p.name != "one"), p.name
    return got


@pytest.mark.parametrize("tag", SETS)
def test_group_counts_against_the_reference_emulated(emulated_library, tag):
    """w: water6 (orthorhombic), t: tric6 (changing triclinic cell), d: dppc64 (chains differ from residues), p: 1a64 (structures span residues)"""
    got = run_golden(tag, batch_frames=2)
    assert np.array_equal(got["aw"], got["one"])   # 'atom' is the one-argument count


@pytest.mark.parametrize("tag", SETS)
def test_mirror_groups_are_the_references(tag):
    """'structure' groups from the bond graph are md_util_system_infer_structures' (same order, same atoms), 'residue' groups the components"""
    import viamd_b200 as vb
    g, s, _, _ = golden_set(tag)
    st = vb.count_groups_of(s, "structure"); off = g[f"{tag}_struct_off"]; atoms = g[f"{tag}_struct_atoms"]
    assert len(st) == len(off) - 1 and all(np.array_equal(st[k], atoms[off[k]:off[k + 1]]) for k in range(len(st)))
    res = vb.count_groups_of(s, "residue"); comp = g[f"{tag}_comp_off"]
    assert len(res) == len(comp) - 1 and all(r[0] == comp[k] and r[-1] == comp[k + 1] - 1 for k, r in enumerate(res) if len(r))
    ch = vb.count_groups_of(s, "chain")
    assert [(int(c[0]), int(c[-1]) + 1) for c in ch if len(c)] == [tuple(int(v) for v in r) for r in g[f"{tag}_chains"] if r[1] > r[0]]


REPORTED = ["n = count(not within(3.0, residue(1)), 'residue');", "n = count(within(3.0, residue(1)) or element('O'), 'residue');",
            "n = count(within(3.0, residue(1)) and within_z(1:2), 'structure');", "n = count(within_x(1:2) and within_y(1:2), 'chain');",
            "n = count(within(3.0, residue(1)), 'residue') in residue(1:4);"]


def test_mirror_reports_what_stays_out_of_scope():
    """compositions, `in` contexts, unknown count types, 'chain' without chain ranges: ScriptError; the forms rejected before still are"""
    import viamd_b200 as vb
    s = vb.water_system(6)
    for src in REPORTED + ["n = count(within(3.0, residue(1)), 'molecule');", "n = count(within(3.0, residue(1)), 'chain');",
                           "n = count(residue(1:3), 'residue');", "n = count(element('O'));"]:
        with pytest.raises(vb.ScriptError):
            vb.compile_script(src, s)
    assert vb.count_groups_of(vb.System(3, np.ones(3, np.float32)), "structure") == []   # no bonds: no structures


def _sys_path(tag, tmp_path):
    if tag == "w":
        p = str(tmp_path / "w6.gro"); import subprocess; subprocess.check_call([TOOL, "water-gro", "6", "77", p]); return p
    return os.path.join(count_lower.REF, "test_data", {"d": "dppc64.pdb", "p": "1a64.pdb"}[tag])


@pytest.mark.parametrize("tag", ["w", "d", "p"])
def test_shim_lowering_of_group_counts_matches_python_lowering(tmp_path, tag):
    """integration/md_script_mdgpu.inl lowers every form of count(x, type) as viamd_b200.script does: op, com_args, radius, index lists,
    static side, range bounds, and the groups with their offsets; both report the forms that stay out of scope"""
    import viamd_b200 as vb
    if not count_lower.available(): pytest.skip("needs the reference sources and oracle/_ref (make -C oracle ref)")
    exe = count_lower.build(tmp_path); path = _sys_path(tag, tmp_path)
    g, s, _, _ = golden_set(tag)
    script = str(g[f"{tag}_script"])
    rc, low, log = count_lower.lower(exe, path, script); assert rc == 0, log[-500:]
    props = vb.compile_script(script, s)
    assert [a["name"] for a in low] == [b.name for b in props]
    for a, b in zip(low, props):
        assert a["op"] == b.op and a["com_args"] == b.com_args, a["name"]
        assert np.float32(a["cutoff"][0]) == np.float32(b.cutoff_min) and np.float32(a["cutoff"][1]) == np.float32(b.cutoff_max), a["name"]
        for k in range(4):
            want = np.asarray(b.idx[k], np.int32) if k < len(b.idx) else np.zeros(0, np.int32)
            assert np.array_equal(np.asarray(a["idx"][k], np.int32), want), (a["name"], k)
        if b.com_args & 2:
            assert a["num_structures"] == b.num_structures and np.array_equal(np.asarray(a["structure_offsets"], np.uint32), b.structure_offsets), a["name"]
        else:
            assert a["num_structures"] == 0 and a["structure_offsets"] is None, a["name"]
        d = a["dyn0"]
        if 0 in b.ranges:
            r = b.ranges[0]
            assert d["range"] == 1 and np.array_equal(np.float32(d["lo"]), r.lo) and np.array_equal(np.float32(d["hi"]), r.hi), a["name"]
            assert bool(d["has_and"]) == (r.and_idx is not None) and (r.and_idx is None or np.array_equal(np.asarray(d["and_idx"], np.int32), r.and_idx)), a["name"]
        else:
            assert d["range"] == 0 and d["has_and"] == 0, a["name"]
    for src in REPORTED + ["n = count(within(3.0, residue(1)), 'molecule');"]:
        rc, _, log = count_lower.lower(exe, path, src)
        assert rc in (2, 3), (src, rc, log[-300:])   # the front end rejects an unknown type (2); the shim reports the rest (3)
        if "molecule" not in src: assert rc == 3 and "mdgpu" in log, (src, log[-300:])


def test_invalid_group_arguments_are_rejected(emulated_library):
    """mdgpu_plan_create: an atom in two groups, an atom out of range, offsets that do not rise from 0 to idx_count[1] -> MDGPU_ERR_INVALID_ARG;
    no groups at all is valid and counts 0"""
    import viamd_b200 as vb
    g, s, frames, cells = golden_set("w")
    w = vb.Within(4.5, np.arange(15, dtype=np.int32))
    bad = [([np.arange(0, 6), np.arange(5, 9)], "two groups"), ([np.arange(0, 3), np.array([s.num_atoms])], "out of range"),
           ([np.array([-1])], "out of range")]
    for groups, msg in bad:
        with pytest.raises(vb.MdgpuError, match=msg):
            vb.Plan(s, [vb.count_groups("c", w, groups)], 2)
    for off in ([0, 3, 2, 6], [1, 3, 6], [0, 3, 7]):
        p = vb.count_groups("c", w, [np.arange(0, 3), np.arange(3, 6)]); p.structure_offsets = np.array(off, np.uint32); p.num_structures = len(off) - 1
        with pytest.raises(vb.MdgpuError, match="group offsets"):
            vb.Plan(s, [p], 2)
    p = vb.count_groups("c", vb.Range.axis(2, 0.0, 100.0), [np.arange(0, 3)]); p.structure_offsets = None; p.structure_size = 4   # 1 x 4 atoms, 3 given
    with pytest.raises(vb.MdgpuError, match="group offsets"):
        vb.Plan(s, [p], 2)
    p = vb.count_groups("c", vb.Range.axis(2, 0.0, 100.0), [np.arange(0, 3), np.arange(3, 6)]); p.structure_offsets = None; p.structure_size = 3   # runs of 3
    plan = vb.Plan(s, [p, vb.count_groups("none", w, [])], 2); plan.eval_host_frames(frames[:2], cells[:2], 0)
    assert list(plan.property_data("none").values) == [0.0, 0.0] and list(plan.property_data("c").values) == [2.0, 2.0]
    plan.close()


def test_two_devices_give_the_single_device_group_counts(emulated_library, monkeypatch):
    """mdgpu_plan_options_t.num_devices = 2 under the emulation (frame blocks per device, rows merged onto devices[0]): the same values"""
    import build_emul
    import viamd_b200 as vb
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    g, s, frames, cells = golden_set("t")
    src = "r = count(within(4.5, residue(1:5)), 'residue'); st = count(within_z(6:9) and element('O'), 'structure'); c = count(within(2.5:5, residue(1:5)), 'chain');"
    out = []
    for devices in (None, [0, 1]):
        plan = vb.Plan(s, vb.compile_script(src, s), len(frames), devices=devices)
        plan.eval_host_frames(frames, cells, 0)
        out.append({k: np.array(plan.property_data(k).values) for k in ("r", "st", "c")})
        plan.close()
    for k in out[0]: assert np.array_equal(out[0][k], out[1][k]), k
    assert np.array_equal(out[0]["r"], g["t_rw"]) and np.array_equal(out[0]["c"], g["t_cm"])


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tag", SETS)
def test_group_counts_against_the_reference_on_the_device(tag):
    run_golden(tag)
    run_golden(tag, batch_frames=1)


def _min_image_within(fr, L, sel, r):
    """per atom: within r of an atom of sel (minimum image in a cubic box), sel itself excluded; and the smallest |d - r| over the pairs that
    can decide it (a selected atom and one outside the selection)"""
    pos = fr.T.astype(np.float64)                               # [N, 3]
    d = pos[None, :, :] - pos[sel][:, None, :]                   # [S, N, 3]
    d -= L * np.round(d / L)
    dist = np.sqrt((d * d).sum(-1)); dist[:, sel] = np.inf
    return (dist <= r).any(0), float(np.abs(dist - r).min())


@pytest.mark.gpu
def test_group_counts_equal_a_brute_force_count_frame_by_frame():
    """water_system(16) (12 288 atoms), orthorhombic, 48 frames in batches of 16: count(within(r, residue(1:20)), 'residue' / 'structure')
    equals a numpy minimum-image count for every frame — no distance between a selected atom and another atom lies within 1e-3 A of r, so
    float ties decide nothing — through
    host ingest in both modes and through mdgpu_eval_device_frames"""
    import viamd_b200 as vb
    n, seed, Fn, r = 16, 2024, 48, 1.657   # the H-bond shell: no deciding pair of these frames lies within 1e-3 A of it (at 3.5 A they are 1e-5 apart)
    s = vb.water_system(n)
    base, L = vb.synth_water_base(n, seed)
    fr = vb.synth_water_frames_host(n, seed, base, 0, Fn).astype(np.float32); cells = [vb.UnitCell.from_basis(L, L, L)] * Fn
    sel = np.arange(60)
    want_res, want_str = [], []
    for f in range(Fn):
        m, gap = _min_image_within(fr[f], float(L), sel, r)
        assert gap > 1e-3, (f, gap)
        hit = np.nonzero(m)[0]
        want_res.append(len(np.unique(hit // 3))); want_str.append(len(np.unique(hit // 3)))   # every water is one residue and one structure
    want_res = np.array(want_res, np.float32); want_str = np.array(want_str, np.float32)
    assert want_res.min() > 0 and len(set(want_res.tolist())) > 1
    props = vb.compile_script(f"r = count(within({r}, residue(1:20)), 'residue'); s = count(within({r}, residue(1:20)), 'structure'); "
                              f"a = count(within({r}, residue(1:20)));", s)
    d_fr = vb.device_alloc(0, fr.nbytes)
    try:
        vb.memcpy_h2d(0, d_fr, fr.ctypes.data, fr.nbytes)
        for how in ("host0", "host1", "device"):
            plan = vb.Plan(s, props, Fn, batch_frames=16, ingest_mode=1 if how == "host1" else 0)
            if how == "device": plan.eval_device_frames(d_fr, 3 * fr.shape[2], fr.shape[2], cells, 0, Fn)
            else: plan.eval_host_frames(fr, cells, 0)
            assert np.array_equal(plan.property_data("r").values, want_res), how
            assert np.array_equal(plan.property_data("s").values, want_str), how
            assert plan.property_data("a").values.min() >= want_res.min(), how
            plan.close()
    finally:
        vb.device_free(0, d_fr)
