"""porosity(selection) per frame on the device (MDGPU_OP_POROSITY): the unoccupied fraction of a bit grid over the selection's van der Waals spheres
(_porosity md_script_functions.inl:5858-6003).

The reference is tests/golden/porosity.npz (tests/golden/make_golden_porosity.py): the reference's own per-frame values on a water box (a prefix
selection whose grid has at most 2^23 voxels and which crosses the periodic boundary, and `all`), on 1ALA frames, and on a triclinic cell. The plain-C
restatement (oracle/md_porosity.c, tests/porosity_oracle.py) equals it value for value and also gives the occupied-voxel count of every frame, which
the library returns through mdgpu_plan_property_frame_rows. The CPU tests run the restatement and the whole C ABI of the emulated library (tests/emul)
on the small cases; the GPU tests run the library on the device, at full size too."""
import os
import sys

import numpy as np
import pytest

import oracle_lib as O
import porosity_oracle as P
from helpers import load_golden

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul"))

CASES = (("wx", "px"), ("wx", "pa"), ("tri", "pt"), ("ala", "pa"))
SMALL = (("wx", "px", slice(0, 4)), ("ala", "pa", slice(0, 3)), ("tri", "pt", slice(0, 2)))   # cases small enough for the CPU emulation


def ocell(g, tag, f):
    return O.UnitCell.from_params(*g[f"{tag}_cells"][f], int(g[f"{tag}_flags"][f]))


def vcells(vb, g, tag, frames):
    return [vb.UnitCell(*(float(v) for v in g[f"{tag}_cells"][f]), int(g[f"{tag}_flags"][f])) for f in frames]


def restated(frames, radius, idx, cells):
    return [P.porosity(fr[0], fr[1], fr[2], radius, idx, c) for fr, c in zip(frames, cells)]


def rows(vb, plan, name):
    """(occupied voxels, N) per frame from the plan's u64 rows"""
    out = []
    for which in (0, 1):
        ptr, nbytes, eb = plan.frame_rows(name, which)
        assert eb == 8 and nbytes == 8 * plan.num_frames
        a = np.zeros(plan.num_frames, np.uint64); vb.memcpy_d2h(plan.device, a.ctypes.data, ptr, nbytes); out.append(a)
    return out


def run_case(vb, frames, cells, radius, idx, ingest_mode=0, batch_frames=0, devices=None):
    n = frames.shape[2]
    plan = vb.Plan(vb.System(n, np.ones(n, np.float32), radius=radius), [vb.porosity("p", idx)], len(frames), ingest_mode=ingest_mode,
                   batch_frames=batch_frames, devices=devices)
    plan.eval_host_frames(frames, cells, 0)
    d = plan.property_data("p")
    s, N = rows(vb, plan, "p")
    plan.close()
    return d, s, N


def check_against(d, s, N, want, values=None):
    assert d.dim[:2] == (len(want), 1) and d.min_range[0] == 0.0 and d.max_range[0] == 1.0
    got = d.values.reshape(-1)
    for f, w in enumerate(want):
        assert got[f] == w["value"], (f, got[f], w["value"])
        assert int(s[f]) == w["set"] and int(N[f]) == w["n"], (f, int(s[f]), w["set"], int(N[f]), w["n"])
        if values is not None: assert got[f] == values[f], (f, got[f], values[f])


def run_golden_cases(vb, cases):
    g = load_golden("porosity.npz")
    for tag, name, sl in cases:
        frames = g[f"{tag}_frames"][sl]; F = len(frames); idx = g[f"{tag}_{name}_idx"]; radius = g[f"{tag}_radius"]
        want = restated(frames, radius, idx, [ocell(g, tag, f) for f in range(F)])
        d, s, N = run_case(vb, frames, vcells(vb, g, tag, range(F)), radius, idx)
        check_against(d, s, N, want, g[f"{tag}_{name}_values"][sl])


def run_error_paths(vb):
    g = load_golden("porosity.npz"); frames = g["wx_frames"][:1]; n = frames.shape[2]; radius = g["wx_radius"]
    with pytest.raises(vb.MdgpuError, match="no atom radii"):
        vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.porosity("p", np.arange(3))], 1)
    bad = radius.copy(); bad[5] = -1.0
    with pytest.raises(vb.MdgpuError, match="negative or not finite"):
        vb.Plan(vb.System(n, np.ones(n, np.float32), radius=bad), [vb.porosity("p", np.arange(3))], 1)
    bad[5] = np.nan
    with pytest.raises(vb.MdgpuError, match="negative or not finite"):
        vb.Plan(vb.System(n, np.ones(n, np.float32), radius=bad), [vb.porosity("p", np.arange(3))], 1)
    d, s, N = run_case(vb, frames, vcells(vb, g, "wx", [0]), radius, np.zeros(0, np.int32))          # empty selection: 0, no grid
    assert d.values[0] == 0.0 and s[0] == 0 and N[0] == 0
    tri = g["tri_frames"]; d, s, N = run_case(vb, tri, vcells(vb, g, "tri", range(2)), g["tri_radius"], np.arange(9))   # triclinic cell: 0
    assert not np.any(d.values) and not np.any(s) and not np.any(N)
    zero = np.zeros_like(radius); d, s, N = run_case(vb, frames, vcells(vb, g, "wx", [0]), zero, np.arange(9))       # radii 0 everywhere
    w = P.porosity(frames[0][0], frames[0][1], frames[0][2], zero, np.arange(9), ocell(g, "wx", 0))
    assert np.array_equal(d.values, [w["value"]], equal_nan=True) and int(s[0]) == w["set"] and int(N[0]) == w["n"]


# ---------------------------------------------------------------------------------------------------------------------------- CPU
def test_restatement_equals_the_reference():
    g = load_golden("porosity.npz")
    for tag, name in CASES:
        frames = g[f"{tag}_frames"]
        got = restated(frames, g[f"{tag}_radius"], g[f"{tag}_{name}_idx"], [ocell(g, tag, f) for f in range(len(frames))])
        assert np.array_equal([r["value"] for r in got], g[f"{tag}_{name}_values"]), (tag, name)


def test_occupied_counts_in_the_exact_regime():
    """where the grid has at most 2^23 voxels the reference's float value determines its occupied count: it is the restatement's"""
    g = load_golden("porosity.npz"); seen = 0
    for tag, name in CASES:
        frames = g[f"{tag}_frames"]
        for f, r in enumerate(restated(frames, g[f"{tag}_radius"], g[f"{tag}_{name}_idx"], [ocell(g, tag, k) for k in range(len(frames))])):
            if r["grid"] and r["n"] <= 1 << 23:
                assert P.set_from_value(g[f"{tag}_{name}_values"][f], r["n"]) == r["set"]; seen += 1
    assert seen >= 7   # the four water-row frames and three 1ALA frames


def test_water_row_needs_deperiodisation():
    """the golden's prefix selection crosses the periodic boundary: without the cell the value differs"""
    g = load_golden("porosity.npz"); fr = g["wx_frames"][0]
    with_cell = P.porosity(fr[0], fr[1], fr[2], g["wx_radius"], g["wx_px_idx"], ocell(g, "wx", 0))
    no_cell = P.porosity(fr[0], fr[1], fr[2], g["wx_radius"], g["wx_px_idx"], O.UnitCell.from_params(*g["wx_cells"][0], 0))
    assert with_cell["value"] == g["wx_px_values"][0] and no_cell["value"] != with_cell["value"]


def test_script_lowering():
    import viamd_b200 as vb
    s = vb.water_system(3)
    p, q = vb.compile_script("p = porosity(residue(1:6)); q = porosity(element('O') or residue(2));", s)
    assert p.op == vb.OP_POROSITY and np.array_equal(p.idx[0], np.arange(18)) and len(p.idx) == 1
    assert np.array_equal(q.idx[0], np.union1d(np.arange(0, 81, 3), [3, 4, 5]))
    with pytest.raises(vb.ScriptError, match="dynamic"):
        vb.compile_script("p = porosity(within(3.0, residue(1)));", s)


@pytest.fixture
def emulated_library():   # per test: a module-scoped swap would still be active when the GPU tests below run
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    import viamd_b200 as vb
    yield vb
    api.LIB_PATH, api._lib = saved


def test_emulated_library_equals_the_reference(emulated_library):
    run_golden_cases(emulated_library, SMALL)


def test_emulated_library_error_paths(emulated_library):
    run_error_paths(emulated_library)


def test_emulated_library_two_device_plan(emulated_library, monkeypatch):
    """two devices evaluate the water-row frames in two blocks; the rows reduced onto devices[0] equal the one-device plan's"""
    import build_emul
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    vb = emulated_library; g = load_golden("porosity.npz"); frames = g["wx_frames"]; cells = vcells(vb, g, "wx", range(4))
    one = run_case(vb, frames, cells, g["wx_radius"], g["wx_px_idx"])
    two = run_case(vb, frames, cells, g["wx_radius"], g["wx_px_idx"], devices=[0, 1])
    assert np.array_equal(one[0].values, two[0].values) and np.array_equal(one[1], two[1]) and np.array_equal(one[2], two[2])
    assert np.array_equal(one[0].values, g["wx_px_values"])


# ---------------------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_device_equals_the_reference():
    import viamd_b200 as vb
    run_golden_cases(vb, [(tag, name, slice(None)) for tag, name in CASES])


@pytest.mark.gpu
def test_device_error_paths():
    import viamd_b200 as vb
    run_error_paths(vb)


@pytest.mark.gpu
def test_device_full_size_counts():
    """porosity(all) of 1ALA (all 6 golden frames) and of water_system(16) (12 288 atoms, 512^3 grids): occupied voxels voxel for voxel"""
    import viamd_b200 as vb
    g = load_golden("porosity.npz")
    run_golden_cases(vb, [("ala", "pa", slice(None))])
    n, seed, F = 16, 5, 3
    base, L = vb.synth_water_base(n, seed); frames = vb.synth_water_frames_host(n, seed, base, 0, F)
    radius = np.tile(g["wx_radius"][:3], n ** 3); idx = np.arange(3 * n ** 3, dtype=np.int32)
    want = restated(frames, radius, idx, [O.UnitCell.ortho(L, L, L)] * F)
    assert all(w["n"] > 1 << 26 for w in want)
    check_against(*run_case(vb, frames, vb.UnitCell.from_basis(L, L, L), radius, idx), want)


@pytest.mark.gpu
def test_device_non_prefix_selection():
    """element('O') is not a prefix of the atoms: the reference reads its radius array out of bounds there; the library uses each atom's own radius,
    as the restatement does"""
    import viamd_b200 as vb
    g = load_golden("porosity.npz"); frames = g["wx_frames"]; F = len(frames)
    s = vb.water_system(6); (p,) = vb.compile_script("o = porosity(element('O'));", s)
    want = restated(frames, g["wx_radius"], p.idx[0], [ocell(g, "wx", f) for f in range(F)])
    check_against(*run_case(vb, frames, vcells(vb, g, "wx", range(F)), g["wx_radius"], p.idx[0]), want)


@pytest.mark.gpu
def test_device_batches_and_ingest_modes():
    """40 frames (5 sub-batches of 8 in one batch; and batches of 12, which end inside a sub-batch), compact and whole-frame host ingest"""
    import viamd_b200 as vb
    g = load_golden("porosity.npz"); base = g["wx_frames"]; F = 40
    rng = np.random.default_rng(11)
    frames = (base[np.arange(F) % 4].astype(np.float64) + rng.normal(0.0, 0.2, (F,) + base.shape[1:])).astype(np.float32)
    cells = [vb.UnitCell(*(float(v) for v in g["wx_cells"][f % 4]), int(g["wx_flags"][f % 4])) for f in range(F)]
    want = restated(frames, g["wx_radius"], g["wx_px_idx"], [ocell(g, "wx", f % 4) for f in range(F)])
    for mode, bf in ((0, 0), (1, 0), (0, 12)):
        d, s, N = run_case(vb, frames, cells, g["wx_radius"], g["wx_px_idx"], ingest_mode=mode, batch_frames=bf)
        check_against(d, s, N, want)


@pytest.mark.gpu
def test_device_frames_in_hbm():
    """mdgpu_eval_device_frames on frames already in device memory, over two calls"""
    import viamd_b200 as vb
    g = load_golden("porosity.npz"); frames = np.ascontiguousarray(g["wx_frames"]); F, _, n = frames.shape
    d_xyz = vb.device_alloc(0, frames.nbytes)
    try:
        vb.memcpy_h2d(0, d_xyz, frames.ctypes.data, frames.nbytes)
        plan = vb.Plan(vb.System(n, np.ones(n, np.float32), radius=g["wx_radius"]), [vb.porosity("p", g["wx_pa_idx"]), vb.porosity("q", g["wx_px_idx"])], F)
        cells = vcells(vb, g, "wx", range(F))
        plan.eval_device_frames(d_xyz, 3 * n, n, cells[:1], 0, 1)
        plan.eval_device_frames(d_xyz + 4 * 3 * n, 3 * n, n, cells[1:], 1, F - 1)
        assert np.array_equal(plan.property_data("p").values, g["wx_pa_values"]) and np.array_equal(plan.property_data("q").values, g["wx_px_values"])
        plan.close()
    finally:
        vb.device_free(0, d_xyz)
