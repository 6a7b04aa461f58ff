"""Secondary structure per frame on the device (MDGPU_OP_SECONDARY_STRUCTURE / mdgpu_plan_secondary_structure): md_util_backbone_secondary_structure_infer
(md_util.c:2552 -> dssp() :2047-2550), the second call of VIAMD's backbone pass.

The reference is tests/golden/dssp.npz (tests/golden/make_golden_dssp.py): the unmodified reference's rows for 1LAF (as read, jittered, with explicit HN
atoms, in a periodic orthorhombic and a triclinic cell straddling the boundary, without a cell, cut into short ranges) and for tubulin-A-B. The CPU
tests run the plain-C restatement (oracle/md_dssp.c) and the whole C ABI of the emulated library (tests/emul); the GPU tests the library on the device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import dssp_oracle as D
import oracle_lib as O
from helpers import load_golden

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul"))


def cases():
    g = load_golden("dssp.npz")
    return g, [str(c) for c in g["cases"]]


def case(g, c):
    return g[f"{c}_atoms"], g[f"{c}_range_off"], g[f"{c}_xyz"], g[f"{c}_cells"], g[f"{c}_flags"], g[f"{c}_ss"]


def ss_plan(vb, atoms, ro, n, F, **kw):
    return vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.secondary_structure("ss", atoms, ro)], F, **kw)


def run_golden(vb, batch_frames=None, device_frames=False):
    g, names = cases()
    for c in names:
        atoms, ro, xyz, cells, flags, want = case(g, c)
        F, n = xyz.shape[0], xyz.shape[2]
        plan = ss_plan(vb, atoms, ro, n, F, **({"batch_frames": batch_frames} if batch_frames else {}))
        cell = vb.UnitCell(*(float(v) for v in cells[0]), int(flags[0]))
        if device_frames:
            import torch
            d = torch.from_numpy(np.ascontiguousarray(xyz)).cuda()
            plan.eval_device_frames(d.data_ptr(), 3 * n, n, cell, 0, F)
            torch.cuda.synchronize()
        else:
            plan.eval_host_frames(xyz, cell, 0)
        got = plan.secondary_structure("ss")
        bad = np.argwhere(got != want)
        assert not len(bad), f"{c}: {len(bad)} segments differ, first (frame, segment) {tuple(bad[0])}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"
        vals = plan.property_data("ss").values.reshape(F, -1)
        assert np.array_equal(vals, want.astype(np.float32))
        plan.close()


def run_errors(vb):
    g, _ = cases()
    atoms, ro, xyz, cells, flags, _ = case(g, "tub")
    n = xyz.shape[2]
    bad = [(np.zeros((0, 5), np.int32), [0], "no backbone segments"),
           (np.where(np.arange(atoms.size).reshape(atoms.shape) == 7, n + 3, atoms), ro, "atom index out of range"),
           (np.where(np.arange(atoms.size).reshape(atoms.shape) == 1, -1, atoms), ro, "atom index out of range"),
           (atoms, np.array([0, 433, 38, 477, 791, 865]), "not ascending"),
           (atoms, np.array([0, 38, 433, 477, 791, 864]), "start at 0 and end at the segment count"),
           (atoms, np.array([1, 38, 433, 477, 791, 865]), "start at 0 and end at the segment count")]
    for a, r, why in bad:
        with pytest.raises(vb.MdgpuError, match=why):
            ss_plan(vb, a, r, n, 2)
    plan = ss_plan(vb, atoms, ro, n, 2)
    for cell in (vb.UnitCell(20.0, 0, 0, 80.0, 0, 80.0, O.ORTHO | O.PBC_ALL), vb.UnitCell(80.0, 5.0, 0, 80.0, 0, 80.0, O.TRICLINIC | O.PBC_X)):
        with pytest.raises(vb.MdgpuError, match="secondary structure"):
            plan.eval_host_frames(xyz[:2], cell, 0)
    plan.close()
    other = vb.Plan(vb.System(4, np.ones(4, np.float32)), [vb.Property("d", vb.OP_DISTANCE, [np.array([0], np.int32), np.array([1], np.int32)])], 2)
    with pytest.raises(vb.MdgpuError, match="not a secondary-structure property"):
        other.secondary_structure("d")
    other.close()


def run_fetch_layout(vb):
    """the fetch call returns rows [frame_beg, frame_end) as int32 [frames][S]; frames not evaluated are 0 (unknown)"""
    g, _ = cases()
    atoms, ro, xyz, cells, flags, want = case(g, "laf")
    F, n = xyz.shape[0], xyz.shape[2]
    plan = ss_plan(vb, atoms, ro, n, F + 3)
    cell = vb.UnitCell(*(float(v) for v in cells[0]), int(flags[0]))
    plan.eval_host_frames(xyz[2:7], cell, 2)
    got = plan.secondary_structure("ss")
    assert got.dtype == np.int32 and got.shape == (F + 3, len(atoms))
    assert not np.any(got[:2]) and not np.any(got[7:]) and np.array_equal(got[2:7], want[2:7])
    assert np.array_equal(plan.secondary_structure("ss", 3, 5), want[3:5]) and plan.secondary_structure("ss", 4, 4).shape == (0, len(atoms))
    with pytest.raises(vb.MdgpuError):
        plan.secondary_structure("ss", 5, F + 4)
    import viamd_b200.api as api   # the raw 4-byte layout: frame f of the range at out + 4 * S * (f - frame_beg)
    raw = np.full(3 * len(atoms) + 1, -7, np.int32)
    api.lib().mdgpu_plan_secondary_structure.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]
    assert api.lib().mdgpu_plan_secondary_structure(plan._h, 0, 2, 5, raw.ctypes.data) == 0
    assert np.array_equal(raw[:-1].reshape(3, -1), want[2:5]) and raw[-1] == -7
    plan.close()


SHORT_RANGES = np.array([0, 1, 3, 6, 10, 15, 238], np.uint32)   # ranges of 1, 2, 3, 4, 5 and 223 segments over 1LAF's backbone


def run_short_ranges(vb):
    """ranges of 1 and 2 segments: the reference's backbone extraction never yields them, so the restatement is the yardstick. The 1LAF frames
    with their segments split into ranges of 1 .. 5 segments: range ends, estimated H of first segments, the neighbour exclusion across ends"""
    g, _ = cases()
    atoms, _, xyz, cells, flags, _ = case(g, "laf")
    F, n = xyz.shape[0], xyz.shape[2]
    want = []
    for f in range(F):
        rc, row = D.dssp(*xyz[f], O.UnitCell.from_params(*cells[f], int(flags[f])), atoms, SHORT_RANGES)
        assert rc == 0
        want.append(row)
    want = np.stack(want)
    plan = ss_plan(vb, atoms, SHORT_RANGES, n, F, batch_frames=5)
    plan.eval_host_frames(xyz, vb.UnitCell(*(float(v) for v in cells[0]), int(flags[0])), 0)
    got = plan.secondary_structure("ss")
    bad = np.argwhere(got != want)
    assert not len(bad), f"{len(bad)} segments differ, first (frame, segment) {tuple(bad[0])}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"
    plan.close()


@pytest.fixture
def emulated_library():   # per test: a module-scoped swap would still be active when the GPU tests below run
    import build_emul
    import viamd_b200.api as api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = build_emul.build_library(); api._lib = None
    import viamd_b200 as vb
    yield vb
    api.LIB_PATH, api._lib = saved


# ---------------------------------------------------------------------------------------------------------------------------- CPU
def test_restatement_equals_the_reference():
    g, names = cases()
    for c in names:
        atoms, ro, xyz, cells, flags, want = case(g, c)
        for f in range(xyz.shape[0]):
            cell = O.UnitCell.from_params(*cells[f], int(flags[f]))
            rc, got = D.dssp(*xyz[f], cell, atoms, ro)
            assert rc == 0 and np.array_equal(got, want[f]), (c, f, np.nonzero(got != want[f])[0][:10])


def test_restatement_rows_do_not_depend_on_bridge_order():
    """ladders are grown by exact-key lookup whatever `used` says: any order of the bridges gives the same sheet marks"""
    g, names = cases()
    for c in names:
        atoms, ro, xyz, cells, flags, want = case(g, c)
        cell = O.UnitCell.from_params(*cells[-1], int(flags[-1]))
        for seed in (1, 0x9E3779B97F4A7C15, 12345):
            rc, got = D.dssp(*xyz[-1], cell, atoms, ro, shuffle_seed=seed)
            assert rc == 0 and np.array_equal(got, want[-1]), (c, seed)


def test_generator_recorded_the_temporary_memory_hazard():
    g, names = cases()
    for c in names:
        assert bool(g[f"{c}_reverse_equal"]) and bool(g[f"{c}_prefill_differs"]), c


def test_restatement_rejects_malformed_input_and_narrow_cells():
    g, _ = cases()
    atoms, ro, xyz, cells, flags, _ = case(g, "laf")
    cell = O.UnitCell.from_params(*cells[0], int(flags[0]))
    assert D.dssp(*xyz[0], cell, atoms, [0, 100])[0] == -1 and D.dssp(*xyz[0], cell, atoms, [0, 200, 100, 238])[0] == -1
    assert D.dssp(*xyz[0], O.UnitCell.ortho(20.0, 80.0, 80.0), atoms, ro)[0] == -3


def test_emulated_library_equals_the_reference(emulated_library):
    run_golden(emulated_library)


def test_emulated_library_split_batches(emulated_library):
    run_golden(emulated_library, batch_frames=3)


def test_emulated_library_rejects_invalid_input(emulated_library):
    run_errors(emulated_library)


def test_emulated_library_fetch_layout(emulated_library):
    run_fetch_layout(emulated_library)


def test_emulated_library_short_ranges(emulated_library):
    run_short_ranges(emulated_library)


# ---------------------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_device_equals_the_reference_host_frames():
    import viamd_b200 as vb
    run_golden(vb)
    run_golden(vb, batch_frames=7)


@pytest.mark.gpu
def test_device_equals_the_reference_device_frames():
    import viamd_b200 as vb
    run_golden(vb, device_frames=True)
    run_golden(vb, batch_frames=7, device_frames=True)


@pytest.mark.gpu
def test_device_rejects_invalid_input():
    import viamd_b200 as vb
    run_errors(vb)


@pytest.mark.gpu
def test_device_short_ranges():
    import viamd_b200 as vb
    run_short_ranges(vb)


@pytest.mark.gpu
def test_device_fetch_layout():
    import viamd_b200 as vb
    run_fetch_layout(vb)


@pytest.mark.gpu
def test_device_backbone_pass_in_one_plan():
    """VIAMD's backbone pass as one plan: angles and secondary structure over the same frames, each equal to its own single-property plan"""
    import viamd_b200 as vb
    g, _ = cases()
    atoms, ro, xyz, cells, flags, want = case(g, "tub")
    F, n = xyz.shape[0], xyz.shape[2]
    five = np.full((len(atoms), 5), -1, np.int32)
    for r in range(len(ro) - 1):
        b, e = int(ro[r]), int(ro[r + 1])
        if e - b < 4: continue
        for i in range(b + 1, e - 1):
            five[i] = [atoms[i - 1, 2], atoms[i, 0], atoms[i, 1], atoms[i, 2], atoms[i + 1, 0]]
    cell = vb.UnitCell(*(float(v) for v in cells[0]), int(flags[0]))
    both = vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.backbone_angles("bb", five), vb.secondary_structure("ss", atoms, ro)], F, batch_frames=2)
    both.eval_host_frames(xyz, cell, 0)
    alone = vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.backbone_angles("bb", five)], F, batch_frames=2)
    alone.eval_host_frames(xyz, cell, 0)
    assert np.array_equal(both.secondary_structure("ss"), want)
    assert np.array_equal(both.property_data("bb").values, alone.property_data("bb").values)
    both.close(); alone.close()
