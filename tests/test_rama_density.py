"""Ramachandran density maps on the device (mdgpu_plan_rama_density / Plan.rama_density): VIAMD's rama_rep_compute_density
(src/components/ramachandran/ramachandran.cpp:1277-1370) over the (phi, psi) rows a backbone-angles property keeps in HBM.

The reference is tests/golden/rama.npz (tests/golden/make_golden_rama.py): the density task run by the unmodified reference's own blur on 64 jittered frames
of 1LAF. Maps are compared value for value through their digest (-0 taken as +0, the one difference the contract allows) and a stored sample.
The CPU tests run the numpy restatement (tests/rama_oracle.py) and the whole C ABI of the emulated library (tests/emul); the GPU tests the
library on the device."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

import rama_oracle as O
from helpers import load_golden

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul"))

SAMPLE = 17   # make_golden_rama.RAMA_SAMPLE


def digest(tex):
    return hashlib.sha256((np.ascontiguousarray(tex, np.float32) + np.float32(0)).tobytes()).hexdigest()


def assert_map(tex, g, k):
    assert tex.shape == (512, 512, 4) and tex.dtype == np.float32
    got = tex.ravel()[::SAMPLE]; want = g[f"tex{k}_sample"]
    bad = np.nonzero(got != want)[0]
    assert not len(bad), f"case {k}: {len(bad)} sampled values differ, first at flat index {bad[0] * SAMPLE}: {got[bad[0]]!r} vs {want[bad[0]]!r}"
    assert digest(tex) == str(g[f"tex{k}_sha256"]), f"case {k}: the map differs outside the stored sample"


def classes(g):
    off = g["class_off"]
    return [g["seg"][off[c]:off[c + 1]] for c in range(4)]


def angles_plan(vb, five, F, num_atoms=None):
    """a plan with one backbone-angles property `bb` over the segments of `five` [nseg, 5]"""
    n = int(num_atoms or (five.max() + 1))
    return vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.backbone_angles("bb", five)], F)


def inject(vb, plan, angles, done=None):
    """write angles [F, nseg, 2] into the property's rows on the device and declare the frames of `done` (all by default) evaluated"""
    import viamd_b200.api as api
    ptr, nbytes, _ = plan.accum_ptr("bb"); a = np.ascontiguousarray(angles, np.float32)
    assert nbytes == a.nbytes
    api.lib().mdgpu_memcpy_h2d.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]
    assert api.lib().mdgpu_memcpy_h2d(plan.device, ptr, a.ctypes.data, a.nbytes) == 0
    for f in (range(a.shape[0]) if done is None else done): plan.mark_frames_done(int(f), 1)


def golden_plan(vb):
    g = load_golden("rama.npz"); F = g["angles"].shape[0]
    plan = angles_plan(vb, g["five"], F, num_atoms=g["base"].shape[1])
    inject(vb, plan, g["angles"])
    return g, plan


def run_golden_cases(vb):
    g, plan = golden_plan(vb)
    for k, ((beg, end), sigma) in enumerate(zip(g["cases"], g["sigmas"])):
        tex, sums = plan.rama_density("bb", classes(g), int(beg), int(end), float(sigma))
        assert np.array_equal(sums, g[f"sums{k}"]), (k, sums, g[f"sums{k}"])
        assert_map(tex, g, k)
    plan.close()


def run_error_paths_and_edges(vb):
    g, plan = golden_plan(vb)
    cls = classes(g)
    for kw in (dict(frame_beg=5, frame_end=4), dict(frame_end=65), dict(sigma=0.09), dict(sigma=10.5), dict(sigma=float("nan"))):
        with pytest.raises(vb.MdgpuError):
            plan.rama_density("bb", cls, **kw)
    with pytest.raises(vb.MdgpuError, match="out of range"):
        plan.rama_density("bb", [cls[0], cls[1], cls[2], np.array([238], np.uint32)])
    tex, sums = plan.rama_density("bb", [cls[0], [], cls[2], cls[3]], 0, 64, 5.0)      # an empty class: zero channel, zero sum
    assert sums[1] == 0 and np.all(tex[..., 1] == 0) and sums[0] > 0 and np.all(tex[..., [0, 2, 3]].sum(axis=(0, 1)) > 0)
    want, wsums = O.rama_density(g["angles"], np.concatenate([cls[0], cls[2], cls[3]]).astype(np.uint32),
                                 np.cumsum([0, len(cls[0]), 0, len(cls[2]), len(cls[3])]), range(64), 5.0)
    assert np.array_equal(tex, want) and np.array_equal(sums, wsums)
    tex, sums = plan.rama_density("bb", cls, 30, 30, 5.0)                               # an empty frame range: nothing at all
    assert not np.any(tex) and not np.any(sums)
    import viamd_b200.api as api                                                         # class offsets that decrease, through the C ABI itself
    seg = np.zeros(4, np.uint32); off = np.array([0, 3, 2, 4, 4], np.uint32)
    assert api.lib().mdgpu_plan_rama_density(plan._h, 0, seg.ctypes.data, off.ctypes.data, 0, 64, 5.0, tex.ctypes.data, sums.ctypes.data) == -1
    plan.close()
    other = vb.Plan(vb.System(4, np.ones(4, np.float32)), [vb.Property("d", vb.OP_DISTANCE, [np.array([0], np.int32), np.array([1], np.int32)])], 2)
    with pytest.raises(vb.MdgpuError, match="not a backbone-angles property"):
        other.rama_density("d", [[0], [], [], []])
    other.close()


def run_unevaluated_frame(vb):
    """a frame of the range whose mask bit is not set contributes nothing (as mdgpu_plan_property_histogram counts only evaluated frames)"""
    g = load_golden("rama.npz"); F = g["angles"].shape[0]
    plan = angles_plan(vb, g["five"], F, num_atoms=g["base"].shape[1])
    inject(vb, plan, g["angles"], done=[f for f in range(F) if f != 11])
    tex, sums = plan.rama_density("bb", classes(g), 0, 24, 5.0)
    want, wsums = O.rama_density(g["angles"], g["seg"], g["class_off"], [f for f in range(24) if f != 11], 5.0)
    assert np.array_equal(tex, want) and np.array_equal(sums, wsums) and sums[0] == 23 * 204
    plan.close()


def run_texel_edges(vb):
    """phi / psi = -pi (float) sits a hair below u = 0 and truncates into texel 0, +pi gives u = 1 and wraps to texel 0; the neighbours of the edges"""
    pi = np.float32(np.pi); lo, hi = np.nextafter(-pi, np.float32(0)), np.nextafter(pi, np.float32(0))
    rows = np.array([[-pi, -pi], [pi, pi], [lo, hi], [hi, lo], [np.float32(0), -pi], [-pi, np.float32(0)], [np.float32(0), np.float32(0)]], np.float32)
    S = len(rows); five = np.tile(np.arange(5, dtype=np.int32), (S, 1))
    plan = angles_plan(vb, five, 1, num_atoms=5)
    inject(vb, plan, rows.reshape(1, S, 2))
    seg = np.arange(S, dtype=np.uint32)
    tex, sums = plan.rama_density("bb", [seg[:2], seg[2:4], seg[4:5], seg[5:]], 0, 1, 0.1)
    want, wsums = O.rama_density(rows.reshape(1, S, 2), seg, [0, 2, 4, 5, S], [0], 0.1)
    assert np.array_equal(sums, [2, 2, 1, 1]) and np.array_equal(sums, wsums) and np.array_equal(tex, want)
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
def test_box_radii_of_the_slider_range():
    assert O.rama_box_radii(5.0) == [9, 9, 11] and O.rama_box_radii(0.1) == [1, 1, 1] and O.rama_box_radii(10.0) == [19, 19, 21]
    assert max(max(O.rama_box_radii(s)) for s in np.linspace(0.1, 10.0, 100)) < 256


def test_texel_edges():
    """phi = -pi (float) lands slightly below u = 0 and truncates to texel 0; phi = pi (float) gives u = 1 and wraps to 0"""
    pi = np.float32(np.pi)
    assert O.rama_texel(-pi) == 0 and O.rama_texel(pi) == 0 and O.rama_texel(np.float32(0)) == 256
    assert O.rama_texel(np.nextafter(-pi, np.float32(0))) == 0


def test_numpy_restatement_equals_the_reference():
    g = load_golden("rama.npz")
    for k, ((beg, end), sigma) in enumerate(zip(g["cases"], g["sigmas"])):
        tex, sums = O.rama_density(g["angles"], g["seg"], g["class_off"], range(beg, end), sigma)
        assert np.array_equal(sums, g[f"sums{k}"])
        assert_map(tex, g, k)


def test_emulated_library_equals_the_reference(emulated_library):
    run_golden_cases(emulated_library)


def test_emulated_library_error_paths_and_edges(emulated_library):
    run_error_paths_and_edges(emulated_library)


def test_emulated_library_skips_unevaluated_frames(emulated_library):
    run_unevaluated_frame(emulated_library)


def test_emulated_library_texel_edges(emulated_library):
    run_texel_edges(emulated_library)


def test_emulated_library_two_device_plan(emulated_library, monkeypatch):
    """a plan over two devices evaluates the 1LAF frames in two blocks; the call reduces the rows onto devices[0] (its sync) and gives the
    one-device plan's map, which is the numpy restatement of the evaluated angles"""
    import build_emul
    monkeypatch.setenv("MDGPU_EMUL_DEVICES", "2"); monkeypatch.setenv("MDGPU_NCCL_LIB", build_emul.build_fake_nccl())
    vb = emulated_library; g = load_golden("rama.npz"); F = 8; n = g["base"].shape[1]
    frames = (g["base"][None].astype(np.float64) + np.random.default_rng(int(g["seed"])).normal(0.0, float(g["jitter"]), (F,) + g["base"].shape)).astype(np.float32)
    cell = vb.UnitCell(*(float(v) for v in g["cell"]), int(g["cell_flags"]))
    out = []
    for devices in (None, [0, 1]):
        plan = vb.Plan(vb.System(n, np.ones(n, np.float32)), [vb.backbone_angles("bb", g["five"])], F, devices=devices)
        plan.eval_host_frames(frames, cell, 0)
        out.append(plan.rama_density("bb", classes(g), 1, F, 5.0) + (plan.property_data("bb").values.reshape(F, -1, 2),))
        plan.close()
    (t1, s1, a1), (t2, s2, a2) = out
    want, wsums = O.rama_density(a1, g["seg"], g["class_off"], range(1, F), 5.0)
    assert np.array_equal(a1, a2) and np.array_equal(t1, t2) and np.array_equal(s1, s2) and np.array_equal(t1, want) and np.array_equal(s1, wsums)


# ---------------------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_device_equals_the_reference():
    import viamd_b200 as vb
    run_golden_cases(vb)


@pytest.mark.gpu
def test_device_error_paths_and_edges():
    import viamd_b200 as vb
    run_error_paths_and_edges(vb)


@pytest.mark.gpu
def test_device_skips_unevaluated_frames():
    import viamd_b200 as vb
    run_unevaluated_frame(vb)


@pytest.mark.gpu
def test_device_texel_edges():
    import viamd_b200 as vb
    run_texel_edges(vb)


@pytest.mark.gpu
def test_device_angles_to_density_end_to_end():
    """1LAF frames through MDGPU_OP_BACKBONE_ANGLES on the device, then the density from the rows left in HBM: equal to the numpy restatement of
    the device's own angles (a last-ulp atan2f difference may move a sample across a texel edge, so the golden map is not the yardstick here)"""
    import viamd_b200 as vb
    g = load_golden("rama.npz"); F = 48
    rng = np.random.default_rng(int(g["seed"]))                                        # make_golden.rama_frames: the golden's first 48 frames
    frames = (g["base"][None].astype(np.float64) + rng.normal(0.0, float(g["jitter"]), (F,) + g["base"].shape)).astype(np.float32)
    plan = angles_plan(vb, g["five"], F, num_atoms=g["base"].shape[1])
    cell = vb.UnitCell(*(float(v) for v in g["cell"]), int(g["cell_flags"]))
    plan.eval_host_frames(frames, cell, 0)
    ang = plan.property_data("bb").values.reshape(F, -1, 2)
    np.testing.assert_allclose(ang, g["angles"][:F], rtol=1e-5, atol=2e-6)
    for beg, end, sigma in ((0, F, 5.0), (7, 29, 0.1), (3, 44, 10.0)):
        tex, sums = plan.rama_density("bb", classes(g), beg, end, sigma)
        want, wsums = O.rama_density(ang, g["seg"], g["class_off"], range(beg, end), sigma)
        assert np.array_equal(sums, wsums) and np.array_equal(tex, want), (beg, end, sigma)
    plan.close()


@pytest.mark.gpu
def test_device_texel_saturates_at_2_pow_24():
    """70 000 frames x 256 identical segments put 17 920 000 samples into one texel: the reference's float `+= 1.0f` stops at 2^24"""
    import viamd_b200 as vb
    F, S = 70000, 256
    five = np.tile(np.arange(5, dtype=np.int32), (S, 1))
    plan = angles_plan(vb, five, F, num_atoms=5)
    row = np.tile(np.array([-1.1, -0.75], np.float32), S)           # a helix texel
    inject(vb, plan, np.broadcast_to(row, (F, 2 * S)).reshape(F, S, 2))
    seg = np.arange(S, dtype=np.uint32)
    tex, sums = plan.rama_density("bb", [seg, [], [], []], 0, F, 0.1)
    assert sums[0] == np.float32(F * S) and not np.any(sums[1:])
    counts, n = O.rama_counts(row.reshape(1, S, 2), seg, [0, S, S, S, S], [0])
    assert n[0] == S and counts[0].max() == S
    spike = (counts[0] > 0).astype(np.float32) * np.float32(1 << 24)
    want = O.rama_blur(np.stack([spike, 0 * spike, 0 * spike, 0 * spike]), 0.1)
    assert np.array_equal(tex, want)
    unsaturated = O.rama_blur(np.stack([(counts[0] > 0).astype(np.float32) * np.float32(F * S), 0 * spike, 0 * spike, 0 * spike]), 0.1)
    assert not np.array_equal(tex, unsaturated)
    plan.close()
