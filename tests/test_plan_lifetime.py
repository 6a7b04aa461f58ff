"""The plan's host-side bookkeeping, on the emulated library (tests/emul): no GPU, no nvcc build.

- Plan creation rejects malformed CSR offsets with the same messages at every site that takes them (groups of distance_pair, arrays of
  selections as arguments, rdf centre-of-mass references and target groups, shape_weights, contact_count sets).
- A device allocation that fails while a plan builds its stream slots or an XTC input stage leaves no half-built state behind: the call
  reports MDGPU_ERR_CUDA, the next call builds again and gives the results of a fresh plan, and destroying the plan frees everything once.
  Failures come from `emul_fail_malloc_after`, which a copy of the emulated library, relinked in a temporary directory, wraps around the
  allocations of tests/emul/fake_cudart.cpp. Each case runs in a child process, so that a plan that enqueues kernels on null buffers shows
  up as a dead child, not a dead test session.
"""
import ctypes as C
import json
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MDGPU_ERR_CUDA = -2


@pytest.fixture(scope="module")
def emulated_library():
    sys.path.insert(0, os.path.join(HERE, "emul"))
    import build_emul
    return build_emul.build_library()


# tests/emul/fake_cudart.cpp with an allocation-failure switch: after `n` more successful cudaMalloc / cudaMallocHost calls every further one
# fails, -1 lets them all succeed again; the call returns what was left of the previous budget, so a large budget also counts allocations
FAILING_CUDART = r"""
#include <cuda_runtime.h>
#define cudaMalloc emul_plain_cudaMalloc
#define cudaMallocHost emul_plain_cudaMallocHost
#include "fake_cudart.cpp"
#undef cudaMalloc
#undef cudaMallocHost
static long g_budget = -1;
static bool allowed() { if (g_budget == 0) return false; if (g_budget > 0) --g_budget; return true; }
extern "C" {
long emul_fail_malloc_after(long n) { const long left = g_budget; g_budget = n < 0 ? -1 : n; return left; }
cudaError_t cudaMalloc(void** p, size_t n) { if (!allowed()) { *p = nullptr; return cudaErrorMemoryAllocation; } return emul_plain_cudaMalloc(p, n); }
cudaError_t cudaMallocHost(void** p, size_t n) { if (!allowed()) { *p = nullptr; return cudaErrorMemoryAllocation; } return emul_plain_cudaMallocHost(p, n); }
}
"""


@pytest.fixture(scope="module")
def failing_library(emulated_library, tmp_path_factory):
    """the objects of the emulated library linked with FAILING_CUDART instead of fake_cudart.o, in a temporary directory"""
    import build_emul
    asan = ["-fsanitize=address", "-g"] if os.environ.get("MDGPU_EMUL_ASAN") else []
    objs = sorted(glob.glob(os.path.join(build_emul.HERE, "build", "asan" if asan else "", "*_emullib.o")))
    assert len(objs) >= 10, objs
    out = tmp_path_factory.mktemp("failing_library")
    src, obj, lib = out / "failing_cudart.cpp", out / "failing_cudart.o", str(out / "libmdgpu_emul_failing.so")
    src.write_text(FAILING_CUDART)
    subprocess.check_call(["g++", "-std=c++20", "-O2", "-fPIC", "-w", f"-I{build_emul.CUDA_INC}", f"-I{build_emul.HERE}", *asan, "-c", str(src), "-o", str(obj)])
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", lib, *objs, str(obj), "-lpthread", "-lm", "-ldl", *asan[:1]])
    return lib


# ----------------------------------------------------------------------------------------------------------------- offset validation
def _p(op, idx, **kw):
    from viamd_b200 import api
    return api.Property("p", op, [np.asarray(a, np.int32) for a in idx], **kw)


def _u32(*v):
    return np.array(v, np.uint32)


def _null_arg_offsets(d):
    d.arg_offsets[0] = None


def _null_target_groups(d):
    d.structure_offsets_b = None; d.num_structures_b = 2


def _validation_cases():
    """(id, property, descriptor edit or None, last_error)"""
    from viamd_b200 import api as A
    ab = ([0, 1, 2, 3, 4, 5], [6, 7, 8, 9])
    ref6 = [0, 1, 2, 3, 4, 5]
    cases = []
    # distance_pair: argument 0 / 1 as arrays of selections (take_groups)
    for tag, kw in (("short", dict(structure_offsets=_u32(0, 3, 5))), ("late_start", dict(structure_offsets=_u32(1, 3, 6))),
                    ("missing", dict()), ("short_b", dict(structure_offsets_b=_u32(0, 2, 3)))):
        cases.append((f"groups_{tag}", _p(A.OP_DISTANCE_PAIR, ab, num_structures=0 if tag == "short_b" else 2, **kw), None,
                      "'p': group offsets do not cover the index list"))
    cases.append(("groups_decreasing", _p(A.OP_DISTANCE_PAIR, ab, num_structures=3, structure_offsets=_u32(0, 4, 3, 6)), None,
                  "'p': group offsets must be non-decreasing"))
    # distance: argument 0 as an array of selections (take_arg_parts)
    dist = ([0, 1, 2], [5])
    cases += [("args_short", _p(A.OP_DISTANCE, dist, arg_offsets={0: _u32(0, 1, 2)}), None, "'p': argument offsets do not cover the index list"),
              ("args_missing", _p(A.OP_DISTANCE, dist, arg_offsets={0: _u32(0, 1, 3)}), _null_arg_offsets, "'p': argument offsets do not cover the index list"),
              ("args_decreasing", _p(A.OP_DISTANCE, dist, arg_offsets={0: _u32(0, 2, 1, 3)}), None, "'p': argument offsets must be non-decreasing")]
    # rdf target groups
    rdf = dict(cutoff_max=5.0)
    cases += [("rdf_targets_short", _p(A.OP_RDF, ab, structure_offsets_b=_u32(0, 2, 3), **rdf), None, "rdf 'p': target group offsets do not cover idx[1]"),
              ("rdf_targets_missing", _p(A.OP_RDF, ab, **rdf), _null_target_groups, "rdf 'p': target group offsets do not cover idx[1]"),
              ("rdf_targets_decreasing", _p(A.OP_RDF, ab, structure_offsets_b=_u32(0, 3, 2, 4), **rdf), None, "rdf 'p': target group offsets must be non-decreasing")]
    # structure offsets (given, or num_structures runs of structure_size atoms) of rdf, shape_weights and contact_count
    for site, op, idx, kw, who in (("rdf", A.OP_RDF, ab, rdf, "rdf 'p'"), ("shape", A.OP_SHAPE_WEIGHTS, (ref6,), {}, "'p'"),
                                   ("contact", A.OP_CONTACT_COUNT, ab, dict(cutoff_max=3.0), "'p'")):
        cases += [(f"{site}_structures_short", _p(op, idx, num_structures=2, structure_offsets=_u32(0, 3, 5), **kw), None, f"{who}: structure offsets do not cover idx[0]"),
                  (f"{site}_structures_late_start", _p(op, idx, num_structures=2, structure_offsets=_u32(1, 3, 6), **kw), None, f"{who}: structure offsets do not cover idx[0]"),
                  (f"{site}_structures_decreasing", _p(op, idx, num_structures=3, structure_offsets=_u32(0, 4, 2, 6), **kw), None, f"{who}: structure offsets must be non-decreasing"),
                  (f"{site}_structures_missing_size", _p(op, idx, num_structures=2, **kw), None, f"{who}: structure_size or structure_offsets required"),
                  (f"{site}_structure_size_short", _p(op, idx, num_structures=2, structure_size=2, **kw), None, f"{who}: structure offsets do not cover idx[0]")]
    return cases


def _create_error(api, prop, edit):
    """the error of mdgpu_plan_create for one property, with its descriptor edited on the way in (a null pointer the Python API never passes)"""
    L = api.lib()

    class Edit:
        def __getattr__(self, n): return getattr(L, n)

        def mdgpu_plan_create(self, sd, descs, n, F, o):
            if edit: edit(descs[0])
            return L.mdgpu_plan_create(sd, descs, n, F, o)
    api._lib = Edit()
    try:
        with pytest.raises(api.MdgpuError) as e:
            api.Plan(api.System(20, np.ones(20, np.float32)), [prop], 2)
    finally:
        api._lib = L
    return str(e.value)


def test_malformed_offsets_are_rejected_with_their_site_s_message(emulated_library):
    """Every offset site: offsets that do not start at 0 or end at the list size, decrease, are missing, or (structure_size) expand to the
    wrong length -> plan creation fails with exactly the message of that site."""
    from viamd_b200 import api
    saved = (api.LIB_PATH, api._lib)
    api.LIB_PATH = emulated_library; api._lib = None
    try:
        cases = _validation_cases()
        assert len(cases) == 26
        bad = []
        for cid, prop, edit, want in cases:
            got = _create_error(api, prop, edit)
            if got != want: bad.append(f"{cid}: {got!r} != {want!r}")
        assert not bad, "\n".join(bad)
    finally:
        api.LIB_PATH, api._lib = saved


# ----------------------------------------------------------------------------------------------------------------- allocation failures
SCRIPT = "r = rdf(element('O'), element('O'), 6.0); v = sdf(residue(1:20), element('O'), 5.0); d = distance(1,10);"
PLAN_OPTS = dict(batch_frames=3, num_streams=2)
BIG = 1 << 40


def _worker(lib_path, mode, n):
    """one case in this process; prints one JSON line. mode: slots | xtc; n < 0: only count the allocations of the first evaluation"""
    sys.path[:0] = [ROOT, HERE]
    from viamd_b200 import api
    api.LIB_PATH = lib_path; api._lib = None
    import viamd_b200 as vb
    from helpers import load_golden, golden_system, vb_system, vb_cell
    L = api.lib(); L.emul_fail_malloc_after.restype = C.c_long; L.emul_fail_malloc_after.argtypes = [C.c_long]
    g = load_golden("water6.npz"); sysm = vb_system(golden_system(g)); F = g["frames"].shape[0]
    cells = [vb_cell(g["cells"][f], g["cell_flags"][f]) for f in range(F)]
    x = load_golden("xtc_cases.npz"); blob = x["water6__xtc"]; offs, _ = vb.xtc_frame_offsets(blob)

    def new_plan():
        plan = vb.Plan(sysm, vb.compile_script(SCRIPT, sysm), F, **PLAN_OPTS)
        plan.set_initial_frame(*g["frames"][0], cells[0])
        return plan

    def evaluate(plan):
        if mode == "xtc": plan.eval_xtc_frames(blob, offs, 0)
        else: plan.eval_host_frames(g["frames"], cells, 0)

    def results(plan):
        return [plan.counts("r"), plan.counts("v"), plan.property_data("d").values.copy(), plan.frame_mask().copy()]

    plan = new_plan()
    if mode == "xtc":   # the slots exist already: the allocations of the XTC evaluation are the stage's (and the slots' decode buffers)
        plan.eval_host_frames(g["frames"], cells, 0); plan.clear()
    L.emul_fail_malloc_after(BIG if n < 0 else n)
    try:
        evaluate(plan); err = None
    except api.MdgpuError as e:
        err = str(e)
    left = L.emul_fail_malloc_after(-1)
    if n < 0:
        assert err is None, err
        print(json.dumps({"allocations": BIG - left})); plan.close()
        return 0
    assert err is not None and err.startswith(f"mdgpu error {MDGPU_ERR_CUDA}:"), err
    plan.clear()   # an XTC failure after the first batch leaves that batch's counts behind; a slot failure leaves nothing to clear
    evaluate(plan)
    fresh = new_plan(); evaluate(fresh)
    for a, b in zip(results(plan), results(fresh)):
        assert np.array_equal(a, b)
    plan.close(); fresh.close()
    print(json.dumps({"ok": True}))
    return 0


def _child(lib_path, mode, n):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--worker", lib_path, mode, str(n)]
    return subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)


def _allocations(lib_path, mode):
    r = _child(lib_path, mode, -1)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])["allocations"]


def _every_budget(lib_path, mode):
    total = _allocations(lib_path, mode)
    assert total > 0
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        runs = list(ex.map(lambda n: (n, _child(lib_path, mode, n)), range(total)))
    dead = [f"budget {n}: exit {r.returncode}\n{r.stderr[-1500:]}" for n, r in runs if r.returncode != 0]
    assert not dead, f"{len(dead)} of {total} cases failed\n" + "\n".join(dead[:3])


def test_failed_slot_build_is_retried_by_the_next_evaluation(failing_library):
    """rdf + sdf + distance on the golden water box, 2 stream slots: for every allocation of the first mdgpu_eval_host_frames (slots and host
    staging), failing there gives MDGPU_ERR_CUDA; the next evaluation of the same plan equals a fresh plan's, and the plan closes cleanly."""
    _every_budget(failing_library, "slots")


def test_failed_xtc_stage_set_up_is_retried_by_the_next_evaluation(failing_library):
    """As above for the allocations of mdgpu_eval_xtc_frames on a plan whose slots exist: the XTC stage's buffers and the slots' decode buffers."""
    _every_budget(failing_library, "xtc")


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "--worker":
    sys.exit(_worker(sys.argv[2], sys.argv[3], int(sys.argv[4])))
