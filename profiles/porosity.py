"""porosity(all) on the synthetic water box water_system(16) (12 288 atoms; a 512^3-voxel grid per frame) with the frames already in HBM, against
the reference's CPU evaluation of the same script.

Prints one JSON line (and writes it to --out when given): GPU name and power limit read in this run; frames/s of mdgpu_eval_device_frames (host clock around
calls that end in a device synchronise, best and median of --repeat passes over --frames frames after --warmup passes); the device time per kernel
from a torch.profiler pass of its own; sphere-voxel tests per frame (the voxels of every sphere's clamped index box, from the plain-C restatement
oracle/md_porosity.c on the first frames) and tests/s; and, where oracle/_ref/ref_harness_fast exists (the reference built with its shipped flags),
its `time` mode on the same frames with one thread and with every core of this host.

  python profiles/porosity.py [--frames 264] [--repeat 5] [--warmup 1] [--ref-frames 16] [--out porosity_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

N_SIDE, SEED = 16, 2024
RADII = {"O": 1.52, "H": 1.1}   # the reference's van der Waals radii of the water atoms (md_atom_extract_radii; tests/golden/porosity.npz)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        r = [s.strip() for s in out.strip().split(",")]
        return {"name": r[0], "power_limit_w": float(r[1]), "sm_clock_mhz": float(r[2]), "sm_max_mhz": float(r[3])}
    except Exception as e:
        return {"error": str(e)}


def reference_times(F, cpu_threads):
    harness = os.path.join(ROOT, "oracle", "_ref", "ref_harness_fast"); synth = os.path.join(ROOT, "oracle", "build", "synth_tool")
    if not (os.path.exists(harness) and os.path.exists(synth)):
        return {"skipped": "oracle/_ref/ref_harness_fast not built"}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        gro = os.path.join(tmp, "w.gro"); subprocess.check_call([synth, "water-gro", str(N_SIDE), str(SEED), gro], stdout=subprocess.DEVNULL)
        for t in sorted({1, cpu_threads}):
            r = subprocess.run([harness, "time", "--sys", gro, "--traj", f"synthwater:{N_SIDE}:{SEED}:{F}", "--script", "p = porosity(all);",
                                "--frames", f"0:{F}", "--threads", str(t), "--repeat", "2", "--warmup", "1"], capture_output=True, text=True, check=True)
            out[f"threads_{t}"] = json.loads(r.stdout.strip().splitlines()[-1])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=264); ap.add_argument("--repeat", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-frames", type=int, default=16); ap.add_argument("--tests-frames", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import viamd_b200 as vb
    import oracle_lib as O
    import porosity_oracle as P
    info = {"gpu": gpu_info(), "system": f"water_system({N_SIDE})", "atoms": 3 * N_SIDE ** 3, "frames": a.frames, "repeat": a.repeat, "warmup": a.warmup}
    s = vb.water_system(N_SIDE); s.radius = np.array([RADII[e] for e in s.element], np.float32)
    base, L = vb.synth_water_base(N_SIDE, SEED); n = s.num_atoms; F = a.frames
    d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
    d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes)
    vb.synth_water_frames_device(0, N_SIDE, SEED, d_base, 0, F, d_xyz, 3 * n, n); vb.device_synchronize(0)
    cell = vb.UnitCell.from_basis(L, L, L)
    plan = vb.Plan(s, vb.compile_script("p = porosity(all);", s), F)
    times = []
    for r in range(a.warmup + a.repeat):
        plan.clear(); vb.device_synchronize(0)
        t0 = time.perf_counter(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); dt = time.perf_counter() - t0
        if r >= a.warmup: times.append(dt)
    vals = plan.property_data("p").values.copy()
    info["frames_per_s"] = {"best": F / min(times), "median": F / float(np.median(times))}
    info["call_s"] = times
    # occupied voxels and tests of the first frames from the restatement; the device's rows must agree
    frames = vb.synth_water_frames_host(N_SIDE, SEED, base, 0, a.tests_frames)
    ref = [P.porosity(fr[0], fr[1], fr[2], s.radius, np.arange(n, dtype=np.int32), O.UnitCell.ortho(L, L, L)) for fr in frames]
    ptr, nbytes, _ = plan.frame_rows("p", 0); occ = np.zeros(F, np.uint64); vb.memcpy_d2h(0, occ.ctypes.data, ptr, nbytes)
    info["check"] = {"values_equal": bool(all(vals[f] == r["value"] for f, r in enumerate(ref))), "occupied_equal": bool(all(int(occ[f]) == r["set"] for f, r in enumerate(ref)))}
    tests = float(np.mean([r["tests"] for r in ref])); info["tests_per_frame"] = tests; info["voxels_per_frame"] = float(np.mean([r["n"] for r in ref]))
    info["tests_per_s"] = tests * info["frames_per_s"]["best"]
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.clear(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        if "porosity" in e.key:
            dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kt[e.key.split("(")[0].split("::")[-1]] = {"calls": e.count, "total_ms": dev / 1e3, "per_frame_us": dev / F}
    info["kernels"] = kt
    plan.close(); vb.device_free(0, d_xyz); vb.device_free(0, d_base)
    info["reference_cpu"] = reference_times(a.ref_frames, os.cpu_count() or 1)
    for k, r in info["reference_cpu"].items():
        if isinstance(r, dict) and "frames_per_s" in r: info[f"speedup_vs_{k}"] = info["frames_per_s"]["best"] / r["frames_per_s"]
    line = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f: f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
