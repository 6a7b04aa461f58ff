"""count(x, 'residue' | 'structure') of a per-frame within() selection against the one-argument count(x), on the synthetic water box
water_system(32) (98 304 atoms, 32 768 waters) with the frames already in HBM:

  residue  : n = count(within(3.5, residue(1:1000)), 'residue');
  structure: n = count(within(3.5, residue(1:1000)), 'structure');
  atom     : n = count(within(3.5, residue(1:1000)));

Prints one JSON line (and writes it to --out when given): GPU name, power limit and SM clock read in this run; frames/s of the three plans
through mdgpu_eval_device_frames (host clock around calls that end in a device synchronise, best and median of --repeat passes over --frames
frames after --warmup passes, the plans alternating); from a torch.profiler pass of its own over the 'residue' plan, the device time of
k_group_count, k_within_mark and the cell-list kernels; and, where oracle/_ref/ref_harness_fast exists, the reference's CPU
md_script_eval_frame_range on --ref-frames frames of the same box with 1 thread and with all cores.

  python profiles/group_count.py [--frames 528] [--repeat 5] [--warmup 1] [--ref-frames 64] [--out profiles/group_count_h100.json]
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
sys.path.insert(0, ROOT)

N_SIDE, SEED = 32, 1234
SCRIPTS = {"residue": "n = count(within(3.5, residue(1:1000)), 'residue');",
           "structure": "n = count(within(3.5, residue(1:1000)), 'structure');",
           "atom": "n = count(within(3.5, residue(1:1000)));"}


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
        gro = os.path.join(tmp, "s.gro")
        subprocess.check_call([synth, "water-gro", str(N_SIDE), str(SEED), gro], stdout=subprocess.DEVNULL)
        for k, script in SCRIPTS.items():
            for t in sorted({1, cpu_threads}):
                r = subprocess.run([harness, "time", "--sys", gro, "--traj", f"synthwater:{N_SIDE}:{SEED}:{F}", "--script", script, "--frames", f"0:{F}",
                                    "--threads", str(t), "--repeat", "2", "--warmup", "1"], capture_output=True, text=True, check=True)
                out[f"{k}_threads_{t}"] = json.loads(r.stdout.strip().splitlines()[-1])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=528); ap.add_argument("--repeat", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-frames", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import viamd_b200 as vb
    assert vb.device_count() > 0, "profiles/group_count.py measures on a CUDA device"
    s = vb.water_system(N_SIDE); n = s.num_atoms; F = a.frames
    base, L = vb.synth_water_base(N_SIDE, SEED)
    info = {"gpu": gpu_info(), "system": f"water_system({N_SIDE})", "atoms": n, "frames": F, "repeat": a.repeat, "warmup": a.warmup, "scripts": SCRIPTS}
    d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
    d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes)
    vb.synth_water_frames_device(0, N_SIDE, SEED, d_base, 0, F, d_xyz, 3 * n, n); vb.device_synchronize(0)
    cell = vb.UnitCell.from_basis(L, L, L)
    plans = {k: vb.Plan(s, vb.compile_script(src, s), F) for k, src in SCRIPTS.items()}
    times = {k: [] for k in plans}
    for r in range(a.warmup + a.repeat):
        for k, plan in plans.items():
            plan.clear(); vb.device_synchronize(0)
            t0 = time.perf_counter(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); dt = time.perf_counter() - t0
            if r >= a.warmup: times[k].append(dt)
    for k, t in times.items():
        info[f"{k}_frames_per_s"] = {"best": F / min(t), "median": F / float(np.median(t))}
    vals = {k: np.array(p.property_data("n").values) for k, p in plans.items()}
    info["values_first_frames"] = {k: v[:4].tolist() for k, v in vals.items()}
    info["residue_equals_structure"] = bool(np.array_equal(vals["residue"], vals["structure"]))   # every water is one residue and one structure
    import torch
    from torch.profiler import ProfilerActivity, profile
    plan = plans["residue"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.clear(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("::")[-1]
        if name.startswith("k_"):
            dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kt[name] = {"calls": e.count, "total_ms": dev / 1e3, "per_call_us": dev / max(e.count, 1)}
    info["kernels_residue"] = kt
    for p in plans.values(): p.close()
    vb.device_free(0, d_xyz); vb.device_free(0, d_base)
    info["reference_cpu"] = reference_times(a.ref_frames, os.cpu_count() or 1)
    info["reference_cpu_cores"] = os.cpu_count()
    line = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f: f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
