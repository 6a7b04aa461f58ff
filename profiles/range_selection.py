"""rdf() of a coordinate-range selection against the same rdf() of a static selection of the same size, on the synthetic water box
water_system(32) (98 304 atoms) with the frames already in HBM:

  dynamic: rdf(element('O') and within_z(a:b), element('O'), 10.0)   a slab of about a quarter of the box, marked per frame on the device
  static : rdf(<the oxygens that slab holds in frame 0>, element('O'), 10.0)

Prints one JSON line (and writes it to --out when given): GPU name, power limit and SM clock read in this run; frames/s of both plans through
mdgpu_eval_device_frames (host clock around calls that end in a device synchronise, best and median of --repeat passes over --frames frames after
--warmup passes, the two plans alternating); and, from a torch.profiler pass of its own over the dynamic plan, the device time per batch of
k_range_mark (one call per batch), of the compaction k_within_compact and of the rdf kernels.

  python profiles/range_selection.py [--frames 528] [--repeat 5] [--warmup 1] [--out profiles/range_selection_h100.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_SIDE, SEED, CUTOFF = 32, 1234, 10.0


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        r = [s.strip() for s in out.strip().split(",")]
        return {"name": r[0], "power_limit_w": float(r[1]), "sm_clock_mhz": float(r[2]), "sm_max_mhz": float(r[3])}
    except Exception as e:
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=528); ap.add_argument("--repeat", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import viamd_b200 as vb
    assert vb.device_count() > 0, "profiles/range_selection.py measures on a CUDA device"
    s = vb.water_system(N_SIDE); n = s.num_atoms; F = a.frames
    base, L = vb.synth_water_base(N_SIDE, SEED)
    za, zb = 0.375 * L, 0.625 * L
    dyn_src = f"r = rdf(element('O') and within_z({za:.3f}:{zb:.3f}), element('O'), {CUTOFF});"
    dyn_props = vb.compile_script(dyn_src, s)
    f0 = vb.synth_water_frames_host(N_SIDE, SEED, base, 0, 1)[0]
    O = np.nonzero(np.asarray(s.element) == "O")[0].astype(np.int32)
    sel0 = np.nonzero(dyn_props[0].ranges[0].mask(*f0))[0].astype(np.int32)
    info = {"gpu": gpu_info(), "system": f"water_system({N_SIDE})", "atoms": n, "frames": F, "repeat": a.repeat, "warmup": a.warmup,
            "script": dyn_src, "slab_atoms_frame0": int(sel0.size), "oxygens": int(O.size)}
    d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
    d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes)
    vb.synth_water_frames_device(0, N_SIDE, SEED, d_base, 0, F, d_xyz, 3 * n, n); vb.device_synchronize(0)
    cell = vb.UnitCell.from_basis(L, L, L)
    plans = {"dynamic": vb.Plan(s, dyn_props, F), "static": vb.Plan(s, [vb.rdf("r", sel0, O, CUTOFF)], F)}
    times = {k: [] for k in plans}
    for r in range(a.warmup + a.repeat):
        for k, plan in plans.items():
            plan.clear(); vb.device_synchronize(0)
            t0 = time.perf_counter(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); dt = time.perf_counter() - t0
            if r >= a.warmup: times[k].append(dt)
    for k, t in times.items():
        info[f"{k}_frames_per_s"] = {"best": F / min(t), "median": F / float(np.median(t))}
    info["dynamic_over_static"] = info["dynamic_frames_per_s"]["best"] / info["static_frames_per_s"]["best"]
    import torch
    from torch.profiler import ProfilerActivity, profile
    plan = plans["dynamic"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.clear(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("::")[-1]
        if any(w in name for w in ("k_range_mark", "k_within_compact", "k_rdf")):
            dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kt[name] = {"calls": e.count, "total_ms": dev / 1e3, "per_call_us": dev / max(e.count, 1)}
    info["kernels_dynamic"] = kt
    for p in plans.values(): p.close()
    vb.device_free(0, d_xyz); vb.device_free(0, d_base)
    line = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f: f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
