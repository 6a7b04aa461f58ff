"""Temporal expressions on the synthetic water box water_system(32) (98 304 atoms) with the frames already in HBM:

  plain      : 64 distances d0 .. d63 between oxygens of water molecules far apart
  expressions: the same 64 distances and 64 expressions over them, e_k = abs(d_k - d_(k+1)) * 10 + sqrt(d_k) / 3 (a few operators and a function
               each, one dependency level)

Prints one JSON line (and writes it to --out when given): GPU name, power limit and SM clock read in this run; frames/s of both plans through
mdgpu_eval_device_frames (host clock around calls that end in a device synchronise, best and median of --repeat passes over --frames frames
after --warmup passes, the two plans alternating); and, from a torch.profiler pass of its own over the expression plan, the device time of
k_temporal_expr (one launch per batch) next to that of the distance kernel.

  python profiles/temporal_expr.py [--frames 1056] [--repeat 5] [--warmup 1] [--out profiles/temporal_expr_h100.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from range_selection import gpu_info  # noqa: E402

N_SIDE, SEED, NPROP = 32, 1234, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1056); ap.add_argument("--repeat", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import viamd_b200 as vb
    assert vb.device_count() > 0, "profiles/temporal_expr.py measures on a CUDA device"
    s = vb.water_system(N_SIDE); n = s.num_atoms; F = a.frames
    base, L = vb.synth_water_base(N_SIDE, SEED)
    dist = " ".join(f"d{k} = distance({3 * 97 * k + 1}, {3 * (97 * k + 5000) + 1});" for k in range(NPROP))
    expr = " ".join(f"e{k} = abs(d{k} - d{(k + 1) % NPROP}) * 10 + sqrt(d{k}) / 3;" for k in range(NPROP))
    info = {"gpu": gpu_info(), "system": f"water_system({N_SIDE})", "atoms": n, "frames": F, "repeat": a.repeat, "warmup": a.warmup,
            "plain": f"{NPROP} distances", "expressions": f"{NPROP} distances + {NPROP} x `e_k = abs(d_k - d_k+1) * 10 + sqrt(d_k) / 3`"}
    d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
    d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes)
    vb.synth_water_frames_device(0, N_SIDE, SEED, d_base, 0, F, d_xyz, 3 * n, n); vb.device_synchronize(0)
    cell = vb.UnitCell.from_basis(L, L, L)
    plans = {"plain": vb.Plan(s, vb.compile_script(dist, s), F), "expressions": vb.Plan(s, vb.compile_script(dist + " " + expr, s), F)}
    times = {k: [] for k in plans}
    for r in range(a.warmup + a.repeat):
        for k, plan in plans.items():
            plan.clear(); vb.device_synchronize(0)
            t0 = time.perf_counter(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); dt = time.perf_counter() - t0
            if r >= a.warmup: times[k].append(dt)
    for k, t in times.items():
        info[f"{k}_frames_per_s"] = {"best": F / min(t), "median": F / float(np.median(t))}
    info["expressions_over_plain"] = info["expressions_frames_per_s"]["best"] / info["plain_frames_per_s"]["best"]
    v = plans["expressions"]; want = np.abs(v.property_data("d0").values - v.property_data("d1").values) * np.float32(10) + np.sqrt(v.property_data("d0").values) / np.float32(3)
    info["e0_matches_host_arithmetic"] = bool(np.array_equal(v.property_data("e0").values, want))
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        v.clear(); v.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); v.sync(); torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        name = e.key.split("(")[0].split("::")[-1]
        if any(w in name for w in ("k_temporal_expr", "k_temporal")):
            dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            kt[name] = {"calls": e.count, "total_ms": dev / 1e3, "per_call_us": dev / max(e.count, 1)}
    info["kernels_expressions"] = kt
    for p in plans.values(): p.close()
    vb.device_free(0, d_xyz); vb.device_free(0, d_base)
    line = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f: f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
