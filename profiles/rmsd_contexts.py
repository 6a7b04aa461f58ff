"""rmsd() inside `in` contexts: one fit per context and frame (k_rmsd_groups, one thread per group), with the frames already in HBM, against
the reference's CPU evaluation of the same scripts. Workloads:

  all      : r = rmsd(all) in residue(:);         water_system(32), 98 304 atoms: 32 768 contexts of 3 atoms
  first1k  : r = rmsd(all) in residue(1:1000);    the same box, 1 000 contexts
  lipids   : r = rmsd(all) in resname('LIP');     the synthetic membrane: one context per 12-bead lipid

Prints one JSON line (and writes it to --out when given): GPU name, power limit and SM clock read in this run; per workload the frames/s of
mdgpu_eval_device_frames (host clock around calls that end in a device synchronise, best and median of --repeat passes over --frames frames after
--warmup passes), fits/s, the device time of k_rmsd_groups from a torch.profiler pass of its own, and, where oracle/_ref/ref_harness_fast exists
(the reference built with its shipped flags), its `time` mode on the same frames with one thread and with every core of this host.

  python profiles/rmsd_contexts.py [--frames 264] [--repeat 5] [--warmup 1] [--ref-frames 8] [--out profiles/rmsd_contexts_h100.json]
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
MEMB = (64, 96, 4, 4321)   # 8 192 lipids of 12 beads + 73 728 solvent beads
WORKLOADS = {"all": ("water", "r = rmsd(all) in residue(:);"), "first1k": ("water", "r = rmsd(all) in residue(1:1000);"),
             "lipids": ("membrane", "r = rmsd(all) in resname('LIP');")}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        r = [s.strip() for s in out.strip().split(",")]
        return {"name": r[0], "power_limit_w": float(r[1]), "sm_clock_mhz": float(r[2]), "sm_max_mhz": float(r[3])}
    except Exception as e:
        return {"error": str(e)}


def reference_times(system, script, F, cpu_threads):
    harness = os.path.join(ROOT, "oracle", "_ref", "ref_harness_fast"); synth = os.path.join(ROOT, "oracle", "build", "synth_tool")
    if not (os.path.exists(harness) and os.path.exists(synth)):
        return {"skipped": "oracle/_ref/ref_harness_fast not built"}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        gro = os.path.join(tmp, "s.gro")
        if system == "water":
            subprocess.check_call([synth, "water-gro", str(N_SIDE), str(SEED), gro], stdout=subprocess.DEVNULL); traj = f"synthwater:{N_SIDE}:{SEED}:{F}"
        else:
            subprocess.check_call([synth, "membrane-gro", *map(str, MEMB), gro], stdout=subprocess.DEVNULL); traj = "synthmembrane:%d:%d:%d:%d:" % MEMB + str(F)
        for t in sorted({1, cpu_threads}):
            r = subprocess.run([harness, "time", "--sys", gro, "--traj", traj, "--script", script, "--frames", f"0:{F}", "--threads", str(t),
                                "--repeat", "2", "--warmup", "1"], capture_output=True, text=True, check=True)
            out[f"threads_{t}"] = json.loads(r.stdout.strip().splitlines()[-1])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=264); ap.add_argument("--repeat", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-frames", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import viamd_b200 as vb
    assert vb.device_count() > 0, "profiles/rmsd_contexts.py measures on a CUDA device"
    import torch
    from torch.profiler import ProfilerActivity, profile
    F = a.frames
    info = {"gpu": gpu_info(), "frames": F, "repeat": a.repeat, "warmup": a.warmup, "workloads": {}}
    for system in ("water", "membrane"):
        if system == "water":
            s = vb.water_system(N_SIDE); base, L = vb.synth_water_base(N_SIDE, SEED); n = s.num_atoms
            d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
            d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes); d_mol = None
            vb.synth_water_frames_device(0, N_SIDE, SEED, d_base, 0, F, d_xyz, 3 * n, n)
            cell = vb.UnitCell.from_basis(L, L, L); first = vb.synth_water_frames_host(N_SIDE, SEED, base, 0, 1)[0]
        else:
            s = vb.membrane_system(*MEMB[:3]); base, _, mol, L3 = vb.synth_membrane_base(*MEMB); n = s.num_atoms
            d_xyz = vb.device_alloc(0, 4 * 3 * n * F)
            d_base = vb.device_alloc(0, base.nbytes); vb.memcpy_h2d(0, d_base, base.ctypes.data, base.nbytes)
            d_mol = vb.device_alloc(0, mol.nbytes); vb.memcpy_h2d(0, d_mol, mol.ctypes.data, mol.nbytes)
            vb.synth_membrane_frames_device(0, *MEMB, d_base, d_mol, 0, F, d_xyz, 3 * n, n)
            cell = vb.UnitCell.from_basis(*L3); first = vb.synth_membrane_frames_host(*MEMB, base, mol, 0, 1)[0]
        vb.device_synchronize(0)
        for wl, (wsys, script) in WORKLOADS.items():
            if wsys != system: continue
            props = vb.compile_script(script, s); groups = props[0].num_structures
            plan = vb.Plan(s, props, F)
            plan.set_initial_frame(*first, cell)
            times = []
            for r in range(a.warmup + a.repeat):
                plan.clear(); vb.device_synchronize(0)
                t0 = time.perf_counter(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); dt = time.perf_counter() - t0
                if r >= a.warmup: times.append(dt)
            vals = plan.property_data("r").values.reshape(F, groups)
            w = {"system": f"water_system({N_SIDE})" if system == "water" else "membrane%s" % (MEMB,), "atoms": n, "script": script, "contexts": groups,
                 "atoms_in_groups": int(props[0].idx[0].size), "frames_per_s": {"best": F / min(times), "median": F / float(np.median(times))}, "call_s": times,
                 "value_range": [float(vals[1:].min()), float(vals[1:].max())]}
            w["fits_per_s"] = w["frames_per_s"]["best"] * groups
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                plan.clear(); plan.eval_device_frames(d_xyz, 3 * n, n, cell, 0, F); plan.sync(); torch.cuda.synchronize()
            kt = {}
            for e in prof.key_averages():
                name = e.key.split("(")[0].split("::")[-1]
                if "k_rmsd" in name:
                    dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                    kt[name] = {"calls": e.count, "total_ms": dev / 1e3, "per_frame_us": dev / F}
            w["kernels"] = kt
            plan.close()
            w["reference_cpu"] = reference_times(system, script, a.ref_frames, os.cpu_count() or 1)
            for k, r in w["reference_cpu"].items():
                if isinstance(r, dict) and "frames_per_s" in r: w[f"speedup_vs_{k}"] = w["frames_per_s"]["best"] / r["frames_per_s"]
            info["workloads"][wl] = w
        vb.device_free(0, d_xyz); vb.device_free(0, d_base)
        if d_mol is not None: vb.device_free(0, d_mol)
    line = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f: f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
