"""Secondary structure per frame on the device (MDGPU_OP_SECONDARY_STRUCTURE): throughput with the frames in HBM, device time per kernel, and
VIAMD's whole backbone pass (angles + secondary structure) as one plan.

  python profiles/secondary_structure.py [--frames 4096] [--out profiles/secondary_structure_h100.json]
  python profiles/secondary_structure.py --reference   # the reference's fast build, 1 thread and all cores: md_util_backbone_secondary_structure_infer,
                                                        # md_util_backbone_angles_compute, and both per frame (VIAMD's backbone pass, frames in memory)

Frames are the golden fixture's frames (tests/golden/dssp.npz) repeated. Rates are best and median of 5 runs of mdgpu_eval_device_frames + sync,
timed with CUDA events around the whole call sequence."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def five_of(atoms, ro):
    five = np.full((len(atoms), 5), -1, np.int32)
    for r in range(len(ro) - 1):
        b, e = int(ro[r]), int(ro[r + 1])
        if e - b < 4: continue
        for i in range(b + 1, e - 1): five[i] = [atoms[i - 1, 2], atoms[i, 0], atoms[i, 1], atoms[i, 2], atoms[i + 1, 0]]
    return five


def device(args):
    import torch
    import viamd_b200 as vb
    g = np.load(os.path.join(ROOT, "tests", "golden", "dssp.npz"))
    res = dict(gpu=torch.cuda.get_device_name(0), frames=args.frames, cases={})
    for c in ("laf", "tub"):
        atoms, ro, xyz = g[f"{c}_atoms"], g[f"{c}_range_off"], g[f"{c}_xyz"]
        F, n = args.frames, xyz.shape[2]
        frames = np.ascontiguousarray(np.resize(xyz, (F,) + xyz.shape[1:]), np.float32)
        d = torch.from_numpy(frames).cuda()
        cell = vb.UnitCell(*(float(v) for v in g[f"{c}_cells"][0]), int(g[f"{c}_flags"][0]))
        out = dict(segments=int(len(atoms)))
        for label, props in (("ss", [vb.secondary_structure("ss", atoms, ro)]),
                             ("angles", [vb.backbone_angles("bb", five_of(atoms, ro))]),
                             ("angles+ss", [vb.backbone_angles("bb", five_of(atoms, ro)), vb.secondary_structure("ss", atoms, ro)])):
            plan = vb.Plan(vb.System(n, np.ones(n, np.float32)), props, F)
            times = []
            for rep in range(6):
                plan.clear(); torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); plan.eval_device_frames(d.data_ptr(), 3 * n, n, cell, 0, F); plan.sync(); b.record(); torch.cuda.synchronize()
                if rep: times.append(a.elapsed_time(b) / 1e3)
            out[label] = dict(best_frames_per_s=F / min(times), median_frames_per_s=F / float(np.median(times)), seconds=times)
            if label == "ss":
                from torch.profiler import profile, ProfilerActivity
                plan.clear(); torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    plan.eval_device_frames(d.data_ptr(), 3 * n, n, cell, 0, F); plan.sync(); torch.cuda.synchronize()
                k = {}
                for e in prof.key_averages():
                    if e.key.startswith(("void mdg::k_ss", "mdg::k_ss", "void mdg::k_frame_geom", "void mdg::k_aabb")) or "k_ss_" in e.key:
                        k[e.key] = dict(total_ms=e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3, calls=e.count)
                out["kernels_ms_per_run"] = k
            plan.close()
        res["cases"][c] = out
    return res


def reference(args):
    g = np.load(os.path.join(ROOT, "tests", "golden", "dssp.npz"))
    sys.path.insert(0, os.path.join(ROOT, "tests")); import refio
    h = os.path.join(ROOT, "oracle", "_ref", "dssp_harness_fast"); data = "/root/reference/ext/mdlib/test_data"
    res = dict(cpu=open("/proc/cpuinfo").read().split("model name")[1].split("\n")[0].strip("\t: "), cores=os.cpu_count(), cases={})
    with tempfile.TemporaryDirectory() as tmp:
        for c, pdb in (("laf", "1LAF.pdb"), ("tub", "tubulin-A-B.pdb")):
            si = os.path.join(tmp, "s.sys"); subprocess.check_call([os.path.join(ROOT, "oracle", "_ref", "ref_harness_strict"), "sysinfo", "--sys", os.path.join(data, pdb), "--out", si], stdout=subprocess.DEVNULL)
            s = refio.read_sysinfo(si); base = np.stack([s["x"], s["y"], s["zc"]]).astype(np.float32)
            F = 256; raw = os.path.join(tmp, "t.raw")
            refio.write_raw_traj(raw, np.repeat(base[None], F, 0), np.tile(np.array(s["cell"][:6]), (F, 1)), np.full(F, s["cell"][6], np.uint32))
            out = {}
            for T in (1, os.cpu_count()):
                r = subprocess.run([h, "dssp", "--sys", os.path.join(data, pdb), "--traj", f"raw:{raw}", "--time", "8", "--threads", str(T)], capture_output=True, text=True, check=True)
                out[f"threads_{T}"] = json.loads(r.stdout.strip().splitlines()[-1])
            res["cases"][c] = out
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser(); ap.add_argument("--frames", type=int, default=4096); ap.add_argument("--out", default=None); ap.add_argument("--reference", action="store_true")
    a = ap.parse_args()
    r = reference(a) if a.reference else device(a)
    s = json.dumps(r)
    print(s)
    if a.out:
        with open(a.out, "w") as f: f.write(s + "\n")
