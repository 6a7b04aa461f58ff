"""Ramachandran density maps on the device at trajectory scale: a backbone-angles property of 1 000 000 frames x 256 segments (2 GB of angles in HBM,
filled on the device with seeded angles clustered in the helix and sheet basins), then Plan.rama_density over the full range and over 10 % of it at
sigma = 5, as VIAMD's Ramachandran component calls rama_rep_compute_density for the whole trajectory and for its timeline filter.

Prints one JSON line: GPU name, power limit and SM clock read in this run; per call the time of the whole C call (host clock around a call that
ends in a device synchronise, best and median of --calls after --warmup); the kernels' device time from a torch.profiler pass over a few more calls
(after the timed window): the scatter, the blur alone, the conversion; the scatter's bytes of angles read per second against 3.35 TB/s, also for
a fill where every pair lands in one texel and one where every pair is (0, 0) and skipped (DESIGN.md §8c).

  python profiles/rama_density.py [--frames 1000000] [--segments 256] [--calls 20] [--warmup 3]
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

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        r = [s.strip() for s in out.strip().split(",")]
        return {"name": r[0], "power_limit_w": float(r[1]), "sm_clock_mhz": float(r[2]), "sm_max_mhz": float(r[3])}
    except Exception as e:   # the numbers below still stand, without the card's settings
        return {"error": str(e)}


def fill_angles(view, F, S, seed):
    """[F][S] (phi, psi) in radians: 45 % around the helix basin (-63, -43 deg), 45 % around the sheet basin (-120, 130 deg), sd 12 deg, 10 % uniform"""
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    deg = np.pi / 180.0; chunk = 1 << 24
    n = F * S
    for b in range(0, n, chunk):
        m = min(chunk, n - b)
        r = torch.rand(m, device="cuda", generator=g)
        noise = torch.randn(m, 2, device="cuda", generator=g) * (12.0 * deg)
        centre = torch.where((r < 0.45)[:, None], torch.tensor([-63.0 * deg, -43.0 * deg], device="cuda"), torch.tensor([-120.0 * deg, 130.0 * deg], device="cuda"))
        uni = (torch.rand(m, 2, device="cuda", generator=g) * 2.0 - 1.0) * np.pi
        a = torch.where((r < 0.9)[:, None], centre + noise, uni)
        view[2 * b:2 * (b + m)] = a.reshape(-1).to(torch.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1_000_000)
    ap.add_argument("--segments", type=int, default=256)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import viamd_b200 as vb
    from viamd_b200.dist import _CudaView
    if vb.device_count() < 1:
        raise SystemExit("rama_density.py measures on a CUDA device; none found")
    F, S = args.frames, args.segments
    info = gpu_info()
    five = np.tile(np.arange(5, dtype=np.int32), (S, 1))
    plan = vb.Plan(vb.System(5, np.ones(5, np.float32)), [vb.backbone_angles("bb", five)], F)
    ptr, nbytes, _ = plan.accum_ptr("bb"); assert nbytes == F * S * 8
    fill_angles(torch.as_tensor(_CudaView(ptr, F * S * 2, "<f4"), device="cuda"), F, S, args.seed); torch.cuda.synchronize()
    plan.mark_frames_done(0, F)
    seg = np.arange(S, dtype=np.uint32); q = S // 16
    classes = [seg[:S - 3 * q], seg[S - 3 * q:S - 2 * q], seg[S - 2 * q:S - q], seg[S - q:]]   # general, glycine, proline, pre-proline
    cases = {"full": (0, F), "range10": (0, F // 10), "empty": (0, 0)}
    out = {"gpu": info, "frames": F, "segments": S, "sigma": 5.0, "angle_bytes": nbytes, "calls": args.calls, "warmup": args.warmup}
    sums = {}
    for name, (b, e) in cases.items():
        for _ in range(args.warmup): tex, s = plan.rama_density("bb", classes, b, e, 5.0)
        sums[name] = [float(v) for v in s]
        t = []
        for _ in range(args.calls):
            t0 = time.perf_counter(); plan.rama_density("bb", classes, b, e, 5.0); t.append(time.perf_counter() - t0)   # the call ends in a D2H copy
        out[f"{name}_call_ms"] = {"best": 1e3 * min(t), "median": 1e3 * float(np.median(t))}
    out["samples"] = sums
    # kernel device times, after the timed window: a torch.profiler pass (CUPTI sees the library's kernels in this process)
    from torch.profiler import profile, ProfilerActivity
    reps = 5; kern = {}
    for name in ("full", "range10"):
        b, e = cases[name]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps): plan.rama_density("bb", classes, b, e, 5.0)
            torch.cuda.synchronize()
        tot = {}
        for ev in prof.key_averages():
            k = next((n for n in ("k_rama_scatter", "k_rama_blur_lines", "k_rama_convert") if n in ev.key), None)
            if k: tot[k] = tot.get(k, 0.0) + (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)) / 1e3 / reps   # us -> ms per call
        scatter_ms = tot.get("k_rama_scatter", float("nan")); bytes_read = (e - b) * S * 8
        kern[name] = {"scatter_ms": scatter_ms, "blur_ms": tot.get("k_rama_blur_lines", float("nan")), "convert_ms": tot.get("k_rama_convert", float("nan")),
                      "scatter_angle_bytes_per_s": bytes_read / (scatter_ms * 1e-3), "scatter_share_of_hbm_peak": bytes_read / (scatter_ms * 1e-3) / HBM_BYTES_PER_S}
    # two fills that bracket the scatter: every pair in ONE texel (the worst pile-up: the warp merge leaves one atomic per 32 samples, all on one
    # address) and every pair (0, 0), which the task skips (the angles are read, no atomic is issued: the scatter's read cost alone)
    view = torch.as_tensor(_CudaView(ptr, F * S * 2, "<f4"), device="cuda")
    for name, fill in (("full_one_texel", (-1.1, -0.75)), ("full_all_skipped", (0.0, 0.0))):
        view[0::2] = fill[0]; view[1::2] = fill[1]; torch.cuda.synchronize()
        for _ in range(args.warmup): plan.rama_density("bb", classes, 0, F, 5.0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps): plan.rama_density("bb", classes, 0, F, 5.0)
            torch.cuda.synchronize()
        ms = sum((getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)) for ev in prof.key_averages() if "k_rama_scatter" in ev.key) / 1e3 / reps
        kern[name] = {"scatter_ms": ms, "scatter_angle_bytes_per_s": F * S * 8 / (ms * 1e-3), "scatter_share_of_hbm_peak": F * S * 8 / (ms * 1e-3) / HBM_BYTES_PER_S}
    del view
    out["kernels"] = kern
    plan.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
