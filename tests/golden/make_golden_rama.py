"""Generate tests/golden/rama.npz from the UNMODIFIED reference: VIAMD's Ramachandran density task (oracle/_ref/rama_harness_strict, built by
`make -C oracle -f rama.mk`; needs /root/reference). The fixture stores the inputs together with the reference's outputs, so the tests need
neither the reference nor the harness.

  rama.npz : the density task on 64 jittered frames of mdlib's 1LAF (238 residues, all four classes): backbone angles, class lists, and per case
             (full range at sigma 5, sub-ranges at sigma 0.1 and 10) the sums, a digest of the blurred map and every 17th value of it.

  python tests/golden/make_golden_rama.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import refio  # noqa: E402

HARNESS = os.path.join(ROOT, "oracle", "_ref", "rama_harness_strict")
SYSINFO = os.path.join(ROOT, "oracle", "_ref", "ref_harness_strict")


def run(*a):
    subprocess.check_call(list(a), stdout=subprocess.DEVNULL)



RAMA_PDB = "/root/reference/ext/mdlib/test_data/1LAF.pdb"
RAMA_CASES = ((0, 64, 5.0), (8, 40, 0.1), (20, 52, 10.0))   # (frame_beg, frame_end, sigma) of the density task


RAMA_SAMPLE = 17   # every 17th value of a map is stored (all four channels); the whole map is pinned by its digest


def rama_tex_digest(tex):
    """sha256 of a [512, 512, 4] float32 map with -0 turned into +0: the box passes of the reference leave float residues in almost every texel, so
    the maps do not compress (about 3 MB each); the digest pins every value, the stored sample shows where a map differs"""
    import hashlib
    return hashlib.sha256((np.ascontiguousarray(tex, np.float32) + np.float32(0)).tobytes()).hexdigest()


def rama_frames(base, seed, F, jitter):
    """F frames of the 1LAF structure, every atom displaced by a Gaussian of `jitter` Angstrom per axis (numpy's PCG64, seeded)"""
    rng = np.random.default_rng(seed)
    return (base[None].astype(np.float64) + rng.normal(0.0, jitter, (F,) + base.shape)).astype(np.float32)


def rama(tmp):
    """VIAMD's Ramachandran density task (harness mode `rama`: md_util_backbone_angles_compute per frame, the class lists of segment.rama_type, the
    task's accumulation loop and the reference's own blur_density_gaussian) on 64 jittered frames of mdlib's 1LAF (238 residues, all four classes):
    the segments' five atoms, the angles [F][nseg][2], the class lists (CSR), and per case in RAMA_CASES the sums, the digest of the blurred map and
    every RAMA_SAMPLE-th value of it."""
    si = os.path.join(tmp, "laf.sys"); raw = os.path.join(tmp, "laf.raw"); o = os.path.join(tmp, "laf.bin")
    run(SYSINFO, "sysinfo", "--sys", RAMA_PDB, "--out", si)
    s = refio.read_sysinfo(si); base = np.stack([s["x"], s["y"], s["zc"]]); seed, jitter, F = 2024, 0.3, 64
    frames = rama_frames(base, seed, F, jitter)
    refio.write_raw_traj(raw, frames, np.tile(np.array(s["cell"][:6], np.float64), (F, 1)), np.full(F, s["cell"][6], np.uint32))
    out = dict(base=base, cell=np.array(s["cell"][:6], np.float64), cell_flags=np.uint32(s["cell"][6]), seed=np.int64(seed), jitter=np.float64(jitter),
               cases=np.array([c[:2] for c in RAMA_CASES], np.int64), sigmas=np.array([c[2] for c in RAMA_CASES], np.float32))
    for k, (beg, end, sigma) in enumerate(RAMA_CASES):
        run(HARNESS, "rama", "--sys", RAMA_PDB, "--traj", f"raw:{raw}", "--range", f"{beg}:{end}", "--sigma", repr(sigma), "--out", o)
        b = open(o, "rb").read(); assert b[:8] == b"MDRAMADN"
        nf, ns = (int(v) for v in np.frombuffer(b, np.uint64, 2, 8)); off = 24
        five = np.frombuffer(b, np.int32, ns * 5, off).reshape(ns, 5); off += ns * 20
        ang = np.frombuffer(b, np.float32, nf * ns * 2, off).reshape(nf, ns, 2); off += nf * ns * 8
        ncls = np.frombuffer(b, np.uint32, 4, off); off += 16
        seg = np.frombuffer(b, np.uint32, int(ncls.sum()), off); off += 4 * int(ncls.sum())
        rb, re_ = np.frombuffer(b, np.int64, 2, off); off += 16
        sg = np.frombuffer(b, np.float32, 1, off)[0]; off += 4
        tex = np.frombuffer(b, np.float32, 512 * 512 * 4, off).reshape(512, 512, 4); off += 512 * 512 * 16
        sums = np.frombuffer(b, np.float32, 4, off); off += 16
        assert off == len(b) and (rb, re_) == (beg, end) and sg == np.float32(sigma)
        if k == 0:
            out.update(five=five.copy(), angles=ang.copy(), seg=seg.copy(), class_off=np.concatenate([[0], np.cumsum(ncls)]).astype(np.uint32))
        assert np.array_equal(out["angles"], ang) and np.array_equal(out["seg"], seg)
        out[f"tex{k}_sha256"] = np.array(rama_tex_digest(tex)); out[f"tex{k}_sample"] = tex.ravel()[::RAMA_SAMPLE].copy(); out[f"sums{k}"] = sums.copy()
    np.savez_compressed(os.path.join(HERE, "rama.npz"), **out)


if __name__ == "__main__":
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "_ref/ref_harness_strict"])
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "-f", "rama.mk"])
    with tempfile.TemporaryDirectory() as tmp:
        rama(tmp)
    print("rama.npz", os.path.getsize(os.path.join(HERE, "rama.npz")), "bytes")
