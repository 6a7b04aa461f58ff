"""Generate tests/golden/dssp.npz from the UNMODIFIED reference: md_util_backbone_secondary_structure_infer per frame (oracle/_ref/dssp_harness_strict,
built by `make -C oracle -f dssp.mk`; needs /root/reference). The fixture stores the inputs together with the reference's rows, so the tests need
neither the reference nor the harness.

Cases (each: the segments' atoms N, CA, C, O, HN remapped to a compact atom list, the range offsets, frames [F][3][n] of those atoms, cells, rows):
  laf      mdlib's 1LAF (one chain, helices and sheets): the structure as read, then jittered frames
  laf_hn   1LAF with an explicit HN atom (the CB) for every third segment
  tub      tubulin-A-B (two proteins, five backbone ranges): chain-pair bridges and range ends
  pbc      1LAF centred on a corner of a periodic orthorhombic cell, coordinates not wrapped: the walk's periodic images
  tric     the same in a triclinic cell
  open     1LAF without a cell (flags 0): the walk's grid fitted to the data
  short    1LAF with its chain ids rewritten into chains of 1, 2, 3, 4, 5 and 223 residues; the reference's backbone extraction drops the
           chains of 1 and 2 residues, so the case holds ranges of 3, 4, 5 and 223 segments

The reference's turn masks and flags live in uncleared temporary memory; the harness clears the arena region before each call. The generator
checks that this works (rows equal when the frames run in reverse order) and that the hazard is real (a 0xFF pre-fill changes the rows).
The device library and the restatement use 1 / sqrtf where the reference uses rsqrtps + one Newton step, and atan2f may differ in the last
ulp, so every frame must keep its decisions away from the thresholds: a float64 evaluation checks that every pair energy is at least 1e-3 from
-0.5, that each donor's 2nd and 3rd lowest energies <= -0.5 differ by at least 1e-3 and that every bend angle is at least 1e-4 rad from 70
degrees. A jittered frame that fails is drawn again with the next seed; the seeds used are stored.

  python tests/golden/make_golden_dssp.py
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

HARNESS = os.path.join(ROOT, "oracle", "_ref", "dssp_harness_strict")
SYSINFO = os.path.join(ROOT, "oracle", "_ref", "ref_harness_strict")
DATA = "/root/reference/ext/mdlib/test_data"
TRI, PBC_ALL, ORTHO = 2, 28, 1


def run(*a):
    subprocess.check_call(list(a), stdout=subprocess.DEVNULL)


def harness(pdb, frames, cells, flags, tmp, extra=()):
    raw = os.path.join(tmp, "t.raw"); o = os.path.join(tmp, "t.bin")
    refio.write_raw_traj(raw, frames, cells, flags)
    run(HARNESS, "dssp", "--sys", pdb, "--traj", f"raw:{raw}", "--out", o, *extra)
    b = open(o, "rb").read(); assert b[:8] == b"MDSSPRED"
    F, S, R = (int(v) for v in np.frombuffer(b, np.uint64, 3, 8)); off = 32
    atoms = np.frombuffer(b, np.int32, S * 5, off).reshape(S, 5).copy(); off += S * 20
    ro = np.frombuffer(b, np.uint32, R + 1, off).copy(); off += 4 * (R + 1)
    ss = np.frombuffer(b, np.int32, F * S, off).reshape(F, S).copy(); off += 4 * F * S
    assert off == len(b)
    return atoms, ro, ss


def margins_ok(xyz, atoms, ro):
    """float64 evaluation of the thresholds of one frame (xyz [3][n] over the atoms the segments name)"""
    P = lambda k: xyz[:, atoms[:, k]].T.astype(np.float64)
    N, CA, C, O = P(0), P(1), P(2), P(3)
    S = len(atoms); rid = np.zeros(S, np.int64)
    for r in range(len(ro) - 1): rid[ro[r]:ro[r + 1]] = r
    nrm = lambda v: v / np.linalg.norm(v, axis=-1, keepdims=True)
    H = np.where(atoms[:, 4:5] >= 0, xyz[:, np.maximum(atoms[:, 4], 0)].T.astype(np.float64), 0.0)
    for i in range(S):
        if atoms[i, 4] >= 0: continue
        Cp = C[i - 1] if i > ro[rid[i]] else N[i] + (CA[i] - C[i])
        H[i] = N[i] + nrm(nrm(N[i] - CA[i]) + nrm(N[i] - Cp)) * 1.01
    d = lambda a, b: np.linalg.norm(a[:, None, :] - b[None, :, :], axis=-1)   # [donor, acceptor]
    dNO, dHC, dNC, dHO = d(N, O), d(H, C), d(N, C), d(H, O)
    e = 27.888 * (1 / dNO + 1 / dHC - 1 / dNC - 1 / dHO)
    close = (np.minimum(np.minimum(dNO, dHC), np.minimum(dNC, dHO)) < 0.5)
    e = np.where(close, -9.9, np.maximum(e, -9.9))
    ii, jj = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    valid = (ii != jj) & ~((rid[ii] == rid[jj]) & (np.abs(ii - jj) <= 1)) & ~close
    if np.any(valid & (np.abs(e + 0.5) < 1e-3)): return False
    for dn in range(S):
        rec = np.sort(e[dn][(e[dn] <= -0.5) & (ii[dn] != jj[dn])])
        if len(rec) >= 3 and rec[2] - rec[1] < 1e-3: return False
    for r in range(len(ro) - 1):
        for i in range(ro[r] + 2, ro[r + 1] - 2):
            v1, v2 = CA[i - 2] - CA[i], CA[i + 2] - CA[i]
            ang = np.arctan2(np.linalg.norm(np.cross(v1, v2)), v1 @ v2)
            if abs(ang - np.deg2rad(70.0)) < 1e-4: return False
    return True


def short_ranges_pdb(tmp):
    """1LAF with its chain id rewritten so that the residues form ranges of 1, 2, 3, 4, 5 and the rest (TER between them)"""
    out, res_seen, chain_of = [], [], {}
    cuts = np.cumsum([1, 2, 3, 4, 5]); ids = "ABCDEF"
    for line in open(os.path.join(DATA, "1LAF.pdb")):
        if line.startswith(("ATOM", "HETATM")) and line.startswith("ATOM"):
            key = line[22:27]
            if key not in chain_of:
                k = len(res_seen); res_seen.append(key)
                chain_of[key] = ids[int(np.searchsorted(cuts, k, side="right"))]
            c = chain_of[key]
            if out and out[-1].startswith("ATOM") and out[-1][21] != c: out.append("TER\n")
            out.append(line[:21] + c + line[22:])
        elif line.startswith(("CRYST1", "END")):
            out.append(line)
    p = os.path.join(tmp, "short.pdb"); open(p, "w").writelines(out); return p


def make_case(name, pdb, tmp, nframes, jitter, seed, cell, flags, shift=None, extra=(), with_base=True):
    si = os.path.join(tmp, "s.sys"); run(SYSINFO, "sysinfo", "--sys", pdb, "--out", si)
    s = refio.read_sysinfo(si); base = np.stack([s["x"], s["y"], s["zc"]]).astype(np.float64)
    if shift is not None: base = base + np.asarray(shift, np.float64)[:, None]
    cell = np.asarray(s["cell"][:6] if cell is None else cell, np.float64); flags = int(s["cell"][6] if flags is None else flags)
    atoms, ro, _ = harness(pdb, base[None].astype(np.float32), cell[None], np.array([flags], np.uint32), tmp, extra)
    frames, seeds = [], []
    if with_base:
        f0 = base.astype(np.float32)
        assert margins_ok(f0, atoms, ro), f"{name}: the unjittered structure has a decision at a threshold"
        frames.append(f0); seeds.append(-1)
    k = seed
    while len(frames) < nframes:
        f = (base + np.random.default_rng(k).normal(0.0, jitter, base.shape)).astype(np.float32)
        if margins_ok(f, atoms, ro): frames.append(f); seeds.append(k)
        k += 1
    frames = np.stack(frames); F = len(frames)
    cells = np.tile(cell, (F, 1)); fl = np.full(F, flags, np.uint32)
    a2, r2, ss = harness(pdb, frames, cells, fl, tmp, extra)
    assert np.array_equal(a2, atoms) and np.array_equal(r2, ro)
    _, _, ss_rev = harness(pdb, frames, cells, fl, tmp, (*extra, "--reverse", "1"))
    _, _, ss_ff = harness(pdb, frames, cells, fl, tmp, (*extra, "--prefill", "255"))
    assert np.array_equal(ss, ss_rev), f"{name}: rows depend on the frame order although the arena is cleared"
    used = np.unique(atoms[atoms >= 0]); remap = np.full(frames.shape[2], -1, np.int32); remap[used] = np.arange(len(used), dtype=np.int32)
    local = np.where(atoms >= 0, remap[np.maximum(atoms, 0)], -1).astype(np.int32)
    print(f"{name}: F={F} S={len(atoms)} ranges={len(ro) - 1} seeds={seeds} prefill_changes_rows={not np.array_equal(ss, ss_ff)}")
    return {f"{name}_atoms": local, f"{name}_range_off": ro, f"{name}_xyz": frames[:, :, used], f"{name}_cells": cells, f"{name}_flags": fl,
            f"{name}_ss": ss, f"{name}_seeds": np.array(seeds, np.int64), f"{name}_reverse_equal": np.bool_(np.array_equal(ss, ss_rev)),
            f"{name}_prefill_differs": np.bool_(not np.array_equal(ss, ss_ff))}


if __name__ == "__main__":
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "_ref/ref_harness_strict"])
    subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "-f", "dssp.mk"])
    laf, tub = os.path.join(DATA, "1LAF.pdb"), os.path.join(DATA, "tubulin-A-B.pdb")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        out.update(make_case("laf", laf, tmp, 12, 0.2, 1000, None, None))
        out.update(make_case("laf_hn", laf, tmp, 5, 0.2, 2000, None, None, extra=("--hn-cb-every", "3")))
        out.update(make_case("tub", tub, tmp, 5, 0.2, 3000, None, None, with_base=False))   # the deposited structure has a pair energy within 1e-3 of -0.5
        corner = (-35.0, -20.0, -45.0)   # moves 1LAF's centre near the origin: the protein straddles three faces of the cell
        out.update(make_case("pbc", laf, tmp, 5, 0.2, 4000, (61.0, 0, 0, 57.5, 0, 64.0), ORTHO | PBC_ALL, shift=corner))
        out.update(make_case("tric", laf, tmp, 5, 0.2, 5000, (62.0, 9.0, 7.5, 58.0, 11.0, 66.0), TRI | PBC_ALL, shift=corner))
        out.update(make_case("open", laf, tmp, 4, 0.2, 6000, (0, 0, 0, 0, 0, 0), 0))
        out.update(make_case("short", short_ranges_pdb(tmp), tmp, 5, 0.2, 7000, None, None))
    out["cases"] = np.array(["laf", "laf_hn", "tub", "pbc", "tric", "open", "short"])
    np.savez_compressed(os.path.join(HERE, "dssp.npz"), **out)
    print("dssp.npz", os.path.getsize(os.path.join(HERE, "dssp.npz")), "bytes")
