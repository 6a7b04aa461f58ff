"""Generate tests/golden/expr6.npz from the UNMODIFIED reference (oracle/_ref/ref_harness_strict, `eval`, as make_golden_range.py does):
temporal expressions — the operators + - * / and unary - (md_script_functions.inl:505-571) and the functions (:576-603) over other temporal
properties of the script, with constants, PI / TAU / E and integer literals — on three frame sets:
  a : the ala50 frames of 1ALA
  w : the water6 frames (orthorhombic cell)
  t : the tric6 frames (triclinic cell changing every frame)
The script has every operator and function, identifiers two levels deep (e2 reads e1, which reads s2), an inline call (x), array temporals of
`angle in residue(1:5)` with floats and with arrays of equal length, `float - array` (the reference applies it as `array - float`), a unary minus
before a chain (the reference negates the whole left operand of the chain's last operator), division by zero, sqrt and log of negative values,
and NaN operands. For each statement the generator checks that the reference lists it as a temporal property with the expected [F, dim] layout,
and stores its values, the per-frame aggregates of the array ones and the reported min / max value and range.

Run here (needs /root/reference + `make -C oracle ref oracle`):   python tests/golden/make_golden_expr.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import refio  # noqa: E402
from make_golden import HARNESS, SYNTH, run  # noqa: E402

PDB = "/root/reference/datasets/1ALA-500.pdb"
NCTX = 5   # contexts of the array temporal a1

SCRIPT = ("d1 = distance(1, 10); d2 = distance(4, 20); t1 = dihedral(1, 2, 3, 4); "
          # operators, constants, integer literals, precedence
          "s1 = d1 + d2; s2 = d1 - d2; s3 = d1 * d2; s4 = d1 / d2; s5 = -d1; s6 = d1 * 10 + 2.5; s7 = (d1 - d2) * (d1 + d2) / 3; "
          "s8 = -d1 - d2 - 1; s9 = d1 - d2 * 3 - d1 / 2 + 1; "
          # identifiers two levels deep, an inline call, PI / TAU / E
          "e1 = s2 * 2 - s1; e2 = e1 / 4 + s7; x = distance(1, 10) * 10; h = abs(t1 - PI); c1 = TAU * d1 + E; "
          # every function
          "fl = floor(d1 * 3); ce = ceil(d2 / 3); f1 = sqrt(d1); f2 = cbrt(s2); f3 = cos(t1); f4 = sin(t1); f5 = asin(d2 / 100); f6 = acos(s2 / 50); "
          "f7 = atan(s2); f8 = log(d1); f9 = exp(d1 / 10); f10 = log2(d1); f11 = exp2(d1 / 5); f12 = log10(d1); "
          "g1 = atan(d1, s2); g2 = atan2(s2, d2); g3 = pow(d1, 1.5); g4 = min(d1, d2); g5 = max(d1, d2); g6 = pow(s2, 2); "
          # IEEE edge cases: division by zero, sqrt / log of negative values, NaN operands
          "z1 = d1 / 0; z2 = -d1 / 0; z3 = sqrt(s2); z4 = 0 / (d1 - d1); z5 = z4 + 1; z6 = min(z4, d1); z7 = log(-d1); "
          # array temporals: with floats and with arrays of equal length
          f"a1 = angle(2, 1, 3) in residue(1:{NCTX}); a2 = a1 * 2; a3 = 2 - a1; a4 = a1 - a1 * 0.5; a5 = abs(a3 - 1); a6 = floor(a1) + ceil(a1); "
          "a7 = a1 / d1; a8 = -a1; a9 = a2 / (a1 - a1);")


def dims():
    """[F, dim] of every statement: NCTX values per frame for the a* properties, one for the others"""
    return {st.split("=")[0].strip(): (NCTX if st.strip().startswith("a") else 1) for st in SCRIPT.split(";") if st.strip()}


def main():
    a = np.load(os.path.join(HERE, "ala50.npz")); w = np.load(os.path.join(HERE, "water6.npz")); t = np.load(os.path.join(HERE, "tric6.npz"))
    out = {"script": np.array(SCRIPT)}
    want = dims()
    with tempfile.TemporaryDirectory() as tmp:
        for tag, g, sysfile in (("a", a, PDB), ("w", w, "77"), ("t", t, "91")):
            if sysfile != PDB:
                gro = os.path.join(tmp, tag + ".gro"); run(SYNTH, "water-gro", "6", sysfile, gro); sysfile = gro
            raw, o = os.path.join(tmp, tag + ".raw"), os.path.join(tmp, tag + ".out")
            F = g["frames"].shape[0]
            refio.write_raw_traj(raw, g["frames"], g["cells"], g["cell_flags"])
            run(HARNESS, "eval", "--sys", sysfile, "--traj", f"raw:{raw}", "--script", SCRIPT, "--out", o, "--full", f"0:{F}")
            props = refio.read_refout(o)
            assert list(props) == list(want), (tag, list(props))   # every statement is a property of the script, in order
            for name, p in props.items():
                assert p.flags & refio.FLAG_TEMPORAL and list(p.dim[:2]) == [F, want[name]], (tag, name, p.flags, p.dim)
                k = f"{tag}_{name}"
                out[k + "__full"] = p.full
                m = p.meta[(1, 0)]
                out[k + "__meta"] = np.array([m["min_value"], m["max_value"], m["min_range"][0], m["max_range"][0]], np.float32)
                if p.aggregate is not None: out[k + "__mean"] = p.aggregate["mean"]; out[k + "__var"] = p.aggregate["var"]; out[k + "__ext"] = p.aggregate["ext"]
    path = os.path.join(HERE, "expr6.npz")
    np.savez_compressed(path, **out)
    print("expr6.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
