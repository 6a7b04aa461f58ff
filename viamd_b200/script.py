"""Minimal lowering of md_script property statements to libmdgpu property descriptors.

In VIAMD the script front-end (tokenizer, parser, static type check, static evaluation of selections) is mdlib's own
md_script.c and stays unchanged; INTEGRATION.md shows the shim that walks a compiled md_script_ir_t and emits the same
descriptors. This module exists so that the tests and bench.py can be written the way the reference's own tests are
(mdlib/unittest/test_script.c:1259-1273: `prop1 = rdf(element('C'), element('O'), 20.0);`) without the reference on the box.

Supported statements:  ident = proc(args);   with proc in
    rdf(sel, sel, cutoff | min:max)   sdf(residue(a:b) | sel-array, sel, cutoff)   density_x|_y|_z(sel)
    distance(i, j)   angle(i, j, k)   dihedral(i, j, k, l)            (1-based atom indices as in md_script)
    porosity(sel)                                                        (needs System.radius)
    count(dyn [, 'atom' | 'residue' | 'chain' | 'structure'])           (dyn: a dynamic selection below; 'chain' needs System.chain_atom_range)
and temporal expressions: + - * / and unary -, the functions sqrt cbrt abs floor ceil cos sin asin acos atan log exp log2 exp2 log10
atan(y, x) atan2 pow min max, over numbers, PI / TAU / E, earlier temporal properties and inline calls of the procedures above.
Selections (evaluated once, statically, to ascending atom index lists — md_script.c:5492-5524):
    all | element('O') | name('C2*') | resname('SOL') | atom(a:b) | residue(a:b) | `and` / `or` / `not` of these
Dynamic selections (evaluated per frame on the device), alone or `static and ...` in either order, where a consumer accepts them:
    within([min:]max, sel) | within_x(a:b) | within_y(a:b) | within_z(a:b) | within_xyz(a:b, c:d, e:f)
`residue(a:b)` used as the first argument of sdf() yields one structure per residue (bitfield array semantics).
"""
from __future__ import annotations

import fnmatch
import re
from typing import List

import numpy as np

from . import api

_TOK = re.compile(r"\s*(?:(\d+\.\d*|\.\d+|\d+)|([A-Za-z_][A-Za-z_0-9]*)|'([^']*)'|\"([^\"]*)\"|(.))")


class ScriptError(ValueError):
    pass


_DYNAMIC = ("within", "within_x", "within_y", "within_z", "within_xyz")   # selections whose atoms depend on the frame's coordinates (FLAG_DYNAMIC)


def _tokens(src: str):
    out = []
    for m in _TOK.finditer(src):
        num, ident, s1, s2, ch = m.groups()
        if num is not None: out.append(("num", num))
        elif ident is not None: out.append(("id", ident))
        elif s1 is not None: out.append(("str", s1))
        elif s2 is not None: out.append(("str", s2))
        elif ch and not ch.isspace(): out.append(("ch", ch))
    return out


class _Parser:
    def __init__(self, toks, system: api.System):
        self.t, self.i, self.sys = toks, 0, system

    def peek(self): return self.t[self.i] if self.i < len(self.t) else ("eof", "")
    def next(self): tok = self.peek(); self.i += 1; return tok

    def expect(self, kind, val=None):
        tok = self.next()
        if tok[0] != kind or (val is not None and tok[1] != val):
            raise ScriptError(f"expected {val or kind}, got {tok[1]!r}")
        return tok

    # ---- selections -> boolean masks
    _static_seen = False
    _within = None   # the one dynamic selection met while parsing a selection expression, see dyn_arg(): ("within", min, max, selection) | ("range", lo, hi)

    def sel_or(self):
        m = self.sel_and()
        while self.peek() == ("id", "or"):
            if self._within is not None: raise ScriptError("within() is lowered as `selection and within(...)` only, not under `or`")
            self.next(); m = m | self.sel_and()
            if self._within is not None: raise ScriptError("within() is lowered as `selection and within(...)` only, not under `or`")
        return m

    def sel_and(self):
        m = self.sel_not()
        while self.peek() == ("id", "and"):
            self.next(); m = m & self.sel_not()
        return m

    def sel_not(self):
        if self.peek() == ("id", "not"):
            had = self._within
            self.next(); m = ~self.sel_not()
            if self._within is not had: raise ScriptError("`not within(...)` is not lowered")
            return m
        return self.sel_atom()

    def dyn_arg(self):
        """`within([min:]max, sel)` or a coordinate range within_x / _y / _z / _xyz(...), alone or `static and ...` (either order) -> api.Within /
        api.Range; the dynamic part is evaluated per frame on the device, the static side becomes its AND side (_and md_script_functions.inl:1975)"""
        self._within = None; self._static_seen = False
        m = self.sel_or()
        if self._within is None: raise ScriptError("a within(...) expression was expected")
        w = self._within; self._within = None
        cand = np.nonzero(m)[0].astype(np.int32) if self._static_seen else None
        return api.Range(w[1], w[2], cand) if w[0] == "range" else api.Within(w[2], w[3], w[1], cand)

    def frange(self):
        """a:b | a: | :b | : (the range literal, md_script.c) -> (lo, hi) of the frange the front end hands a procedure that takes one: bounds of a
        float range as floats with open ends at -FLT_MAX / FLT_MAX; an integer range keeps INT32_MIN / INT32_MAX for open ends and is cast
        bound by bound to float (_cast_irng_to_frng md_script_functions.inl:4378)"""
        lo = hi = None; is_float = False
        if self.peek()[0] == "num": t = self.next()[1]; lo = float(t); is_float |= "." in t
        self.expect("ch", ":")
        if self.peek()[0] == "num": t = self.next()[1]; hi = float(t); is_float |= "." in t
        if is_float: return (-api.FLT_MAX if lo is None else float(np.float32(lo)), api.FLT_MAX if hi is None else float(np.float32(hi)))
        return (float(np.float32(-2 ** 31 if lo is None else int(lo))), float(np.float32(2 ** 31 - 1 if hi is None else int(hi))))

    def _range(self, count):
        """a | a:b | : (1-based inclusive, as in md_script) -> python slice bounds (0-based, exclusive end)"""
        lo, hi = 1, count
        if self.peek()[0] == "num":
            lo = int(float(self.next()[1])); hi = lo
        if self.peek() == ("ch", ":"):
            self.next(); hi = count
            if self.peek()[0] == "num": hi = int(float(self.next()[1]))
        return max(lo - 1, 0), min(hi, count)

    def sel_atom(self):
        n = self.sys.num_atoms
        tok = self.next()
        if tok == ("ch", "("):
            m = self.sel_or(); self.expect("ch", ")"); return m
        if tok[0] != "id":
            raise ScriptError(f"unexpected token {tok[1]!r} in selection")
        f = tok[1]
        if f in _DYNAMIC:   # only inside dyn_arg(): stands for "every atom" in the static mask, the device supplies the real set
            if self._within is not None: raise ScriptError("one dynamic selection (within, within_x / _y / _z / _xyz) per expression")
            self.expect("ch", "(")
            if f == "within":
                lo, hi = self.radius(); self.expect("ch", ",")
                seen = self._static_seen; sel = self.selection(); self._static_seen = seen; self.expect("ch", ")")   # within's own argument is not the static side; FLAG_FLATTEN (:673): an array of selections is their union
                self._within = ("within", lo, hi, sel); return np.ones(n, bool)
            lo, hi = [-api.FLT_MAX] * 3, [api.FLT_MAX] * 3   # coordinate_range :2394: unconstrained axes are [-FLT_MAX, FLT_MAX]
            for c in (range(3) if f == "within_xyz" else ["xyz".index(f[-1])]):
                if c and f == "within_xyz": self.expect("ch", ",")
                lo[c], hi[c] = self.frange()
            self.expect("ch", ")")
            self._within = ("range", lo, hi); return np.ones(n, bool)
        self._static_seen = True
        if f == "all": return np.ones(n, bool)
        self.expect("ch", "(")
        if f in ("element", "name", "label", "resname"):
            pats = [self.expect("str")[1]]
            while self.peek() == ("ch", ","):
                self.next(); pats.append(self.expect("str")[1])
            self.expect("ch", ")")
            if f == "element":
                if self.sys.element is None: raise ScriptError("system has no element data")
                src = np.asarray(self.sys.element); return np.isin(np.char.upper(src.astype(str)), [p.upper() for p in pats])
            if f == "resname":
                if self.sys.resname is None: raise ScriptError("system has no residue data")
                rn = np.asarray(self.sys.resname); hit = np.zeros(len(rn), bool)
                for p in pats: hit |= np.array([fnmatch.fnmatchcase(r, p) for r in rn])
                return np.repeat(hit, np.diff(self.sys.res_atom_offset))
            if self.sys.name is None: raise ScriptError("system has no atom names")
            nm = np.asarray(self.sys.name); hit = np.zeros(n, bool)
            for p in pats: hit |= np.array([fnmatch.fnmatchcase(a, p) for a in nm])
            return hit
        if f == "atom":
            lo, hi = self._range(n); self.expect("ch", ")")
            m = np.zeros(n, bool); m[lo:hi] = True; return m
        if f == "residue":
            off = np.asarray(self.sys.res_atom_offset); lo, hi = self._range(len(off) - 1); self.expect("ch", ")")
            m = np.zeros(n, bool); m[off[lo]:off[hi]] = True; return m
        raise ScriptError(f"unsupported selection '{f}'")

    def selection(self) -> np.ndarray:
        m = self.sel_or()
        if self._within is not None: raise ScriptError("a dynamic selection is not lowered as this argument")
        return np.nonzero(m)[0].astype(np.int32)

    def structures(self) -> np.ndarray:
        """first argument of sdf(): residue(a:b) -> one structure per residue; otherwise a single structure"""
        save = self.i
        if self.peek() == ("id", "residue"):
            self.next(); self.expect("ch", "(")
            off = np.asarray(self.sys.res_atom_offset); lo, hi = self._range(len(off) - 1); self.expect("ch", ")")
            if self.peek() in (("ch", ","),):
                sizes = np.diff(off[lo:hi + 1])
                if len(sizes) == 0 or np.any(sizes != sizes[0]):
                    raise ScriptError("The supplied reference bitfields are not identical")   # _sdf validation :5837
                return np.stack([np.arange(off[r], off[r + 1], dtype=np.int32) for r in range(lo, hi)])
            self.i = save
        s = self.selection()
        return s.reshape(1, -1)

    def groups(self):
        """first argument of rdf(): residue(a:b) covering more than one residue is an ARRAY of bitfields -> one group per residue
        (centre-of-mass references, compute_rdf :5274); anything else is a plain selection (returns None, position unchanged)"""
        save = self.i
        if self.peek() == ("id", "residue"):
            self.next(); self.expect("ch", "(")
            off = np.asarray(self.sys.res_atom_offset); lo, hi = self._range(len(off) - 1); self.expect("ch", ")")
            if self.peek() == ("ch", ",") and hi - lo > 1:
                return [np.arange(off[r], off[r + 1], dtype=np.int32) for r in range(lo, hi)]
        self.i = save
        return None

    def single_selection(self) -> np.ndarray:
        """a selection argument where the reference would treat an ARRAY of selections differently from their union (one position per
        selection: coordinate_extract :1414): residue(a:b) over several residues standing alone is rejected instead of being flattened"""
        save = self.i
        if self.peek() == ("id", "residue"):
            self.next(); self.expect("ch", "(")
            lo, hi = self._range(len(np.asarray(self.sys.res_atom_offset)) - 1); self.expect("ch", ")")
            if self.peek() in (("ch", ","), ("ch", ")")) and hi - lo > 1:
                raise ScriptError("an array of selections as one argument (one centre of mass per selection) is not lowered")
        self.i = save
        return self.selection()

    def _has_within_before_comma(self) -> bool:
        """does the argument that starts here (up to its top-level `,` or `)`) contain a within(...) call"""
        depth = 0
        for t in self.t[self.i:]:
            if t == ("ch", "("): depth += 1
            elif t == ("ch", ")"):
                if depth == 0: return False
                depth -= 1
            elif t == ("ch", ",") and depth == 0: return False
            elif t[0] == "id" and t[1] in _DYNAMIC: return True
        return False

    def groups_or_selection(self):
        """residue(a:b) over several residues standing alone -> list of index arrays (array of selections); anything else -> one index array"""
        save = self.i
        if self.peek() == ("id", "residue"):
            self.next(); self.expect("ch", "(")
            off = np.asarray(self.sys.res_atom_offset); lo, hi = self._range(len(off) - 1); self.expect("ch", ")")
            if self.peek() in (("ch", ","), ("ch", ")")) and hi - lo > 1:
                return [np.arange(off[r], off[r + 1], dtype=np.int32) for r in range(lo, hi)]
        self.i = save
        return self.selection()

    def sel_or_within(self, single=False):
        """a selection argument that may be a dynamic one: index array, or api.Within for `within([min:]max, sel)` [and static]"""
        if self._has_within_before_comma(): return self.dyn_arg()
        return self.single_selection() if single else self.selection()

    def number(self) -> float:
        return float(self.expect("num")[1])

    def radius(self):
        """radius | min:max -> (min, max)"""
        a = self.number()
        if self.peek() == ("ch", ":"):
            self.next(); return a, self.number()
        return 0.0, a

    def index(self, flatten=False):
        """argument of distance/angle/dihedral/com: a 1-based atom index (-> int), a selection (-> index array, centre of mass) or an ARRAY of
        selections (residue(a:b) over several residues standing alone -> list of index arrays: the centre of the selections' centres,
        coordinate_extract_com :1826-1842). distance() is FLAG_FLATTEN (md_script_functions.inl:680): its arguments, com(...) inside it included,
        are evaluated flattened -> the union."""
        if self.peek()[0] == "num":
            v = int(float(self.expect("num")[1])) - 1   # md_script atom indices are 1-based
            self.arg_meta.append(("int", v)); return v
        if self.peek() == ("id", "com"):   # com(x) as an argument contributes the position x itself would (_com :4726 = coordinate_extract_com)
            self.next(); self.expect("ch", "("); a = self.index(flatten); self.expect("ch", ")")
            return a
        if self._has_within_before_comma(): self.arg_meta.append(("other",)); return self.sel_or_within()
        if self.peek() == ("id", "atom"):   # atom(a:b) standing alone: relative to the context when the expression is evaluated `in` contexts
            save = self.i; self.next(); self.expect("ch", "("); lo, hi = self._range(self.sys.num_atoms); self.expect("ch", ")")
            if self.peek() in (("ch", ","), ("ch", ")")): self.arg_meta.append(("atomrange", lo, hi))
            else: self.arg_meta.append(("other",))
            self.i = save
            return self.selection()
        ctx_relative = self._arg_mentions(("atom", "residue"))   # inside `in` contexts these count from the context's first atom / residue: only the shim
        a = self.selection() if flatten else self.groups_or_selection()   # (which asks mdlib's own evaluator per context) lowers such arguments
        self.arg_meta.append(("other",) if (isinstance(a, list) or ctx_relative) else ("sel", a))
        return a

    def _arg_mentions(self, names) -> bool:
        """does the argument that starts here (up to its top-level `,` or `)`) call one of `names`"""
        depth = 0
        for t in self.t[self.i:]:
            if t == ("ch", "("): depth += 1
            elif t == ("ch", ")"):
                if depth == 0: return False
                depth -= 1
            elif t == ("ch", ",") and depth == 0: return False
            elif t[0] == "id" and t[1] in names: return True
        return False

    def _is_call_statement(self) -> bool:
        """does the right-hand side that starts here consist of one procedure call (optionally `in` contexts)"""
        if self.peek()[0] != "id" or self.peek()[1] in _FUNCS or self.i + 1 >= len(self.t) or self.t[self.i + 1] != ("ch", "("): return False
        depth = 0
        for j in range(self.i + 1, len(self.t)):
            if self.t[j] == ("ch", "("): depth += 1
            elif self.t[j] == ("ch", ")"):
                depth -= 1
                if depth == 0: return j + 1 < len(self.t) and self.t[j + 1] in (("ch", ";"), ("id", "in"))
        return False

    def statement(self) -> api.Property:
        ident = self.expect("id")[1]; self.expect("ch", "=")
        if not self._is_call_statement(): return self.expression(ident)
        proc = self.expect("id")[1]; self.expect("ch", "(")
        return self.call(ident, proc)

    # ---- temporal expressions: the reference's tree (parse_arithmetic / fix_precedence, md_script.c:2314, :1196), then its operand order
    def expression(self, ident) -> api.Property:
        self.calls, self.ident = 0, ident
        tree = self._expr()
        if self.peek() == ("id", "in"): raise ScriptError("an expression inside `in` contexts is not lowered")
        self.expect("ch", ";")
        prog, n = self._emit(tree)
        p = api.expression(ident, prog); p.values_per_frame = max(n, 1)
        return p

    def _expr(self):
        """right-recursive as the reference parses: operand [op rest], `-` rest; each new node then goes through fix_precedence"""
        if self.peek() == ("ch", "-"):
            self.next(); node = ["neg", self._expr()]
            c = node[1]
            if c[0] in _PREC and c[0] != "neg" and _PREC[c[0]] > _PREC["neg"]: node = [c[0], ["neg", c[1]], c[2]]   # the unary branch rotates once
            return node
        lhs = self._operand()
        if self.peek()[0] == "ch" and self.peek()[1] in "+-*/":
            op = {"+": "add", "-": "sub", "*": "mul", "/": "div"}[self.next()[1]]
            return _fix([op, lhs, self._expr()])
        return lhs

    def _operand(self):
        tok = self.next()
        if tok == ("ch", "("):
            e = self._expr(); self.expect("ch", ")"); return ["paren", e]
        if tok[0] == "num": return ["const", float(np.float32(float(tok[1])))]   # an integer literal is cast to float by the front end
        if tok[0] != "id": raise ScriptError(f"unexpected token {tok[1]!r} in an expression")
        name = tok[1]
        if name in _CONSTANTS: return ["const", _CONSTANTS[name]]
        if self.peek() != ("ch", "("):
            if name not in self.known: raise ScriptError(f"'{name}' is not an earlier temporal property of the script")
            return ["prop", name]
        if name in _FUNCS:
            self.next(); args = [self._expr()]
            while self.peek() == ("ch", ","): self.next(); args.append(self._expr())
            self.expect("ch", ")")
            return ["func", name, args]
        self.next()   # an inline call of a procedure: a hidden property ident#k
        hidden = f"{self.ident}#{self.calls}"; self.calls += 1
        p = self.call(hidden, name, inline=True)
        if p.op in (api.OP_RDF, api.OP_SDF, api.OP_DENSITY_X, api.OP_DENSITY_Y, api.OP_DENSITY_Z): raise ScriptError("arithmetic on distributions and volumes is not lowered")
        self.hidden.append(p); self.known[hidden] = p
        return ["prop", hidden]

    def _emit(self, node):
        """postfix program and value count (0 = float) of a tree, with the reference's typing: `float op array` is applied as `array op float`
        (FLAG_SYMMETRIC_ARGS swaps the operands, md_script.c:3802); functions other than abs / floor / ceil take floats only"""
        k = node[0]
        if k == "paren": return self._emit(node[1])
        if k == "const": return [("const", node[1])], 0
        if k == "prop":
            n = _values_per_frame(self.known[node[1]])
            return [("prop", node[1])], (n if n > 1 else 0)
        if k == "neg":
            p, n = self._emit(node[1]); return p + [("neg",)], n
        if k == "func":
            name, args = node[1], node[2]
            if len(args) not in _FUNCS[name]: raise ScriptError(f"{name}() takes {' or '.join(map(str, _FUNCS[name]))} arguments")
            parts = [self._emit(a) for a in args]
            if any(n for _, n in parts) and name not in ("abs", "floor", "ceil"): raise ScriptError(f"{name}() takes floats only")
            kind = name if len(args) == 1 else {"atan": "atan2"}.get(name, name)
            return sum((p for p, _ in parts), []) + [(kind,)], max(n for _, n in parts)
        (pa, na), (pb, nb) = self._emit(node[1]), self._emit(node[2])
        if na and nb and na != nb: raise ScriptError(f"arrays of different lengths ({na} and {nb})")
        if nb and not na: pa, pb = pb, pa   # the symmetric match puts the array first
        return pa + pb + [(k,)], max(na, nb)

    def call(self, ident, proc, inline=False) -> api.Property:
        self.arg_meta = []   # how each argument of distance / angle / dihedral was written (index()): decides its meaning inside `in` contexts
        if proc == "rdf":
            wr = rr = None
            if self._has_within_before_comma():   # dynamic reference set: within([min:]max, selection) or a coordinate range, optionally `and` a static selection
                d = self.dyn_arg()
                if isinstance(d, api.Range): rr = d
                else: wlo, wr, wsel, wand = d.radius_min, d.radius, d.sel, d.and_idx
            grp = self.groups() if (wr is None and rr is None) else None
            ref = rr if rr is not None else (None if (grp is not None or wr is not None) else self.selection())
            self.expect("ch", ",")
            trg = self.sel_or_within() if self._has_within_before_comma() else self.groups_or_selection()   # an array of selections as target: one centre of mass each
            self.expect("ch", ",")
            a = self.number(); lo, hi = 0.0, a
            if self.peek() == ("ch", ":"):
                self.next(); lo, hi = a, self.number()
            if (wr is not None or rr is not None) and isinstance(trg, list): raise ScriptError("a dynamic reference set with an array of selections as target is not lowered")
            if wr is not None: p = api.rdf(ident, api.Within(wr, wsel, wlo, wand), trg, hi, lo) if isinstance(trg, (api.Within, api.Range)) else api.rdf_within(ident, wr, wsel, trg, hi, lo, wlo, wand)
            else: p = api.rdf_com(ident, grp, trg, hi, lo) if grp is not None else api.rdf(ident, ref, trg, hi, lo)
        elif proc == "sdf":
            st = self.structures(); self.expect("ch", ","); trg = self.sel_or_within(); self.expect("ch", ","); c = self.number()
            p = api.sdf(ident, st, trg, c)
        elif proc in ("density_x", "density_y", "density_z"):
            p = api.density(ident, "xyz".index(proc[-1]), self.sel_or_within())
        elif proc == "distance_pair":   # an array of selections (residue(a:b) over several residues) is one centre of mass per selection
            a = self.groups_or_selection(); self.expect("ch", ","); b = self.groups_or_selection()
            p = api.distance_pair(ident, a, b)
        elif proc in ("distance_min", "distance_max"):
            a = self.sel_or_within() if self._has_within_before_comma() else self.groups_or_selection(); self.expect("ch", ",")   # an array of selections: one centre of mass per selection
            b = self.sel_or_within() if self._has_within_before_comma() else self.groups_or_selection()
            p = {"distance_min": api.distance_min, "distance_max": api.distance_max}[proc](ident, a, b)
        elif proc == "contact_count":   # contact_count(A[], B, cutoff): the only registered signature (md_script_functions.inl:705); _contact_count's path length stays at its default 4 (:2762)
            a = self.groups_or_selection(); self.expect("ch", ","); b = self.selection(); self.expect("ch", ","); c = self.number()
            if self.peek() == ("ch", ","): raise ScriptError("Could not find matching procedure 'contact_count' which takes four arguments")
            p = api.contact_count(ident, a if isinstance(a, list) else [a], b, c, self.sys, 4)
        elif proc == "count":   # count(<dynamic selection> [, 'atom' | 'residue' | 'chain' | 'structure']): the selection is evaluated per frame on the device
            if not self._has_within_before_comma(): raise ScriptError("count() is lowered for within(...) and within_x / _y / _z / _xyz(...) expressions only")
            d = self.dyn_arg(); kind = "atom"
            if self.peek() == ("ch", ","):   # _count_with_arg (md_script_functions.inl:5536): an unknown type fails at compile time
                self.next(); kind = self.expect("str")[1]
                if kind not in api.COUNT_TYPES: raise ScriptError(f"Unknown argument: '{kind}', valid arguments are: {', '.join(api.COUNT_TYPES)}")
            if kind == "atom": p = api.count_range(ident, d) if isinstance(d, api.Range) else api.count_within(ident, d.radius, d.sel, d.radius_min, d.and_idx)
            else:
                try: groups = api.count_groups_of(self.sys, kind)
                except ValueError as e: raise ScriptError(str(e)) from None
                p = api.count_groups(ident, d, groups)
        elif proc in ("coord_x", "coord_y", "coord_z"):
            a = self.index()   # an array of selections: one value per selection (its centre of mass, coordinate_extract :1503)
            p = api.coord(ident, "xyz".index(proc[-1]), a if isinstance(a, list) else ([a] if np.ndim(a) == 0 else a))
        elif proc == "com":
            p = api.com(ident, self.index())
        elif proc == "plane":
            p = api.plane(ident, self.groups_or_selection())   # an array of selections: the plane through their centres of mass
        elif proc == "rmsd":
            ctx_relative = self._arg_mentions(("atom", "residue"))   # inside `in` contexts these count from the context's first atom / residue: shim only
            p = api.rmsd(ident, self.selection())   # an array of selections is flattened into their union (_internal_flatten_bf :4305)
        elif proc == "porosity":   # an array of selections is flattened into their union (:5888-5891); within() is not lowered here
            if self._has_within_before_comma(): raise ScriptError("porosity() of a dynamic selection is not lowered")
            p = api.porosity(ident, self.selection())
        elif proc == "distance":
            a = self.index(True); self.expect("ch", ","); b = self.index(True); p = api.distance(ident, a, b)
        elif proc == "angle":
            a = self.index(); self.expect("ch", ","); b = self.index(); self.expect("ch", ","); c = self.index(); p = api.angle(ident, a, b, c)
        elif proc == "dihedral":
            v = [self.index()]
            for _ in range(3): self.expect("ch", ","); v.append(self.index())
            p = api.dihedral(ident, *v)
        else:
            raise ScriptError(f"procedure '{proc}' is outside the GPU hot-path scope")
        self.expect("ch", ")")
        if inline: return p
        if self.peek() == ("id", "in"):   # `expr in contexts` (evaluate_context md_script.c:3418): one value per context
            self.next(); begs, ends = self.contexts()
            if proc == "rmsd":   # one fit per context of the atoms of (selection AND context)
                if ctx_relative: raise ScriptError("a context-relative argument of rmsd() inside `in` contexts is lowered by the md_script shim only")
                sel = np.asarray(p.idx[0], np.int64)
                p = api.rmsd(ident, [sel[(sel >= b) & (sel < e)].astype(np.int32) for b, e in zip(begs, ends)])
                self.expect("ch", ";")
                return p
            if proc not in ("distance", "angle", "dihedral") or any(m[0] == "other" for m in self.arg_meta) or len(self.arg_meta) != len(p.idx):
                raise ScriptError("`in` is lowered for distance / angle / dihedral with integer or selection arguments, and for rmsd")
            args = []
            for m in self.arg_meta:
                if m[0] == "int":   # remap_index_to_context rejects indices outside the context (md_script_functions.inl:1023-1040)
                    if np.any(begs + m[1] >= ends): raise ScriptError(f"supplied index ({m[1] + 1}) is not within the range of a context")
                    args.append(m[1])
                elif m[0] == "atomrange":   # atom(a:b) inside a context is relative to the context's first atom
                    if np.any(begs + m[2] > ends): raise ScriptError(f"supplied range ({m[1] + 1}:{m[2]}) is not within range of its context")
                    args.append([np.arange(b + m[1], b + m[2], dtype=np.int32) for b in begs])
                else:               # a selection: in context c the centre of mass of (selection AND context) (coordinate_extract_com with ctx->mol_ctx, :1812-1823)
                    sel = np.asarray(m[1], np.int64)
                    args.append([sel[(sel >= b) & (sel < e)].astype(np.int32) for b, e in zip(begs, ends)])
            p = api.in_contexts(ident, p.op, args, begs)
        self.expect("ch", ";")
        return p

    def contexts(self):
        """right-hand side of `in`: residue(a:b) | residue(:) | resname('X') -> (first atom, one past the last atom) of each context (md_bitfield beg_bit / end_bit)"""
        off = np.asarray(self.sys.res_atom_offset)
        f = self.expect("id")[1]; self.expect("ch", "(")
        if f == "residue":
            lo, hi = self._range(len(off) - 1); self.expect("ch", ")")
            return off[lo:hi].astype(np.int64), off[lo + 1:hi + 1].astype(np.int64)
        if f == "resname":
            if self.sys.resname is None: raise ScriptError("system has no residue data")
            pats = [self.expect("str")[1]]
            while self.peek() == ("ch", ","): self.next(); pats.append(self.expect("str")[1])
            self.expect("ch", ")")
            rn = np.asarray(self.sys.resname); hit = np.zeros(len(rn), bool)
            for pt in pats: hit |= np.array([fnmatch.fnmatchcase(r, pt) for r in rn])
            return off[:-1][hit].astype(np.int64), off[1:][hit].astype(np.int64)
        raise ScriptError(f"unsupported context expression '{f}'")


_PREC = {"neg": 2, "mul": 3, "div": 3, "add": 4, "sub": 4}   # operator_precedence (md_script.c:502)
_FUNCS = {f: (1,) for f in ("sqrt", "cbrt", "abs", "floor", "ceil", "cos", "sin", "asin", "acos", "log", "exp", "log2", "exp2", "log10")}
_FUNCS.update(atan=(1, 2), atan2=(2,), pow=(2,), min=(2,), max=(2,))
_CONSTANTS = {"PI": float(np.float32(3.14159265358)), "TAU": float(np.float32(6.28318530718)), "E": float(np.float32(2.71828182845))}   # md_script_functions.inl:456-466


def _fix(node):
    """fix_precedence (md_script.c:1196) on a new binary node whose right child was parsed first: rotate while the right child binds looser or
    equally (left to right), then fix the new left child"""
    c = node[2]
    if c[0] in _PREC and c[0] != "neg" and (_PREC[c[0]] >= _PREC[node[0]]):
        node = [c[0], [node[0], node[1], c[1]], c[2]]
        node[1] = _fix(node[1])
    return node


def _values_per_frame(p: api.Property) -> int:
    """values per frame of a temporal property, 0 for a distribution or volume"""
    if p.op in (api.OP_RDF, api.OP_SDF, api.OP_DENSITY_X, api.OP_DENSITY_Y, api.OP_DENSITY_Z): return 0
    if p.op == api.OP_EXPRESSION: return p.values_per_frame
    if p.op == api.OP_COM: return 3
    if p.op == api.OP_PLANE: return 4
    if p.op == api.OP_DISTANCE_PAIR:
        n = [len(o) - 1 if o is not None else int(np.size(i)) for o, i in ((p.structure_offsets, p.idx[0]), (p.structure_offsets_b, p.idx[1]))]
        return n[0] * n[1]
    if p.op in (api.OP_COORD_X, api.OP_COORD_Y, api.OP_COORD_Z): return p.num_structures or int(np.size(p.idx[0]))
    if p.op in (api.OP_DISTANCE, api.OP_ANGLE, api.OP_DIHEDRAL, api.OP_RMSD, api.OP_CONTACT_COUNT): return max(p.num_structures, 1)
    return 1


def compile_script(src: str, system: api.System) -> List[api.Property]:
    """`md_script_ir_compile_from_source` stand-in for the supported statement subset. The procedure calls inside temporal expressions become
    hidden properties (named ident#k) after the script's own, as the md_script shim appends them."""
    ps = _Parser(_tokens(src), system); out = []
    ps.known, ps.hidden = {}, []
    while ps.peek()[0] != "eof":
        p = ps.statement()
        if _values_per_frame(p): ps.known[p.name] = p
        out.append(p)
    if not out:
        raise ScriptError("No properties present in ir")
    return out + ps.hidden
