"""Host-side Python mirror of the md_script evaluation API on top of the libmdgpu C ABI (include/mdgpu.h).

The reference's API for this path (mdlib/src/md_script.h:226-253):
    md_script_eval_create(num_frames, ir, alloc)      -> Plan(system, properties, num_frames)
    md_script_eval_clear_data(eval)                   -> Plan.clear()
    md_script_eval_frame_range(eval, ir, sys, traj, beg, end) -> Plan.eval_frame_range(traj, beg, end)
    md_script_eval_property_data(eval, name)          -> Plan.property_data(name)
    md_script_eval_frame_mask / _interrupt            -> Plan.frame_mask() / Plan.interrupt()
Everything here is ctypes plumbing: the compute path is the CUDA library, and there is deliberately no CPU fallback —
if libmdgpu.so cannot be loaded or no CUDA device is present the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmdgpu.so")

DIST_BINS = 1024
VOL_DIM = 128

OP_RDF, OP_SDF, OP_DENSITY_X, OP_DENSITY_Y, OP_DENSITY_Z, OP_DISTANCE, OP_ANGLE, OP_DIHEDRAL, OP_DISTANCE_MIN, OP_DISTANCE_MAX, OP_RMSD, OP_DISTANCE_PAIR, OP_COM, OP_PLANE, OP_WITHIN_COUNT, OP_SHAPE_WEIGHTS, OP_COORD_X, OP_COORD_Y, OP_COORD_Z, OP_BACKBONE_ANGLES, OP_CONTACT_COUNT, OP_POROSITY = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22
OP_EXPRESSION = 23
OP_SECONDARY_STRUCTURE = 24
# node kinds of a temporal expression's postfix program (MDGPU_EXPR_*): operands, then operators and functions
EXPR_KINDS = {k: i for i, k in enumerate(("const", "prop", "neg", "add", "sub", "mul", "div", "sqrt", "cbrt", "abs", "floor", "ceil", "cos", "sin", "asin",
                                          "acos", "atan", "log", "exp", "log2", "exp2", "log10", "atan2", "pow", "min", "max"))}
EXPR_MAX_DEPTH = 16
CELL_ORTHO, CELL_TRICLINIC, CELL_PBC_X, CELL_PBC_Y, CELL_PBC_Z, CELL_PBC_ALL = 1, 2, 4, 8, 16, 28


class MdgpuError(RuntimeError):
    pass


class UnitCell(C.Structure):
    """md_unitcell_t (md_types.h:254-259)."""
    _fields_ = [("x", C.c_double), ("xy", C.c_double), ("xz", C.c_double), ("y", C.c_double), ("yz", C.c_double),
                ("z", C.c_double), ("flags", C.c_uint32)]

    @staticmethod
    def from_basis(x, y, z, xy=0.0, xz=0.0, yz=0.0):
        """md_unitcell_from_basis_parameters (md_unitcell.inl:12-31)."""
        flags = 0
        if xy == 0.0 and xz == 0.0 and yz == 0.0:
            if not (x == 0.0 and y == 0.0 and z == 0.0) and not (x == 1.0 and y == 1.0 and z == 1.0):
                flags |= CELL_ORTHO
        else:
            flags |= CELL_TRICLINIC
        if flags:
            if x != 0.0: flags |= CELL_PBC_X
            if y != 0.0: flags |= CELL_PBC_Y
            if z != 0.0: flags |= CELL_PBC_Z
        return UnitCell(float(x), float(xy), float(xz), float(y), float(yz), float(z), flags)

    @staticmethod
    def none():
        return UnitCell(0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0)


class FrameHeader(C.Structure):
    _fields_ = [("num_atoms", C.c_size_t), ("index", C.c_int64), ("timestamp", C.c_double), ("unitcell", UnitCell)]


class _SystemDesc(C.Structure):
    _fields_ = [("num_atoms", C.c_size_t), ("atom_mass", C.POINTER(C.c_float)), ("bond_conn_offset", C.POINTER(C.c_uint32)),
                ("bond_conn_atom_idx", C.POINTER(C.c_int32)), ("bond_conn_offset_count", C.c_size_t),
                ("atom_radius", C.POINTER(C.c_float))]


class _DynArg(C.Structure):   # mdgpu_dynamic_arg_t
    _fields_ = [("radius_min", C.c_float), ("radius_max", C.c_float), ("and_idx", C.POINTER(C.c_int32)), ("and_count", C.c_size_t), ("has_and", C.c_uint32)]


class _RangeArg(C.Structure):   # mdgpu_range_arg_t
    _fields_ = [("prop", C.c_uint32), ("arg", C.c_uint32), ("lo", C.c_float * 3), ("hi", C.c_float * 3)]


class _ExprNode(C.Structure):   # mdgpu_expr_node_t
    _fields_ = [("kind", C.c_uint32), ("value", C.c_float), ("prop", C.c_uint32)]


class _Expr(C.Structure):   # mdgpu_expr_t
    _fields_ = [("prop", C.c_uint32), ("nodes", C.POINTER(_ExprNode)), ("num_nodes", C.c_size_t)]


class _PropertyDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("op", C.c_uint32), ("idx", C.POINTER(C.c_int32) * 4), ("idx_count", C.c_size_t * 4),
                ("num_structures", C.c_size_t), ("structure_size", C.c_size_t), ("cutoff_min", C.c_float), ("cutoff_max", C.c_float),
                ("structure_offsets", C.POINTER(C.c_uint32)), ("com_args", C.c_uint32), ("ref_within_radius", C.c_float), ("ref_within_min", C.c_float),
                ("structure_offsets_b", C.POINTER(C.c_uint32)), ("num_structures_b", C.c_size_t), ("dyn", _DynArg * 4),
                ("arg_offsets", C.POINTER(C.c_uint32) * 4), ("arg_parts", C.c_uint32 * 4)]


class _PropertyData(C.Structure):
    _fields_ = [("dim", C.c_int32 * 4), ("num_values", C.c_size_t), ("values", C.POINTER(C.c_float)), ("weights", C.POINTER(C.c_float)),
                ("min_value", C.c_float), ("max_value", C.c_float), ("min_range", C.c_float * 2), ("max_range", C.c_float * 2),
                ("frames_accumulated", C.c_uint64)]


class _PlanOptions(C.Structure):
    _fields_ = [("device", C.c_int), ("batch_frames", C.c_uint32), ("num_streams", C.c_uint32), ("keep_frame_results", C.c_uint32),
                ("cell_capacity", C.c_uint32), ("rdf_variant", C.c_uint32), ("ingest_mode", C.c_uint32), ("ingest_threads", C.c_uint32),
                ("num_devices", C.c_uint32), ("devices", C.c_int32 * 16)]


# md_trajectory_i-compatible callback table (md_trajectory.h:49-67)
class _Reader(C.Structure):
    pass


_LOAD_FRAME = C.CFUNCTYPE(C.c_bool, C.c_void_p, C.c_int64, C.POINTER(FrameHeader), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float))
_READER_FREE = C.CFUNCTYPE(None, C.POINTER(_Reader))
_Reader._fields_ = [("inst", C.c_void_p), ("free", _READER_FREE), ("load_frame", _LOAD_FRAME)]


class _TrajHeader(C.Structure):
    _fields_ = [("num_frames", C.c_size_t), ("num_atoms", C.c_size_t), ("unit_bits", C.c_uint64), ("unit_mult", C.c_double),
                ("frame_times", C.POINTER(C.c_double))]


class _Traj(C.Structure):
    pass


_GET_HEADER = C.CFUNCTYPE(C.c_bool, C.c_void_p, C.POINTER(_TrajHeader))
_INIT_READER = C.CFUNCTYPE(C.c_bool, C.POINTER(_Reader), C.c_void_p)
_TRAJ_FREE = C.CFUNCTYPE(None, C.POINTER(_Traj))
_Traj._fields_ = [("inst", C.c_void_p), ("free", _TRAJ_FREE), ("get_header", _GET_HEADER), ("init_reader", _INIT_READER)]

PROGRESS_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.c_uint32)   # mdgpu_progress_fn
_lib = None


def lib() -> C.CDLL:
    """Load libmdgpu.so (built in-tree by viamd_b200/build.py). Raises if missing: there is no fallback implementation."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MdgpuError(f"{LIB_PATH} not found: build it with `python -m viamd_b200.build` (or __graft_entry__.build())")
        L = C.CDLL(LIB_PATH)
        L.mdgpu_last_error.restype = C.c_char_p
        L.mdgpu_plan_create.restype = C.c_void_p
        L.mdgpu_plan_create.argtypes = [C.POINTER(_SystemDesc), C.POINTER(_PropertyDesc), C.c_size_t, C.c_size_t, C.POINTER(_PlanOptions)]
        L.mdgpu_plan_create_with_ranges.restype = C.c_void_p
        L.mdgpu_plan_create_with_ranges.argtypes = [C.POINTER(_SystemDesc), C.POINTER(_PropertyDesc), C.c_size_t, C.c_size_t, C.POINTER(_PlanOptions),
                                                    C.POINTER(_RangeArg), C.c_size_t]
        L.mdgpu_plan_create_ex.restype = C.c_void_p
        L.mdgpu_plan_create_ex.argtypes = [C.POINTER(_SystemDesc), C.POINTER(_PropertyDesc), C.c_size_t, C.c_size_t, C.POINTER(_PlanOptions),
                                           C.POINTER(_RangeArg), C.c_size_t, C.POINTER(_Expr), C.c_size_t]
        L.mdgpu_plan_destroy.argtypes = [C.c_void_p]
        L.mdgpu_plan_destroy.restype = None
        L.mdgpu_plan_clear.argtypes = [C.c_void_p]
        L.mdgpu_plan_set_initial_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(UnitCell)]
        for name in ("mdgpu_eval_device_frames", "mdgpu_eval_host_frames"):
            getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32]
        L.mdgpu_eval_trajectory.argtypes = [C.c_void_p, C.POINTER(_Traj), C.c_uint32, C.c_uint32, C.c_uint32]
        L.mdgpu_plan_sync.argtypes = [C.c_void_p]
        L.mdgpu_plan_interrupt.argtypes = [C.c_void_p]
        L.mdgpu_plan_interrupt.restype = None
        L.mdgpu_plan_property_count.argtypes = [C.c_void_p]
        L.mdgpu_plan_property_count.restype = C.c_size_t
        L.mdgpu_plan_property_index.argtypes = [C.c_void_p, C.c_char_p]
        L.mdgpu_plan_property_data.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(_PropertyData)]
        L.mdgpu_plan_property_counts.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.mdgpu_plan_property_aggregate.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.mdgpu_plan_property_frame_counts.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        L.mdgpu_plan_frame_mask.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.mdgpu_plan_mark_frames_done.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.mdgpu_plan_property_frame_rows.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]
        L.mdgpu_plan_property_accum_ptr.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]
        L.mdgpu_plan_set_frames_accumulated.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64]
        L.mdgpu_launch_count.argtypes = [C.c_bool]
        L.mdgpu_launch_count.restype = C.c_uint64
        L.mdgpu_plan_enable_kernel_timing.argtypes = [C.c_void_p, C.c_int]
        L.mdgpu_plan_timer_begin.argtypes = [C.c_void_p]
        L.mdgpu_plan_timer_end.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.mdgpu_plan_kernel_time_ms.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        L.mdgpu_synth_water_desc.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
        L.mdgpu_synth_water_base.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        L.mdgpu_synth_water_frames_host.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_size_t]
        L.mdgpu_synth_water_frames_device.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_size_t]
        L.mdgpu_device_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
        L.mdgpu_device_free.argtypes = [C.c_int, C.c_void_p]
        L.mdgpu_host_alloc_pinned.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
        L.mdgpu_host_free_pinned.argtypes = [C.c_void_p]
        L.mdgpu_memcpy_h2d.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]
        L.mdgpu_memcpy_d2h.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]
        L.mdgpu_device_synchronize.argtypes = [C.c_int]
        L.mdgpu_plan_bind_property_storage.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        L.mdgpu_plan_set_progress_callback.argtypes = [C.c_void_p, PROGRESS_FN, C.c_void_p]
        L.mdgpu_bind_host_to_device.argtypes = [C.c_int]
        L.mdgpu_plan_exchange_stats.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]
        L.mdgpu_plan_ingest_info.argtypes = [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]
        _lib = L
    return _lib


def _check(rc: int) -> None:
    if rc != 0:
        raise MdgpuError(f"mdgpu error {rc}: {lib().mdgpu_last_error().decode(errors='replace')}")


def bind_host_to_device(device: int = 0) -> int:
    """pin this thread (and threads created later) to the CPUs next to `device`; returns the CPU count, or a negative status when sysfs has none"""
    return int(lib().mdgpu_bind_host_to_device(int(device)))


def device_count() -> int:
    return int(lib().mdgpu_device_count())


def launch_count(reset: bool = False) -> int:
    return int(lib().mdgpu_launch_count(reset))


# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class System:
    """What the per-frame procedures read from md_system_t: masses and covalent-bond connectivity, plus optional
    atom metadata (element symbol, atom name, residue name / residue atom offsets) used by viamd_b200.script selections."""
    num_atoms: int
    mass: np.ndarray
    conn_offset: Optional[np.ndarray] = None
    conn_idx: Optional[np.ndarray] = None
    element: Optional[Sequence[str]] = None
    name: Optional[Sequence[str]] = None
    resname: Optional[Sequence[str]] = None        # per residue
    res_atom_offset: Optional[np.ndarray] = None   # [num_res + 1]
    radius: Optional[np.ndarray] = None            # van der Waals radii (md_atom_extract_radii); required by porosity()
    chain_atom_range: Optional[np.ndarray] = None  # [num_chains, 2] (first atom, one past the last) of each instance (md_system_instance_atom_range);
                                                   # required by count(x, 'chain')


@dataclass
class Property:
    name: str
    op: int
    idx: list = field(default_factory=list)   # up to 4 int32 arrays
    num_structures: int = 0
    structure_size: int = 0
    cutoff_min: float = 0.0
    cutoff_max: float = 0.0
    structure_offsets: Optional[np.ndarray] = None   # rdf_com: CSR offsets of the groups in idx[0]
    com_args: int = 0                                # distance/angle/dihedral: bit k = argument k is a selection (centre of mass)
    ref_within: float = 0.0                          # rdf: > 0 -> references = within([ref_within_min:]ref_within, idx[0]) evaluated per frame
    ref_within_min: float = 0.0
    structure_offsets_b: Optional[np.ndarray] = None  # distance_pair: CSR groups of argument 1 (argument 0 uses structure_offsets)
    dyn: dict = field(default_factory=dict)           # {k: (radius_min, radius_max, and_idx | None)}: argument k is within([min:]max, idx[k]) [and and_idx], per frame
    arg_offsets: dict = field(default_factory=dict)   # {k: CSR offsets}: argument k of distance / angle / dihedral / com is an ARRAY of selections (centre of their centres)
    ranges: dict = field(default_factory=dict)        # {k: Range}: argument k is a coordinate range within_x / _y / _z / _xyz(...) [and static], per frame
    program: Optional[list] = None                    # OP_EXPRESSION: the postfix program, see expression()


class Within:
    """within([radius_min:]radius, selection) [and a static selection] as a property argument: the atoms of the system within reach of the
    selection in each frame, the selection itself excluded (md_script_functions.inl:2485-2720) — evaluated per frame on the device."""

    def __init__(self, radius, sel_idx, radius_min=0.0, and_idx=None):
        self.radius, self.radius_min = float(radius), float(radius_min)
        self.sel = np.asarray(sel_idx, np.int32); self.and_idx = None if and_idx is None else np.asarray(and_idx, np.int32)


FLT_MAX = float(np.finfo(np.float32).max)


class Range:
    """within_x(a:b) / within_y / within_z / within_xyz(a:b, c:d, e:f) [and a static selection] as a property argument (coordinate_range
    md_script_functions.inl:2394): per frame the atoms with lo <= (x, y, z) <= hi on every axis, by their raw coordinates; unconstrained axes are
    [-FLT_MAX, FLT_MAX]. and_idx: the static side of `selection and within_*(...)` (None: no static side). Evaluated per frame on the device."""

    def __init__(self, lo, hi, and_idx=None):
        self.lo = np.asarray(lo, np.float32).reshape(3); self.hi = np.asarray(hi, np.float32).reshape(3)
        self.and_idx = None if and_idx is None else np.asarray(and_idx, np.int32)

    @staticmethod
    def axis(axis, lo, hi, and_idx=None):
        """within_x / _y / _z (axis 0 / 1 / 2)"""
        l = [-FLT_MAX] * 3; h = [FLT_MAX] * 3; l[axis] = lo; h[axis] = hi
        return Range(l, h, and_idx)

    def mask(self, x, y, z):
        """the selection of one frame (numpy, the reference's comparison)"""
        m = (self.lo[0] <= x) & (x <= self.hi[0]) & (self.lo[1] <= y) & (y <= self.hi[1]) & (self.lo[2] <= z) & (z <= self.hi[2])
        if self.and_idx is not None:
            keep = np.zeros(len(m), bool); keep[self.and_idx] = True; m &= keep
        return m


def _split_dyn(args, ranges=None):
    """[index array | Within | Range, ...] -> (idx lists, dyn dict); the coordinate ranges go to `ranges` (their idx list stays empty)"""
    idx, dyn = [], {}
    for k, a in enumerate(args):
        if isinstance(a, Within): idx.append(a.sel); dyn[k] = (a.radius_min, a.radius, a.and_idx)
        elif isinstance(a, Range): idx.append(np.zeros(0, np.int32)); ranges[k] = a
        else: idx.append(np.asarray(a, np.int32))
    return idx, dyn


def _trg_groups(trg):
    """a target that is a LIST of index arrays is an ARRAY of selections: one centre of mass per selection is the target point (coordinate_extract
    md_script_functions.inl:1503 -> extract_com :857; compute_rdf :5293-5302). Returns (concatenated indices | the argument itself, CSR offsets | None)."""
    if not isinstance(trg, list): return trg, None
    groups = [np.asarray(g, np.int32) for g in trg]
    if len(groups) == 1: return groups[0], None
    off = np.zeros(len(groups) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in groups])
    return np.concatenate(groups).astype(np.int32), off


def rdf(name, ref_idx, trg_idx, cutoff, cutoff_min=0.0):
    """ref_idx / trg_idx: atom index arrays, or Within(...) for a selection evaluated per frame; trg_idx may be a list of index arrays (an array of
    selections: their centres of mass are the targets)"""
    trg_idx, toff = _trg_groups(trg_idx)
    rng = {}; idx, dyn = _split_dyn([ref_idx, trg_idx], rng)
    return Property(name, OP_RDF, idx, cutoff_min=float(cutoff_min), cutoff_max=float(cutoff), dyn=dyn, structure_offsets_b=toff, ranges=rng)


def rdf_within(name, radius, sel_idx, trg_idx, cutoff, cutoff_min=0.0, radius_min=0.0, and_idx=None):
    """rdf(within(radius, selection), targets, cutoff): the reference atoms are the dynamic selection within() of each frame — every atom of the
    system within `radius` of the selection, the selection itself excluded (md_script_functions.inl:2485) — then compute_rdf as usual."""
    idx = [np.asarray(sel_idx, np.int32), np.asarray(trg_idx, np.int32)] + ([np.asarray(and_idx, np.int32)] if and_idx is not None else [])
    return Property(name, OP_RDF, idx, cutoff_min=float(cutoff_min), cutoff_max=float(cutoff), ref_within=float(radius), ref_within_min=float(radius_min),
                    com_args=0 if and_idx is None else 1)   # and_idx: the static side of `selection and within(...)`


def rdf_com(name, groups, trg_idx, cutoff, cutoff_min=0.0):
    """rdf() whose reference argument is an ARRAY of selections (e.g. residue(1:100)): references are the groups' centres of mass
    and a group's own atoms are excluded from its pairs (compute_rdf md_script_functions.inl:5274-5275, rdf_cb_excl_mask :5243)."""
    groups = [np.asarray(g, np.int32) for g in groups]
    off = np.zeros(len(groups) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in groups])
    trg_idx, toff = _trg_groups(trg_idx)   # targets may be an array of selections too: with the reference's exclusion test on the target ORDINAL (rdf_cb_excl_mask :5252)
    return Property(name, OP_RDF, [np.concatenate(groups).astype(np.int32), np.asarray(trg_idx, np.int32)], num_structures=len(groups),
                    cutoff_min=float(cutoff_min), cutoff_max=float(cutoff), structure_offsets=off, structure_offsets_b=toff)


def sdf(name, structures, trg_idx, cutoff):
    """sdf(): structures is [num_structures, structure_size] atom indices, each row strictly ascending (an atom set, as the reference's
    bitfields give it; Plan() raises MdgpuError for a row that is not, repeated atoms included). Row 0 of the initial frame is the
    reference orientation; the target atoms are counted in a 128^3 volume around each structure, its own atoms excluded."""
    s = np.ascontiguousarray(structures, np.int32)
    assert s.ndim == 2, "structures: [num_structures, structure_size] atom indices"
    rng = {}; idx, dyn = _split_dyn([s.reshape(-1), trg_idx], rng)
    return Property(name, OP_SDF, idx, num_structures=s.shape[0], structure_size=s.shape[1], cutoff_max=float(cutoff), dyn=dyn, ranges=rng)


def density(name, axis, idx):
    rng = {}; lst, dyn = _split_dyn([idx], rng)
    return Property(name, OP_DENSITY_X + int(axis), lst, dyn=dyn, ranges=rng)


def in_contexts(name, op, local_idx, context_first_atoms):
    """`name = distance|angle|dihedral(i, j, ...) in <contexts>`: the integer arguments (0-based here) are relative to each context's first atom
    (remap_index_to_context); an argument given as a LIST of index arrays (one per context) is a selection: the atoms of (selection AND context),
    whose centre of mass is the position. One value per context and frame -> [F, n_contexts] (evaluate_context md_script.c:3418)."""
    beg = np.asarray(context_first_atoms, np.int64)
    idx, parts, mask = [], {}, 0
    for k, a in enumerate(local_idx):
        if isinstance(a, list):   # a selection argument: per context the atoms of (selection AND context); its position there is their centre of mass
            assert len(a) == len(beg)
            off = np.zeros(len(a) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in a])
            idx.append(np.concatenate(a).astype(np.int32) if off[-1] else np.zeros(0, np.int32)); parts[k] = off; mask |= 1 << k
        else: idx.append((beg + int(a)).astype(np.int32))
    return Property(name, op, idx, num_structures=len(beg), com_args=mask, arg_offsets=parts)


def _temporal(name, op, args):
    """each argument: an int (0-based atom index -> that atom's position) or an index array (a selection -> centre of mass,
    coordinate_extract_com md_script_functions.inl:1717)"""
    idx, mask, dyn, parts, rng = [], 0, {}, {}, {}
    for k, a in enumerate(args):
        if isinstance(a, Within): idx.append(a.sel); mask |= 1 << k; dyn[k] = (a.radius_min, a.radius, a.and_idx)   # the frame's dynamic selection: its centre of mass
        elif isinstance(a, Range): idx.append(np.zeros(0, np.int32)); mask |= 1 << k; rng[k] = a
        elif isinstance(a, list):   # an ARRAY of selections: the centre of the selections' centres (coordinate_extract_com :1826-1842)
            sels = [np.asarray(g, np.int32) for g in a]; mask |= 1 << k
            if len(sels) == 1: idx.append(sels[0])
            else:
                off = np.zeros(len(sels) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in sels])
                idx.append(np.concatenate(sels).astype(np.int32)); parts[k] = off
        elif np.ndim(a) == 0: idx.append(np.asarray([int(a)], np.int32))
        else: idx.append(np.asarray(a, np.int32)); mask |= 1 << k
    return Property(name, op, idx, com_args=mask, dyn=dyn, arg_offsets=parts, ranges=rng)


def distance(name, a, b):
    return _temporal(name, OP_DISTANCE, (a, b))


def _groups_or_idx(args):
    """index array -> (array, None); LIST of index arrays (an array of selections: one centre of mass each, extract_com :857) -> (concatenated, CSR offsets)"""
    idx, offs = [], []
    for arg in args:
        if isinstance(arg, (list, tuple)) and len(arg) > 1:
            g = [np.asarray(x, np.int32) for x in arg]; off = np.zeros(len(g) + 1, np.uint32); off[1:] = np.cumsum([len(x) for x in g])
            idx.append(np.concatenate(g).astype(np.int32)); offs.append(off)
        else: idx.append(arg[0] if isinstance(arg, (list, tuple)) else arg); offs.append(None)
    return idx, offs


def _min_distance(name, op, a_idx, b_idx):
    (a_idx, b_idx), offs = _groups_or_idx([a_idx, b_idx])
    rng = {}; idx, dyn = _split_dyn([a_idx, b_idx], rng)
    return Property(name, op, idx, dyn=dyn, num_structures=0 if offs[0] is None else len(offs[0]) - 1, structure_offsets=offs[0], structure_offsets_b=offs[1], ranges=rng)


def distance_min(name, a_idx, b_idx):
    """distance_min(a, b): smallest pair distance between the atoms of two selections (md_script_functions.inl:3892); an argument given as a LIST of
    index arrays is an array of selections: its positions are the selections' centres of mass (coordinate_extract :1503)"""
    return _min_distance(name, OP_DISTANCE_MIN, a_idx, b_idx)


def distance_max(name, a_idx, b_idx):
    """distance_max(a, b): the reference evaluates md_util_min_distance here as well (md_script_functions.inl:3944) — reproduced"""
    return _min_distance(name, OP_DISTANCE_MAX, a_idx, b_idx)


def distance_pair(name, a, b):
    """distance_pair(a, b): all |a| x |b| pair distances per frame, a temporal with |a|*|b| values per frame (md_script_functions.inl:3972).
    a / b: an index array (the atoms of one selection) or a LIST of index arrays (an array of selections: one centre of mass each, extract_com :857)."""
    idx, offs = [], []
    for arg in (a, b):
        if isinstance(arg, (list, tuple)):
            g = [np.asarray(x, np.int32) for x in arg]; off = np.zeros(len(g) + 1, np.uint32); off[1:] = np.cumsum([len(x) for x in g])
            idx.append(np.concatenate(g).astype(np.int32)); offs.append(off)
        else: idx.append(np.asarray(arg, np.int32)); offs.append(None)
    return Property(name, OP_DISTANCE_PAIR, idx, num_structures=0 if offs[0] is None else len(offs[0]) - 1, structure_offsets=offs[0], structure_offsets_b=offs[1])


def com(name, a):
    """com(x): [F, 3] — the position of an atom (int) or the periodic centre of mass of a selection (index array), as distance() sees its arguments"""
    return _temporal(name, OP_COM, (a,))


def plane(name, idx):
    """plane(selection): [F, 4] — unit normal of the best-fit plane through the atoms (third principal axis) and normal . centre (_plane :4755);
    a LIST of index arrays (an array of selections) fits the plane through the selections' centres of mass"""
    (idx,), offs = _groups_or_idx([idx])
    return Property(name, OP_PLANE, [np.asarray(idx, np.int32)], num_structures=0 if offs[0] is None else len(offs[0]) - 1, structure_offsets=offs[0])


def count_within(name, radius, sel_idx, radius_min=0.0, and_idx=None):
    """count(within(radius, selection)): per frame, the number of atoms of the system within `radius` of any atom of the selection, the
    selection itself excluded (_within_expl_flt md_script_functions.inl:2485, _count :2868) — a dynamic selection evaluated on the device"""
    idx = [np.asarray(sel_idx, np.int32)] + ([np.zeros(0, np.int32), np.asarray(and_idx, np.int32)] if and_idx is not None else [])
    return Property(name, OP_WITHIN_COUNT, idx, cutoff_min=float(radius_min), cutoff_max=float(radius), com_args=0 if and_idx is None else 1)   # min:max form: _within_expl_frng :2609


def count_range(name, rng: Range):
    """count(within_x / _y / _z / _xyz(...) [and static]): per frame the number of atoms in the coordinate range (coordinate_range
    md_script_functions.inl:2394, _count :2868) — MDGPU_OP_WITHIN_COUNT with the range as dyn[0]"""
    return Property(name, OP_WITHIN_COUNT, [np.zeros(0, np.int32)], ranges={0: rng})


COUNT_TYPES = ("atom", "residue", "chain", "structure")   # count_type_str (md_script_functions.inl:5448-5452); 'chain' counts instances


def count_groups_of(system: System, count_type: str) -> list:
    """the groups count(x, count_type) counts over (internal_count md_script_functions.inl:5465-5531), as atom index arrays:
    'residue' the residues of System.res_atom_offset, 'chain' the instances of System.chain_atom_range, 'structure' the connected components of
    the bond graph in the order md_util_system_infer_structures finds them (a breadth-first walk from every atom not yet visited; an atom without
    bonds is a structure of its own, and a system without bonds has no structures)."""
    if count_type == "residue":
        off = np.asarray(system.res_atom_offset, np.int64)
        return [np.arange(off[i], off[i + 1], dtype=np.int32) for i in range(len(off) - 1)]
    if count_type == "chain":
        if system.chain_atom_range is None: raise ValueError("count(x, 'chain'): the system has no chain atom ranges (System.chain_atom_range)")
        return [np.arange(int(b), int(e), dtype=np.int32) for b, e in np.asarray(system.chain_atom_range, np.int64).reshape(-1, 2)]
    if count_type == "structure":
        if system.conn_offset is None or len(system.conn_idx) == 0: return []
        co = np.asarray(system.conn_offset, np.int64); ci = np.asarray(system.conn_idx, np.int64)
        seen = np.zeros(system.num_atoms, bool); out = []
        for i in range(system.num_atoms):
            if seen[i]: continue
            seen[i] = True; order = [i]; head = 0
            while head < len(order):
                a = order[head]; head += 1
                for b in ci[co[a]:co[a + 1]] if a + 1 < len(co) else ():
                    if not seen[b]: seen[b] = True; order.append(int(b))
            out.append(np.asarray(order, np.int32))
        return out
    raise ValueError(f"unknown count type {count_type!r}; valid types are {', '.join(COUNT_TYPES)}")


def count_groups(name, sel, groups):
    """count(x, 'residue' | 'chain' | 'structure'): per frame the number of groups (atom index arrays, each atom in at most one) that hold an
    atom of the dynamic selection x — Within(...) or Range(...), optionally with its static `and` side (internal_count md_script_functions.inl:5465).
    MDGPU_OP_WITHIN_COUNT with bit 1 of com_args: the groups back to back in idx[1], their CSR offsets in structure_offsets."""
    base = count_range(name, sel) if isinstance(sel, Range) else count_within(name, sel.radius, sel.sel, sel.radius_min, sel.and_idx)
    groups = [np.asarray(g, np.int32) for g in groups]
    off = np.zeros(len(groups) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in groups])
    idx = list(base.idx) + [np.zeros(0, np.int32)] * (2 - len(base.idx))
    idx[1] = np.concatenate(groups).astype(np.int32) if off[-1] else np.zeros(0, np.int32)
    base.idx = idx; base.com_args |= 2; base.num_structures = len(groups); base.structure_offsets = off
    return base


def shape_weights(name, groups, use_mass=True):
    """(linear, planar, isotropic) shape weights of every structure and frame -> [F, n*3]: what VIAMD's shape-space component evaluates per frame
    (shapespace.cpp:404-431; `use_mass` is its checkbox) and what _shape_weights returns (md_script_functions.inl:6005)."""
    groups = [np.asarray(g, np.int32) for g in groups]
    off = np.zeros(len(groups) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in groups])
    return Property(name, OP_SHAPE_WEIGHTS, [np.concatenate(groups).astype(np.int32)], num_structures=len(groups), structure_offsets=off, com_args=1 if use_mass else 0)


def coord(name, axis, idx):
    """coord_x / coord_y / coord_z(selection): the atoms' coordinates along `axis` -> [F, n] (md_script_functions.inl:5077); a LIST of index arrays
    (an array of selections) yields one value per selection, the coordinate of its centre of mass (coordinate_extract :1503)"""
    (idx,), offs = _groups_or_idx([idx])
    return Property(name, OP_COORD_X + int(axis), [np.asarray(idx, np.int32)], num_structures=0 if offs[0] is None else len(offs[0]) - 1, structure_offsets=offs[0])


def grow_by_bonds(atoms, conn_offset, conn_idx, extent: int):
    """md_util_mask_grow_by_bonds (md_util.c:5537-5595) as intended: every atom within `extent` bonds of the given atoms (the reference walks
    a depth array it never zeroes; with zeroed memory it is this breadth-first search)."""
    atoms = [int(a) for a in atoms]
    if not atoms or conn_offset is None: return np.asarray(sorted(atoms), np.int32)
    depth = {a: 0 for a in atoms}; queue = list(atoms)
    while queue:
        a = queue.pop(0)
        if depth[a] >= extent: continue
        for k in range(int(conn_offset[a]), int(conn_offset[a + 1])):
            b = int(conn_idx[k])
            if b not in depth or depth[a] + 1 < depth[b]:
                depth[b] = depth[a] + 1; queue.append(b)
    return np.asarray(sorted(depth), np.int32)


def contact_count(name, groups, b_idx, cutoff, system: "System" = None, path_length: int = 4):
    """contact_count(A[], B, cutoff [, path_length]): per frame and set A_i the pairs (a in A_i, b in B) within the cutoff, b outside the set's
    exclusion list = (A_i & B) grown by `path_length` bonds (md_script_functions.inl:2756-2866); the values of a frame are RUNNING totals over
    the sets, as the reference's never-reset counter produces them. -> temporal [F, |A|]"""
    groups = [np.asarray(g, np.int32) for g in groups]; b = np.unique(np.asarray(b_idx, np.int32))
    off = np.zeros(len(groups) + 1, np.uint32); off[1:] = np.cumsum([len(g) for g in groups])
    excl = []
    for g in groups:
        ov = np.intersect1d(g, b)
        excl.append(grow_by_bonds(ov, None if system is None else system.conn_offset, None if system is None else system.conn_idx, path_length) if len(ov) else np.zeros(0, np.int32))
    eoff = np.zeros(len(groups) + 1, np.uint32); eoff[1:] = np.cumsum([len(e) for e in excl])
    return Property(name, OP_CONTACT_COUNT, [np.concatenate(groups).astype(np.int32), b, np.concatenate(excl).astype(np.int32) if eoff[-1] else np.zeros(0, np.int32)],
                    num_structures=len(groups), cutoff_max=float(cutoff), structure_offsets=off, structure_offsets_b=eoff)


def backbone_angles(name, five):
    """(phi, psi) of every backbone segment per frame (MDGPU_OP_BACKBONE_ANGLES): `five` is [n_segments, 5] = atoms C(i-1), N, CA, C, N(i+1) of each segment,
    -1 rows for segments without angles (chain ends). The property is [F, 2 * n_segments] = md_backbone_angles_t per segment."""
    five = np.ascontiguousarray(five, np.int32).reshape(-1, 5)
    return Property(name, OP_BACKBONE_ANGLES, [five.reshape(-1)], num_structures=len(five))


def secondary_structure(name, atoms, range_offsets):
    """The secondary structure of every backbone segment per frame (MDGPU_OP_SECONDARY_STRUCTURE, md_util_backbone_secondary_structure_infer):
    `atoms` is [n_segments, 5] = N, CA, C, O, HN of each segment (md_protein_backbone_data_t::segment.atoms; HN -1 when estimated),
    `range_offsets` the backbone ranges (chains) as range.count + 1 ascending offsets from 0 to n_segments. The property is [F, n_segments]
    md_secondary_structure_t codes as floats; Plan.secondary_structure returns them as int32."""
    atoms = np.ascontiguousarray(atoms, np.int32).reshape(-1, 5)
    return Property(name, OP_SECONDARY_STRUCTURE, [atoms.reshape(-1)], num_structures=len(atoms),
                    structure_offsets_b=np.ascontiguousarray(range_offsets, np.uint32))


def rmsd(name, idx):
    """rmsd(selection): mass-weighted RMSD of the selection's atoms against the initial frame after wrap, bond-walk unwrap and an optimal
    rotation (_rmsd md_script_functions.inl:4287). Needs System.conn_offset / conn_idx to make molecules whole, as the reference does.
    A LIST of index arrays is `rmsd(x) in <contexts>`: one group per context (the atoms of x AND the context), each fitted on its own -> [F, n];
    an empty group evaluates to 0."""
    if isinstance(idx, list):
        g = [np.asarray(x, np.int32) for x in idx]
        off = np.zeros(len(g) + 1, np.uint32); off[1:] = np.cumsum([len(x) for x in g])
        return Property(name, OP_RMSD, [np.concatenate(g).astype(np.int32) if off[-1] else np.zeros(0, np.int32)], num_structures=len(g), structure_offsets=off)
    return Property(name, OP_RMSD, [np.asarray(idx, np.int32)])


def expression(name, program):
    """A temporal expression: arithmetic and math functions over other temporal properties of the plan, evaluated per frame on the device
    (operators md_script_functions.inl:505-571, functions :576-603; MDGPU_OP_EXPRESSION). `program` is postfix, a list of nodes:
    ("const", value) | ("prop", name or index of a temporal property of the same plan) | (kind,) for kind in EXPR_KINDS — "neg", "add", "sub",
    "mul", "div" and the functions. Element-wise on arrays as the reference: see include/mdgpu.h (mdgpu_expr_t) for the rules."""
    prog = []
    for n in program:
        if n[0] not in EXPR_KINDS: raise ValueError(f"unknown expression node {n!r}")
        prog.append((n[0], float(n[1]) if n[0] == "const" else 0.0, n[1] if n[0] == "prop" else None))
    return Property(name, OP_EXPRESSION, program=prog)


def porosity(name, idx):
    """porosity(selection): per frame, the unoccupied fraction of a bit grid (longest axis 512 voxels) over the bounding box of the selection's van
    der Waals spheres (_porosity md_script_functions.inl:5858). Needs System.radius. 0 for a triclinic cell or an empty selection."""
    return Property(name, OP_POROSITY, [np.asarray(idx, np.int32)])


def angle(name, a, b, c):
    return _temporal(name, OP_ANGLE, (a, b, c))


def dihedral(name, a, b, c, d):
    return _temporal(name, OP_DIHEDRAL, (a, b, c, d))


@dataclass
class PropertyData:
    """md_script_property_data_t view (md_script.h:73-92)."""
    name: str
    dim: tuple
    values: np.ndarray
    weights: Optional[np.ndarray]
    min_value: float
    max_value: float
    min_range: tuple
    max_range: tuple
    frames_accumulated: int


class Trajectory:
    """Python frame source exposed to the library through the md_trajectory_i vtable (md_trajectory.h:56-67).
    Subclass and implement num_frames / num_atoms / load_frame(idx) -> (x, y, z, UnitCell)."""

    def num_frames(self) -> int: raise NotImplementedError
    def num_atoms(self) -> int: raise NotImplementedError
    def load_frame(self, idx: int): raise NotImplementedError

    def _as_c(self):
        if getattr(self, "_c_traj", None) is not None:   # one vtable per trajectory object: concurrent evaluations share it (the callbacks must outlive every call)
            return self._c_traj
        n = self.num_atoms()

        def get_header(inst, hdr):
            hdr[0].num_frames = self.num_frames(); hdr[0].num_atoms = n; hdr[0].unit_bits = 0; hdr[0].unit_mult = 0.0
            hdr[0].frame_times = None
            return True

        def load_frame(inst, idx, hdr, px, py, pz):
            try:
                x, y, z, cell = self.load_frame(int(idx))
            except Exception:
                return False
            if hdr:
                hdr[0].num_atoms = n; hdr[0].index = idx; hdr[0].timestamp = float(idx); hdr[0].unitcell = cell
            if px:
                C.memmove(px, np.ascontiguousarray(x, np.float32).ctypes.data, 4 * n)
                C.memmove(py, np.ascontiguousarray(y, np.float32).ctypes.data, 4 * n)
                C.memmove(pz, np.ascontiguousarray(z, np.float32).ctypes.data, 4 * n)
            return True

        def reader_free(r):
            return None

        self._cb_load = _LOAD_FRAME(load_frame); self._cb_rfree = _READER_FREE(reader_free)

        def init_reader(reader, inst):
            reader[0].inst = 1; reader[0].free = self._cb_rfree; reader[0].load_frame = self._cb_load
            return True

        def traj_free(t):
            return None

        self._cb_hdr = _GET_HEADER(get_header); self._cb_init = _INIT_READER(init_reader); self._cb_tfree = _TRAJ_FREE(traj_free)
        t = _Traj(); t.inst = 1; t.free = self._cb_tfree; t.get_header = self._cb_hdr; t.init_reader = self._cb_init
        self._c_traj = t
        return t


class ArrayTrajectory(Trajectory):
    """In-memory trajectory: frames [F,3,N] float32, cells: list of UnitCell (or one cell for all frames)."""

    def __init__(self, frames: np.ndarray, cells):
        self.frames = np.ascontiguousarray(frames, np.float32)
        self.cells = cells

    def num_frames(self): return self.frames.shape[0]
    def num_atoms(self): return self.frames.shape[2]

    def load_frame(self, idx):
        c = self.cells if isinstance(self.cells, UnitCell) else self.cells[idx]
        return self.frames[idx, 0], self.frames[idx, 1], self.frames[idx, 2], c


class Plan:
    """md_script_eval_t equivalent: owns device accumulators and the host-visible property data."""

    def __init__(self, system: System, properties: Sequence[Property], num_frames: int, device: int = 0, batch_frames: int = 0,
                 num_streams: int = 0, keep_frame_results: bool = False, cell_capacity: int = 0, rdf_variant: int = 0,
                 ingest_mode: int = 0, ingest_threads: int = 0, devices: Optional[Sequence[int]] = None):
        """devices: more than one CUDA ordinal -> ONE process drives several GPUs (frame blocks per device, one NCCL reduce at sync)."""
        L = lib()
        if devices is not None and len(devices) == 1: device, devices = int(devices[0]), None
        self.system, self.properties, self.num_frames, self.device = system, list(properties), int(num_frames), int(devices[0] if devices else device)
        self._keep = []
        mass = np.ascontiguousarray(system.mass, np.float32); self._keep.append(mass)
        sd = _SystemDesc(); sd.num_atoms = system.num_atoms; sd.atom_mass = mass.ctypes.data_as(C.POINTER(C.c_float))
        if system.conn_offset is not None:
            co = np.ascontiguousarray(system.conn_offset, np.uint32); ci = np.ascontiguousarray(system.conn_idx, np.int32); self._keep += [co, ci]
            sd.bond_conn_offset = co.ctypes.data_as(C.POINTER(C.c_uint32)); sd.bond_conn_atom_idx = ci.ctypes.data_as(C.POINTER(C.c_int32))
            sd.bond_conn_offset_count = len(co)
        if system.radius is not None:
            rad = np.ascontiguousarray(system.radius, np.float32); self._keep.append(rad)
            if rad.shape != (system.num_atoms,): raise ValueError("System.radius: one radius per atom expected")
            sd.atom_radius = rad.ctypes.data_as(C.POINTER(C.c_float))
        descs = (_PropertyDesc * len(self.properties))(); ranges = []
        for i, p in enumerate(self.properties):
            d = descs[i]; nm = p.name.encode(); self._keep.append(nm)
            d.name = nm; d.op = p.op; d.num_structures = p.num_structures; d.structure_size = p.structure_size
            d.cutoff_min = p.cutoff_min; d.cutoff_max = p.cutoff_max
            d.com_args = p.com_args; d.ref_within_radius = p.ref_within; d.ref_within_min = p.ref_within_min
            if p.structure_offsets is not None:
                so = np.ascontiguousarray(p.structure_offsets, np.uint32); self._keep.append(so)
                d.structure_offsets = so.ctypes.data_as(C.POINTER(C.c_uint32))
            if p.structure_offsets_b is not None:
                sb = np.ascontiguousarray(p.structure_offsets_b, np.uint32); self._keep.append(sb)
                d.structure_offsets_b = sb.ctypes.data_as(C.POINTER(C.c_uint32)); d.num_structures_b = len(sb) - 1
            for k, arr in enumerate(p.idx):
                a = np.ascontiguousarray(arr, np.int32); self._keep.append(a)
                d.idx[k] = a.ctypes.data_as(C.POINTER(C.c_int32)); d.idx_count[k] = a.size
            for k, off in p.arg_offsets.items():
                ao = np.ascontiguousarray(off, np.uint32); self._keep.append(ao)
                d.arg_offsets[k] = ao.ctypes.data_as(C.POINTER(C.c_uint32)); d.arg_parts[k] = len(ao) - 1
            for k, r in p.ranges.items():   # beside the descriptors: mdgpu_range_arg_t; the static side in dyn[k]
                ranges.append((i, k, r))
                if r.and_idx is not None:
                    m = np.ascontiguousarray(r.and_idx, np.int32); self._keep.append(m)
                    d.dyn[k].and_idx = m.ctypes.data_as(C.POINTER(C.c_int32)); d.dyn[k].and_count = m.size; d.dyn[k].has_and = 1
            for k, (rmin, rmax, and_idx) in p.dyn.items():
                d.dyn[k].radius_min = rmin; d.dyn[k].radius_max = rmax
                if and_idx is not None:
                    m = np.ascontiguousarray(and_idx, np.int32); self._keep.append(m)
                    d.dyn[k].and_idx = m.ctypes.data_as(C.POINTER(C.c_int32)); d.dyn[k].and_count = m.size; d.dyn[k].has_and = 1
        o = _PlanOptions(); o.device = device; o.batch_frames = batch_frames; o.num_streams = num_streams
        o.keep_frame_results = 1 if keep_frame_results else 0; o.cell_capacity = cell_capacity; o.rdf_variant = rdf_variant
        o.ingest_mode = ingest_mode; o.ingest_threads = ingest_threads
        if devices:
            o.num_devices = len(devices)
            for g, dv in enumerate(devices): o.devices[g] = int(dv)
        rarr = (_RangeArg * len(ranges))()
        for j, (i, k, r) in enumerate(ranges):
            rarr[j].prop = i; rarr[j].arg = k
            for c in range(3): rarr[j].lo[c] = float(r.lo[c]); rarr[j].hi[c] = float(r.hi[c])
        exprs = [(i, p.program) for i, p in enumerate(self.properties) if p.program is not None]
        if exprs:   # beside the descriptors: mdgpu_expr_t, operands named by property index
            index = {p.name: i for i, p in enumerate(self.properties)}
            earr = (_Expr * len(exprs))()
            for j, (i, prog) in enumerate(exprs):
                nodes = (_ExprNode * len(prog))(); self._keep.append(nodes)
                for m, (kind, value, ref) in enumerate(prog):
                    nodes[m].kind = EXPR_KINDS[kind]; nodes[m].value = value
                    if kind == "prop": nodes[m].prop = index[ref] if isinstance(ref, str) else int(ref)
                earr[j].prop = i; earr[j].nodes = nodes; earr[j].num_nodes = len(prog)
            self._h = L.mdgpu_plan_create_ex(C.byref(sd), descs, len(self.properties), self.num_frames, C.byref(o), rarr, len(ranges), earr, len(exprs))
        elif ranges:
            self._h = L.mdgpu_plan_create_with_ranges(C.byref(sd), descs, len(self.properties), self.num_frames, C.byref(o), rarr, len(ranges))
        else:
            self._h = L.mdgpu_plan_create(C.byref(sd), descs, len(self.properties), self.num_frames, C.byref(o))
        if not self._h:
            raise MdgpuError(L.mdgpu_last_error().decode(errors="replace"))
        self._names = [p.name for p in self.properties]

    def close(self):
        if getattr(self, "_h", None):
            lib().mdgpu_plan_destroy(self._h); self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self): return self
    def __exit__(self, *a): self.close()

    # -- md_script_eval_* mirror
    def clear(self): _check(lib().mdgpu_plan_clear(self._h))
    def interrupt(self): lib().mdgpu_plan_interrupt(self._h)
    def sync(self): _check(lib().mdgpu_plan_sync(self._h))

    def set_progress_callback(self, fn):
        """fn(frame_beg, frame_count) after every completed batch (mdgpu_plan_set_progress_callback); None removes it."""
        self._progress = PROGRESS_FN(lambda user, b, n: fn(int(b), int(n))) if fn else PROGRESS_FN(0)
        _check(lib().mdgpu_plan_set_progress_callback(self._h, self._progress, None))

    def bind_property_storage(self, name, values: np.ndarray, agg_mean=None, agg_var=None, agg_ext=None):
        """results of `name` are written into `values` (float32, C-contiguous) from now on (mdgpu_plan_bind_property_storage)"""
        assert values.dtype == np.float32 and values.flags.c_contiguous
        self._keep += [values, agg_mean, agg_var, agg_ext]
        ptr = lambda a: None if a is None else a.ctypes.data
        _check(lib().mdgpu_plan_bind_property_storage(self._h, self._index(name), values.ctypes.data, values.size, ptr(agg_mean), ptr(agg_var), ptr(agg_ext)))

    def histogram(self, name, num_bins: int, range_min: float, range_max: float, aggregate: bool = False):
        """VIAMD's compute_histogram_masked (src/main.cpp:172-226) of a temporal over the evaluated frames, counted on the device: ([rows, num_bins], (min, max))"""
        i = self._index(name); dim = self.properties[i].num_structures if False else None
        d = self.property_data(name); rows = 1 if aggregate else int(d.dim[1])
        out = np.zeros((rows, num_bins), np.float32); mm = np.zeros(2, np.float32)
        lib().mdgpu_plan_property_histogram.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
        _check(lib().mdgpu_plan_property_histogram(self._h, i, num_bins, range_min, range_max, 1 if aggregate else 0, out.ctypes.data, mm.ctypes.data))
        return out, (float(mm[0]), float(mm[1]))

    def rama_density(self, name, classes, frame_beg: int = 0, frame_end: Optional[int] = None, sigma: float = 5.0):
        """VIAMD's Ramachandran density maps (rama_rep_compute_density) from the backbone-angles property `name`, computed on the device over the
        evaluated frames of [frame_beg, frame_end). classes: four arrays of segment indices (general, glycine, proline, pre-proline).
        Returns (tex [512, 512, 4] float32 indexed [y, x, class], sums [4] float32 samples per class)."""
        i = self._index(name)
        if len(classes) != 4:
            raise ValueError("classes: four arrays of segment indices (general, glycine, proline, pre-proline)")
        lists = [np.ascontiguousarray(c, np.int64).ravel() for c in classes]
        if any(len(c) and (c.min() < 0 or c.max() > 0xFFFFFFFF) for c in lists):
            raise ValueError("classes: segment indices must be non-negative 32-bit integers")
        seg = np.ascontiguousarray(np.concatenate(lists), np.uint32)
        off = np.zeros(5, np.uint32); off[1:] = np.cumsum([len(c) for c in lists])
        tex = np.zeros((512, 512, 4), np.float32); sums = np.zeros(4, np.float32)
        end = self.num_frames if frame_end is None else int(frame_end)
        L = lib(); L.mdgpu_plan_rama_density.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_void_p, C.c_void_p]
        _check(L.mdgpu_plan_rama_density(self._h, i, seg.ctypes.data if seg.size else None, off.ctypes.data, int(frame_beg), end, float(sigma),
                                          tex.ctypes.data, sums.ctypes.data))
        return tex, sums

    def secondary_structure(self, name, frame_beg: int = 0, frame_end: Optional[int] = None):
        """The rows of secondary-structure property `name` for frames [frame_beg, frame_end) as int32 md_secondary_structure_t [frames, n_segments]
        (mdgpu_plan_secondary_structure); frames not evaluated yet are 0 (unknown)."""
        i = self._index(name)
        end = self.num_frames if frame_end is None else int(frame_end)
        S = int(self.properties[i].num_structures)   # the segment count the property was built with
        out = np.zeros((max(end - int(frame_beg), 0), S), np.int32)
        L = lib(); L.mdgpu_plan_secondary_structure.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]
        _check(L.mdgpu_plan_secondary_structure(self._h, i, int(frame_beg), end, out.ctypes.data if out.size else None))
        return out

    def exchange_stats(self):
        ms = C.c_double(); n = C.c_uint64(); _check(lib().mdgpu_plan_exchange_stats(self._h, C.byref(ms), C.byref(n))); return ms.value, int(n.value)

    def ingest_info(self):
        a = C.c_size_t(); t = C.c_uint32(); _check(lib().mdgpu_plan_ingest_info(self._h, C.byref(a), C.byref(t))); return int(a.value), int(t.value)

    def set_initial_frame(self, x, y, z, cell: UnitCell):
        x, y, z = (np.ascontiguousarray(a, np.float32) for a in (x, y, z))
        _check(lib().mdgpu_plan_set_initial_frame(self._h, x.ctypes.data, y.ctypes.data, z.ctypes.data, C.byref(cell)))

    @staticmethod
    def _cells_arg(cells, count):
        if isinstance(cells, UnitCell):
            arr = (UnitCell * 1)(cells); return arr, 0
        arr = (UnitCell * count)(*cells[:count]); return arr, C.sizeof(UnitCell)

    def eval_host_frames(self, frames: np.ndarray, cells, frame_beg: int = 0):
        """frames: [F,3,N] float32 host array (numpy, or any object exposing .ctypes.data / __array_interface__)."""
        frames = np.ascontiguousarray(frames, np.float32); F, _, N = frames.shape
        carr, cstride = self._cells_arg(cells, F)
        _check(lib().mdgpu_eval_host_frames(self._h, frames.ctypes.data, 3 * N, N, C.addressof(carr), cstride, frame_beg, F))

    def eval_host_ptr(self, ptr: int, frame_stride: int, axis_stride: int, cells, frame_beg: int, count: int):
        carr, cstride = self._cells_arg(cells, count)
        _check(lib().mdgpu_eval_host_frames(self._h, ptr, frame_stride, axis_stride, C.addressof(carr), cstride, frame_beg, count))

    def eval_device_frames(self, d_ptr: int, frame_stride: int, axis_stride: int, cells, frame_beg: int, count: int):
        carr, cstride = self._cells_arg(cells, count)
        _check(lib().mdgpu_eval_device_frames(self._h, d_ptr, frame_stride, axis_stride, C.addressof(carr), cstride, frame_beg, count))

    def eval_xtc_frames(self, blob: np.ndarray, offsets: np.ndarray, frame_beg: int = 0):
        """XTC frames (bytes as in the file + frame offsets): compressed bytes go to the device and are expanded there"""
        blob = np.ascontiguousarray(blob, np.uint8); offsets = np.ascontiguousarray(offsets, np.uint64)
        lib().mdgpu_eval_xtc_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        _check(lib().mdgpu_eval_xtc_frames(self._h, blob.ctypes.data, offsets.ctypes.data, frame_beg, len(offsets) - 1))

    def eval_xtc_file(self, path: str, frame_beg: int, frame_end: int):
        """evaluate frames [frame_beg, frame_end) of an .xtc file (decoded on the device)"""
        lib().mdgpu_eval_xtc_file.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32]
        _check(lib().mdgpu_eval_xtc_file(self._h, path.encode(), frame_beg, frame_end))

    def eval_xtc_ptr(self, blob_ptr: int, offsets: np.ndarray, frame_beg: int = 0):
        """as eval_xtc_frames, the bytes given as a raw host pointer (e.g. pinned memory)"""
        offsets = np.ascontiguousarray(offsets, np.uint64)
        lib().mdgpu_eval_xtc_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        _check(lib().mdgpu_eval_xtc_frames(self._h, blob_ptr, offsets.ctypes.data, frame_beg, len(offsets) - 1))

    def eval_frame_range(self, traj: Trajectory, frame_beg: int, frame_end: int, loader_threads: int = 1) -> bool:
        """md_script_eval_frame_range(eval, ir, sys, traj, beg, end) (md_script.c:6573): returns False on failure."""
        t = traj._as_c()
        rc = lib().mdgpu_eval_trajectory(self._h, C.byref(t), frame_beg, frame_end, loader_threads)
        if rc == 0:
            rc = lib().mdgpu_plan_sync(self._h)
        self._last_rc = rc
        return rc == 0

    def last_error(self) -> str:
        return lib().mdgpu_last_error().decode(errors="replace")

    def _index(self, name) -> int:
        if isinstance(name, int):
            return name
        i = lib().mdgpu_plan_property_index(self._h, name.encode())
        if i < 0:
            raise KeyError(name)
        return i

    def property_data(self, name) -> PropertyData:
        i = self._index(name); d = _PropertyData()
        _check(lib().mdgpu_plan_property_data(self._h, i, C.byref(d)))
        vals = np.ctypeslib.as_array(d.values, shape=(d.num_values,)).copy()
        dim = tuple(d.dim)
        weights = vals[dim[2]:2 * dim[2]].copy() if bool(d.weights) else None
        return PropertyData(self._names[i], dim, vals, weights, float(d.min_value), float(d.max_value), tuple(d.min_range), tuple(d.max_range), int(d.frames_accumulated))

    def aggregate(self, name) -> dict:
        """per-frame mean / population variance / (min, max) of a temporal with several values per frame (md_script_aggregate_t)"""
        i = self._index(name); F = self.num_frames
        mean = np.zeros(F, np.float32); var = np.zeros(F, np.float32); ext = np.zeros((F, 2), np.float32)
        _check(lib().mdgpu_plan_property_aggregate(self._h, i, mean.ctypes.data, var.ctypes.data, ext.ctypes.data, F))
        return dict(mean=mean, var=var, ext=ext)

    def counts(self, name) -> np.ndarray:
        i = self._index(name); op = self.properties[i].op
        n = VOL_DIM ** 3 if op == OP_SDF else DIST_BINS
        out = np.zeros(n, np.uint64)
        _check(lib().mdgpu_plan_property_counts(self._h, i, out.ctypes.data, n))
        return out

    def frame_counts(self, name, frame: int, want_bins: bool = True):
        i = self._index(name); bins = np.zeros(DIST_BINS, np.uint32) if want_bins else None; tot = C.c_uint64(0)
        _check(lib().mdgpu_plan_property_frame_counts(self._h, i, frame, bins.ctypes.data if want_bins else None, C.byref(tot)))
        return bins, int(tot.value)

    def frame_mask(self) -> np.ndarray:
        nw = (self.num_frames + 63) // 64; w = np.zeros(nw, np.uint64)
        _check(lib().mdgpu_plan_frame_mask(self._h, w.ctypes.data, nw))
        bits = np.unpackbits(w.view(np.uint8), bitorder="little")[: self.num_frames]
        return bits.astype(bool)

    def accum_ptr(self, name):
        i = self._index(name); p = C.c_void_p(); b = C.c_size_t(); e = C.c_uint32()
        _check(lib().mdgpu_plan_property_accum_ptr(self._h, i, C.byref(p), C.byref(b), C.byref(e)))
        return int(p.value), int(b.value), int(e.value)

    def frame_rows(self, name, which: int):
        """(device pointer, bytes, element bytes) of a per-frame integer row (0: totals, 1: frame minimum, 2: frame maximum), or (0, 0, 0)"""
        p = C.c_void_p(); n = C.c_size_t(); eb = C.c_uint32()
        _check(lib().mdgpu_plan_property_frame_rows(self._h, self._index(name), int(which), C.byref(p), C.byref(n), C.byref(eb)))
        return int(p.value or 0), int(n.value), int(eb.value)

    def mark_frames_done(self, frame_beg: int, count: int):
        """declare frames evaluated by other ranks done (after their temporal rows were reduced into this plan's buffers)"""
        _check(lib().mdgpu_plan_mark_frames_done(self._h, int(frame_beg), int(count)))

    def set_frames_accumulated(self, name, frames: int):
        _check(lib().mdgpu_plan_set_frames_accumulated(self._h, self._index(name), frames))

    def enable_kernel_timing(self, on=True): _check(lib().mdgpu_plan_enable_kernel_timing(self._h, 1 if on else 0))

    def timer_begin(self): _check(lib().mdgpu_plan_timer_begin(self._h))

    def timer_end(self) -> float:
        ms = C.c_double(); _check(lib().mdgpu_plan_timer_end(self._h, C.byref(ms))); return float(ms.value)

    def kernel_counter(self, which: int) -> int:
        v = C.c_uint64(); lib().mdgpu_plan_kernel_counter.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]
        _check(lib().mdgpu_plan_kernel_counter(self._h, which, C.byref(v))); return int(v.value)

    def kernel_time_ms(self, kernel="k_rdf_pairs"):
        ms = C.c_double(); n = C.c_uint64()
        _check(lib().mdgpu_plan_kernel_time_ms(self._h, kernel.encode(), C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)


# ----------------------------------------------------------------------------------------------------------------------
# synthetic workloads + raw memory helpers
def synth_water_desc(n: int, seed: int):
    na = C.c_uint32(); L = C.c_float()
    _check(lib().mdgpu_synth_water_desc(n, seed, C.byref(na), C.byref(L)))
    return int(na.value), float(L.value)


def synth_water_base(n: int, seed: int, want_whole: bool = False):
    na, L = synth_water_desc(n, seed)
    base = np.zeros((3, na), np.float32); whole = np.zeros((3, na), np.float32) if want_whole else None
    _check(lib().mdgpu_synth_water_base(n, seed, base.ctypes.data, whole.ctypes.data if want_whole else None))
    return (base, whole, L) if want_whole else (base, L)


def synth_water_frames_host(n: int, seed: int, base: np.ndarray, frame_beg: int, count: int, out: Optional[np.ndarray] = None) -> np.ndarray:
    na = base.shape[1]
    if out is None:
        out = np.empty((count, 3, na), np.float32)
    _check(lib().mdgpu_synth_water_frames_host(n, seed, np.ascontiguousarray(base, np.float32).ctypes.data, frame_beg, count, out.ctypes.data, 3 * na, na))
    return out


def synth_water_frames_device(device: int, n: int, seed: int, d_base: int, frame_beg: int, count: int, d_out: int, frame_stride: int, axis_stride: int):
    _check(lib().mdgpu_synth_water_frames_device(device, n, seed, d_base, frame_beg, count, d_out, frame_stride, axis_stride))


def device_alloc(device: int, nbytes: int) -> int:
    p = C.c_void_p(); _check(lib().mdgpu_device_alloc(device, nbytes, C.byref(p))); return int(p.value)


def device_free(device: int, ptr: int): _check(lib().mdgpu_device_free(device, ptr))


def host_alloc_pinned(nbytes: int) -> int:
    p = C.c_void_p(); _check(lib().mdgpu_host_alloc_pinned(nbytes, C.byref(p))); return int(p.value)


def host_free_pinned(ptr: int): _check(lib().mdgpu_host_free_pinned(ptr))
def memcpy_h2d(device, dst, src, nbytes): _check(lib().mdgpu_memcpy_h2d(device, dst, src, nbytes))
def memcpy_d2h(device, dst, src, nbytes): _check(lib().mdgpu_memcpy_d2h(device, dst, src, nbytes))
def device_synchronize(device=0): _check(lib().mdgpu_device_synchronize(device))


LIPID_BEADS = 12
LIPID_NAMES = ["NC3", "PO4", "GL1", "GL2", "C1A", "C2A", "C3A", "C4A", "C1B", "C2B", "C3B", "C4B"]


def synth_membrane_desc(nl: int, nw_xy: int, nwz: int, seed: int):
    na = C.c_uint32(); nlip = C.c_uint32(); L3 = (C.c_float * 3)()
    f = lib().mdgpu_synth_membrane_desc; f.argtypes = [C.c_uint32] * 4 + [C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
    _check(f(nl, nw_xy, nwz, seed, C.byref(na), C.byref(nlip), L3))
    return int(na.value), int(nlip.value), tuple(float(v) for v in L3)


def synth_membrane_base(nl: int, nw_xy: int, nwz: int, seed: int):
    na, nlip, L3 = synth_membrane_desc(nl, nw_xy, nwz, seed)
    base = np.zeros((3, na), np.float32); whole = np.zeros((3, na), np.float32); mol = np.zeros(na, np.uint32)
    f = lib().mdgpu_synth_membrane_base; f.argtypes = [C.c_uint32] * 4 + [C.c_void_p] * 3
    _check(f(nl, nw_xy, nwz, seed, base.ctypes.data, whole.ctypes.data, mol.ctypes.data))
    return base, whole, mol, L3


def synth_membrane_frames_host(nl, nw_xy, nwz, seed, base, mol, frame_beg, count):
    na = base.shape[1]; out = np.empty((count, 3, na), np.float32)
    f = lib().mdgpu_synth_membrane_frames_host; f.argtypes = [C.c_uint32] * 4 + [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_size_t]
    _check(f(nl, nw_xy, nwz, seed, np.ascontiguousarray(base, np.float32).ctypes.data, np.ascontiguousarray(mol, np.uint32).ctypes.data, frame_beg, count, out.ctypes.data, 3 * na, na))
    return out


def synth_membrane_frames_device(device, nl, nw_xy, nwz, seed, d_base, d_mol, frame_beg, count, d_out, frame_stride, axis_stride):
    f = lib().mdgpu_synth_membrane_frames_device
    f.argtypes = [C.c_int] + [C.c_uint32] * 4 + [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_size_t]
    _check(f(device, nl, nw_xy, nwz, seed, d_base, d_mol, frame_beg, count, d_out, frame_stride, axis_stride))


def membrane_system(nl: int, nw_xy: int, nwz: int, mass_lipid: float = 72.0, mass_water: float = 72.0) -> System:
    """Topology of the synthetic membrane: 12-bead lipids (residue LIP) then one-bead solvent residues (SOLW)."""
    nlip = 2 * nl * nl; nw = 2 * nwz * nw_xy * nw_xy; na = nlip * LIPID_BEADS + nw
    names = LIPID_NAMES * nlip + ["W"] * nw
    res_off = np.concatenate([np.arange(nlip, dtype=np.int64) * LIPID_BEADS, nlip * LIPID_BEADS + np.arange(nw + 1, dtype=np.int64)])
    mass = np.concatenate([np.full(nlip * LIPID_BEADS, mass_lipid, np.float32), np.full(nw, mass_water, np.float32)])
    return System(na, mass, None, None, element=["X"] * na, name=names, resname=["LIP"] * nlip + ["SOLW"] * nw, res_atom_offset=res_off)


def xtc_frame_offsets(blob: np.ndarray):
    """frame byte offsets [n+1] and the atom count of an XTC file image (md_xtc.c:436-570)"""
    blob = np.ascontiguousarray(blob, np.uint8); cap = max(2, blob.size // 56 + 2)
    offs = np.zeros(cap, np.uint64); n = C.c_size_t(); na = C.c_size_t()
    lib().mdgpu_xtc_frame_offsets.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    _check(lib().mdgpu_xtc_frame_offsets(blob.ctypes.data, blob.size, offs.ctypes.data, cap, C.byref(n), C.byref(na)))
    return offs[:n.value + 1].copy(), int(na.value)


def xtc_decode_frames(blob: np.ndarray, offsets: np.ndarray, num_atoms: int, device: int = 0):
    """device decode of XTC frames -> (xyz [F,3,N] float32 in Angstrom, cells [F], steps [F], times [F])"""
    blob = np.ascontiguousarray(blob, np.uint8); offsets = np.ascontiguousarray(offsets, np.uint64); F = len(offsets) - 1
    xyz = np.zeros((F, 3, num_atoms), np.float32); cells = (UnitCell * F)(); steps = np.zeros(F, np.int32); times = np.zeros(F, np.float32)
    lib().mdgpu_xtc_decode_frames.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    _check(lib().mdgpu_xtc_decode_frames(device, blob.ctypes.data, offsets.ctypes.data, F, num_atoms, xyz.ctypes.data, C.addressof(cells), steps.ctypes.data, times.ctypes.data))
    return xyz, list(cells), steps, times


def debug_sqrt_sweep(lo_bits: int, hi_bits: int, device: int = 0) -> int:
    n = C.c_uint64()
    lib().mdgpu_debug_sqrt_sweep.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]
    _check(lib().mdgpu_debug_sqrt_sweep(device, lo_bits, hi_bits, C.byref(n)))
    return int(n.value)


def debug_rdf_config() -> str:
    """the rdf candidate cull of this process (mdgpu_debug_rdf_config): full8 | full6 | full4 | half | flat6 | flat8 | flat4"""
    buf = C.create_string_buffer(16)
    lib().mdgpu_debug_rdf_config.argtypes = [C.c_char_p, C.c_size_t]
    _check(lib().mdgpu_debug_rdf_config(buf, len(buf)))
    return buf.value.decode()


def water_system(n: int) -> System:
    """Topology of the synthetic water box (OW,HW1,HW2 per molecule; masses as md_atom_extract_masses yields them)."""
    nm = n ** 3; na = 3 * nm
    mass = np.tile(np.array([15.9994, 1.00794, 1.00794], np.float32), nm)
    conn_off = np.zeros(na + 1, np.uint32); conn_idx = np.zeros(4 * nm, np.int32)
    # per molecule: O bonded to H1,H2; H1 -> O; H2 -> O
    per = np.array([0, 2, 3, 4], np.uint32)
    conn_off[:-1] = (np.repeat(np.arange(nm, dtype=np.uint32) * 4, 3) + np.tile(per[:3], nm))
    conn_off[-1] = 4 * nm
    o = np.arange(nm, dtype=np.int32) * 3
    conn_idx[0::4] = o + 1; conn_idx[1::4] = o + 2; conn_idx[2::4] = o; conn_idx[3::4] = o
    return System(na, mass, conn_off, conn_idx, element=["O", "H", "H"] * nm, name=["OW", "HW1", "HW2"] * nm,
                  resname=["SOL"] * nm, res_atom_offset=np.arange(nm + 1, dtype=np.int64) * 3)
