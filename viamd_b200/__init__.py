"""viamd_b200 — H100-native per-frame trajectory analysis behind VIAMD/mdlib's md_script property API.

The product is viamd_b200/libmdgpu.so (hand-written CUDA for sm_90a behind the C ABI in include/mdgpu.h); this package is
the thin host-side mirror of the md_script evaluation API used by the tests and bench.py.
"""
from .api import (  # noqa: F401
    MdgpuError, UnitCell, System, Property, PropertyData, Plan, Within, Range, Trajectory, ArrayTrajectory,
    rdf, rdf_com, rdf_within, sdf, density, distance, distance_min, distance_max, distance_pair, rmsd, porosity, com, plane, count_within, count_range, in_contexts, shape_weights, coord, angle, dihedral, expression, backbone_angles, secondary_structure, contact_count, water_system, device_count, bind_host_to_device, launch_count, lib,
    synth_membrane_desc, synth_membrane_base, synth_membrane_frames_host, synth_membrane_frames_device, membrane_system,
    synth_water_desc, synth_water_base, synth_water_frames_host, synth_water_frames_device,
    xtc_frame_offsets, xtc_decode_frames,
    device_alloc, device_free, host_alloc_pinned, host_free_pinned, memcpy_h2d, memcpy_d2h, device_synchronize,
    OP_RDF, OP_SDF, OP_DENSITY_X, OP_DENSITY_Y, OP_DENSITY_Z, OP_DISTANCE, OP_ANGLE, OP_DIHEDRAL, OP_DISTANCE_MIN, OP_DISTANCE_MAX, OP_RMSD, OP_DISTANCE_PAIR, OP_COM, OP_PLANE, OP_WITHIN_COUNT, OP_SHAPE_WEIGHTS, OP_COORD_X, OP_COORD_Y, OP_COORD_Z, OP_BACKBONE_ANGLES, OP_CONTACT_COUNT, OP_POROSITY, OP_EXPRESSION, OP_SECONDARY_STRUCTURE, EXPR_KINDS,
    CELL_ORTHO, CELL_TRICLINIC, CELL_PBC_X, CELL_PBC_Y, CELL_PBC_Z, CELL_PBC_ALL, DIST_BINS, VOL_DIM,
)
from .script import compile_script, ScriptError  # noqa: F401
