/* mdgpu.h — C ABI of libmdgpu: H100-native per-frame trajectory analysis behind VIAMD/mdlib's md_script
 * property API (rdf / sdf / density_x,y,z / distance / angle / dihedral evaluated over every frame).
 *
 * Plain C: pointers and sizes only, no CUDA / torch types. This is what the reference's per-frame evaluation
 * (mdlib/src/md_script.c:5730-5973 eval_properties and the procedures it calls) is replaced by; INTEGRATION.md
 * shows the lowering shim a maintainer adds inside md_script.c to drive it from a compiled md_script_ir_t.
 *
 * All paths cited are relative to the reference checkout (scanberg/viamd @ 9f7186f, ext/mdlib @ 77d1f08).
 *
 * Error convention (mirrors the reference's bool + MD_LOG_ERROR, core/md_log.h:7-9): functions return 0 on
 * success and a negative mdgpu_status otherwise; mdgpu_last_error() returns the message of the calling thread's
 * last failure. There is NO CPU fallback: without a usable CUDA device every compute entry point fails with
 * MDGPU_ERR_CUDA.
 */
#ifndef MDGPU_H
#define MDGPU_H

#include <stdint.h>
#include <stddef.h>
#include <stdbool.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDGPU_DIST_BINS 1024 /* MD_DIST_BINS, md_script_functions.inl:5  (ABI constant of the property layout) */
#define MDGPU_VOL_DIM   128  /* MD_VOL_DIM,   md_script_functions.inl:9 */

typedef enum mdgpu_status {
    MDGPU_OK = 0,
    MDGPU_ERR_INVALID_ARG = -1,
    MDGPU_ERR_CUDA = -2,          /* CUDA runtime failure or no device: the product never falls back to the CPU */
    MDGPU_ERR_UNSUPPORTED = -3,   /* operation outside the implemented hot-path scope */
    MDGPU_ERR_CAPACITY = -4,      /* a frame needs more cells than the plan's cell capacity */
    MDGPU_ERR_FRAME_SOURCE = -5,  /* load_frame failed (reference: "Failed to load frame during evaluation", md_script.c:5818) */
    MDGPU_ERR_INTERRUPTED = -6,
} mdgpu_status;

/* Unit cell. Field order and flag values are those of md_unitcell_t / md_unitcell_flags_t (md_types.h:36-43,254-259),
 * so a md_unitcell_t* can be passed as is. */
enum { MDGPU_CELL_ORTHO = 1, MDGPU_CELL_TRICLINIC = 2, MDGPU_CELL_PBC_X = 4, MDGPU_CELL_PBC_Y = 8, MDGPU_CELL_PBC_Z = 16, MDGPU_CELL_PBC_ALL = 28 };
typedef struct mdgpu_unitcell_t {
    double x, xy, xz;
    double y, yz;
    double z;
    uint32_t flags;
} mdgpu_unitcell_t;

/* Frame source: layout-compatible with md_trajectory_frame_header_t / md_trajectory_reader_i / md_trajectory_i
 * (md_trajectory.h:27-32,49-67); a VIAMD md_trajectory_i* can be passed after a pointer cast. */
typedef struct mdgpu_frame_header_t {
    size_t  num_atoms;
    int64_t index;
    double  timestamp;
    mdgpu_unitcell_t unitcell;
} mdgpu_frame_header_t;

struct mdgpu_trajectory_o;
struct mdgpu_trajectory_reader_o;
typedef struct mdgpu_trajectory_reader_i {
    struct mdgpu_trajectory_reader_o* inst;
    void (*free)(struct mdgpu_trajectory_reader_i* self);
    bool (*load_frame)(struct mdgpu_trajectory_reader_o* inst, int64_t idx, mdgpu_frame_header_t* header, float* x, float* y, float* z);
} mdgpu_trajectory_reader_i;

typedef struct mdgpu_trajectory_header_t {   /* md_trajectory_header_t, md_trajectory.h:20-25; md_unit_t = {u64 base; double mult} core/md_unit.h:48-51 */
    size_t num_frames;
    size_t num_atoms;
    struct { uint64_t base_bits; double mult; } time_unit;
    const double* frame_times;
} mdgpu_trajectory_header_t;

typedef struct mdgpu_trajectory_i {
    struct mdgpu_trajectory_o* inst;
    void (*free)(struct mdgpu_trajectory_i* self);
    bool (*get_header)(struct mdgpu_trajectory_o* inst, mdgpu_trajectory_header_t* header);
    bool (*init_reader)(mdgpu_trajectory_reader_i* reader, struct mdgpu_trajectory_o* inst);
} mdgpu_trajectory_i;

/* Static description of the system: what the procedures read from md_system_t besides coordinates
 * (atom masses via md_atom_extract_masses md_script.c:5764; covalent-bond connectivity md_bond_conn_data_t
 * md_system.h:103-111, needed by sdf()'s unwrap md_util.c:8738). */
typedef struct mdgpu_system_desc_t {
    size_t num_atoms;
    const float* atom_mass;            /* [num_atoms] */
    const uint32_t* bond_conn_offset;  /* [bond_conn_offset_count] (= num_atoms + 1), may be NULL if no sdf / rmsd property */
    const int32_t* bond_conn_atom_idx;
    size_t bond_conn_offset_count;
    const float* atom_radius;          /* [num_atoms] van der Waals radii as md_atom_extract_radii(r, 0, num_atoms, &sys->atom) gives them; may be NULL
                                        * unless a property is MDGPU_OP_POROSITY (mdgpu_plan_create then fails with MDGPU_ERR_INVALID_ARG) */
} mdgpu_system_desc_t;

/* Property operations (the procedures[] entries on the hot path, md_script_functions.inl:574-730). */
typedef enum mdgpu_op {
    MDGPU_OP_RDF = 1,        /* rdf(ref, trg, cutoff | min:max)     -> distribution  [1,2,1024]          :5263-5437 */
    MDGPU_OP_SDF = 2,        /* sdf(structures[], trg, cutoff)       -> volume        [1,128,128,128]     :5699-5856 */
    MDGPU_OP_DENSITY_X = 3,  /* density_x/_y/_z(atoms)               -> distribution                      :4825-5015 */
    MDGPU_OP_DENSITY_Y = 4,
    MDGPU_OP_DENSITY_Z = 5,
    MDGPU_OP_DISTANCE = 6,   /* distance(a, b)   atoms or selections -> temporal [F,1]                    :3851-3890 */
    MDGPU_OP_ANGLE = 7,      /* angle(a, b, c)                       -> temporal                          :4099-4114 */
    MDGPU_OP_DIHEDRAL = 8,   /* dihedral(a, b, c, d)                 -> temporal                          :4171-4196 */
    MDGPU_OP_DISTANCE_MIN = 9,  /* distance_min(a, b) over the atoms of two selections -> temporal        :3892-3928 */
    MDGPU_OP_DISTANCE_MAX = 10, /* distance_max(a, b): the reference evaluates md_util_min_distance here too (:3944) */
    MDGPU_OP_DISTANCE_PAIR = 12, /* distance_pair(a, b): |a| x |b| pair distances per frame -> temporal [F, |a|*|b|]  :3972-4064 */
    MDGPU_OP_COM = 13,       /* com(x): position of an atom / centre of mass of a selection -> temporal [F, 3]        :4726-4753 */
    MDGPU_OP_PLANE = 14,     /* plane(selection): (unit normal, normal . centre) of the best-fit plane -> temporal [F, 4] :4755-4822 */
    MDGPU_OP_WITHIN_COUNT = 15, /* count(within(radius, selection)): atoms of the system within radius of the selection -> temporal :2485-2533, :2868 */
    MDGPU_OP_SHAPE_WEIGHTS = 16, /* (linear, planar, isotropic) weights of n structures per frame -> temporal [F, n*3]: VIAMD's shape-space loop
                                  * (src/components/shapespace/shapespace.cpp:404-431) and _shape_weights (md_script_functions.inl:6005-6050) */
    MDGPU_OP_COORD_X = 17, MDGPU_OP_COORD_Y = 18, MDGPU_OP_COORD_Z = 19,   /* coord_x/_y/_z(selection): the atoms' coordinates -> temporal [F, n]  :5077-5169 */
    MDGPU_OP_RMSD = 11,      /* rmsd(selection) against the initial frame -> temporal                     :4287-4345 */
    MDGPU_OP_CONTACT_COUNT = 21, /* contact_count(A[], B, cutoff) -> temporal [F, |A|]; exclusion lists from the caller :2756-2866 */
    MDGPU_OP_BACKBONE_ANGLES = 20, /* (phi, psi) of every backbone segment per frame -> temporal [F, 2 * n_segments]: VIAMD's "Backbone Operations" pass
                                    * (src/viamd.cpp:488-520 -> md_util_backbone_angles_compute md_util.c:2572-2620) */
    MDGPU_OP_POROSITY = 22,  /* porosity(selection): unoccupied fraction of a voxel grid over the selection's van der Waals spheres -> temporal [F, 1] :5858-6003 */
    MDGPU_OP_EXPRESSION = 23, /* arithmetic and math functions over other temporal properties of the plan -> temporal [F, dim]: see mdgpu_expr_t :505-603 */
    MDGPU_OP_SECONDARY_STRUCTURE = 24, /* md_secondary_structure_t of every backbone segment per frame -> temporal [F, n_segments]: the other half of VIAMD's
                                        * "Backbone Operations" pass (src/viamd.cpp:488-525 -> md_util_backbone_secondary_structure_infer md_util.c:2552) */
} mdgpu_op;

/* One property = one `ident = proc(args);` statement whose selections were evaluated statically at compile time
 * (md_script.c:5492-5524) into ascending atom index lists (md_bitfield_iter_extract_indices order).
 *   RDF      : idx[0] = reference atoms, idx[1] = target atoms, cutoff_min/max.
 *              If num_structures > 0 the reference argument was an ARRAY of bitfields (e.g. residue(1:100)): the references are
 *              the centres of mass of `num_structures` atom groups stored back to back in idx[0] (extract_com :857, no periodic
 *              treatment) and a group's own atoms are excluded from its pairs (rdf_cb_excl_mask :5243). Groups are delimited
 *              by structure_offsets[num_structures+1], or are `structure_size` atoms each when that pointer is NULL.
 *              If ref_within_radius > 0 the reference argument was the dynamic selection within(radius, selection): idx[0] holds that
 *              selection and the references of a frame are the atoms of the system within `radius` of it, itself excluded (:2485-2533).
 *   SDF      : idx[0] = num_structures * structure_size atoms (equivalent structures), idx[1] = target atoms, cutoff_max.
 *              Each structure's row of structure_size atoms must be strictly ascending (an atom set, as the reference's bitfields give it):
 *              mdgpu_plan_create fails with MDGPU_ERR_INVALID_ARG for a row that is not, repeated atoms included.
 *   DENSITY_*: idx[0] = atoms.
 *   DISTANCE_MIN/_MAX: idx[0], idx[1] = the atoms of the two selections (brute force over all pairs, md_util_min_distance md_util.c:8242).
 *   DISTANCE_PAIR: an argument that was an ARRAY of selections contributes one position per selection, its centre of mass as for rdf's group references (extract_com :857): groups of
 *              argument 0 in structure_offsets[num_structures + 1], of argument 1 in structure_offsets_b[num_structures_b + 1]. Otherwise
 *              idx[0], idx[1] as for DISTANCE_MIN; row f of the property holds out[i * |b| + j] (md_util_distance_array md_util.c:8210);
 *              at most 1 000 000 values per frame (:4056). Properties with more than one value per frame also carry per-frame aggregates
 *              (mdgpu_plan_property_aggregate).
 *              With num_structures = n > 0 the statement was `expr in <n contexts>` (evaluate_context md_script.c:3418) with integer arguments:
 *              idx[k] holds n atoms, argument k remapped into each context (first atom of the context + k - 1); the property is [F, n].
 *   COM      : idx[0] as argument 0 of DISTANCE (bit 0 of com_args = it was a selection).   PLANE: idx[0] = the atoms (at least 3).
 *              For both within() consumers (WITHIN_COUNT and RDF with ref_within_radius): bit 0 of com_args set = the expression was
 *              `selection and within(...)` (_and :1975) and idx[2] holds that static selection's atoms (possibly none).
 *   WITHIN_COUNT: idx[0] = the selection's atoms, cutoff_max = radius (> 0), cutoff_min = lower bound of the min:max form (else 0). The dynamic selection within() is evaluated per frame over the
 *              system-wide cell list (get_spatial_acc :734); so far its only consumer on the device is count().
 *              count(<coordinate range> [and static]): a mdgpu_range_arg_t for argument 0, its static side in dyn[0], idx[0] empty and
 *              cutoff_min = cutoff_max = 0; the count of the frame's selected atoms (_count :2868).
 *              count(x, 'residue' | 'chain' | 'structure') (_count_with_arg -> internal_count :5465-5531): bit 1 of com_args set = the value of a
 *              frame is the number of groups that hold at least one atom of the frame's selection (the selection count(x) counts: within() minus
 *              its own selection, or the range, `and` its static side). The groups are num_structures lists of atoms in idx[1], delimited by
 *              structure_offsets[num_structures + 1], or structure_size atoms each when that pointer is NULL; num_structures = 0 is valid and
 *              gives 0 in every frame. The reference's groups are the components (md_system_component_atom_range) for 'residue', the instances
 *              (md_system_instance_atom_range) for 'chain', and the bond-connected structures (md_util_system_infer_structures) for 'structure'.
 *              idx[0], idx[2], cutoff_*, dyn[0] and the range argument keep their meaning; 'atom' is count(x) itself, bit 1 clear. mdgpu_plan_create
 *              fails with MDGPU_ERR_INVALID_ARG for an atom out of range, an atom in two groups, and offsets that do not rise from 0 to idx_count[1].
 *              The value is a float holding the exact integer count.
 *   SHAPE_WEIGHTS: idx[0] = the atoms of num_structures structures back to back (structure_offsets, or structure_size each), bit 0 of com_args
 *              = weights are the atom masses (shapespace's use_mass; _shape_weights always uses them), else 1.
 *   COORD_X/_Y/_Z: idx[0] = the atoms.
 *   CONTACT_COUNT: idx[0] = the atoms of the sets A_i back to back (structure_offsets, or structure_size each; num_structures sets), idx[1] = the atoms
 *              of B (flattened), cutoff_max = cutoff. Per frame and set: the number of (a in A_i, b in B) pairs within the cutoff whose b is not
 *              excluded, where the exclusion of set i is A_i & B grown along the bonds by `structure_size_b`... see structure_offsets_b below: the host
 *              passes the exclusion lists it derived (CSR in idx[2] / structure_offsets_b, num_structures_b = num_structures). Value i of a frame is the
 *              RUNNING total over sets 0..i: the reference never resets its counter between the sets of a frame (:2838-2847), reproduced.
 *   BACKBONE_ANGLES: idx[0] = for each of the num_structures backbone segments the five atoms C(i-1), N(i), CA(i), C(i), N(i+1)
 *              (md_protein_backbone_data_t::segment.atoms of the segment and its neighbours), back to back; -1 in any of the five marks a segment without angles (the first / last residue of a chain, chains shorter than 4:
 *              md_util.c:2588-2592) whose two values stay 0. Row f holds md_backbone_angles_t[num_structures] = (phi, psi) pairs in radians:
 *              phi = dihedral(C', N, CA, C), psi = dihedral(N, CA, C, N') with md_util_min_image_vec3 on the bond vectors, as `dihedral` evaluates.
 *   SECONDARY_STRUCTURE: idx[0] = for each of the num_structures backbone segments its atoms N, CA, C, O, HN back to back
 *              (md_protein_backbone_data_t::segment.atoms); HN is -1 when the residue has none, and H is then estimated as the reference does
 *              (estimate_HN from the previous segment's C, estimate_HN_term for the first segment of a range, md_util.c:1974-1989). The backbone
 *              ranges (chains) travel in structure_offsets_b with num_structures_b = the range count: backbone->range.offset, range.count + 1
 *              ascending entries from 0 to num_structures. Row f holds the md_secondary_structure_t code (1 coil .. 8 beta bridge) of every segment
 *              as a float; mdgpu_plan_secondary_structure returns the rows as md_secondary_structure_t. Numerical contract: every float
 *              operation is the reference's, in its order and rounding, with two exceptions: vec4_rsqrt of the H-bond energy is 1.0f / sqrtf(d2)
 *              (the reference's rsqrtps + one Newton step depends on the host CPU), and the bend angle's atan2f is CUDA's, which can differ from
 *              glibc's in the last ulp (the C restatement oracle/md_dssp.c uses glibc's, so the two agree in the bend decisions, not bit for bit in
 *              the angle); turn masks and flags start at zero (the reference takes them
 *              from uncleared temporary memory, md_util.c:2071, 2085). The rows equal the reference's wherever no candidate energy lies within
 *              1e-3 of -0.5, no donor's 2nd and 3rd lowest energies lie within 1e-3 of each other and no bend angle lies within 1e-4 rad of 70
 *              degrees. Candidate pairs are those of the reference's cell-grid walk over the CA positions at 9 A with the frame's cell
 *              (md_spatial_acc_for_each_internal_pair_within_cutoff); energies use the raw coordinates. A frame whose grid has fewer than 2n + 1
 *              cells on a periodic axis (n the neighbour reach; an orthorhombic axis under 27 A), or whose cell is triclinic without periodicity on
 *              all axes, fails with MDGPU_ERR_UNSUPPORTED: that walk can report a pair twice. mdgpu_plan_create fails with MDGPU_ERR_INVALID_ARG for
 *              no segments, an atom out of range (only HN may be -1), and range offsets that are missing, not ascending or not from 0 to num_structures.
 *   RMSD     : idx[0] = the atoms of the (flattened) selection; needs the initial frame and, to make molecules whole, the bond connectivity.
 *              With num_structures = n > 0 the statement was `rmsd(x) in <n contexts>` (evaluate_context md_script.c:3418): idx[0] holds n groups
 *              back to back, group c = the atoms of (flattened x AND context c), delimited by structure_offsets[n+1], or `structure_size` atoms each
 *              when that pointer is NULL (as for rdf). Groups may be empty (their value is 0) and an atom may be in several groups. The property
 *              is [F, n] with the per-frame aggregates; each group is fitted on its own, exactly as the single-selection form fits its selection.
 *   POROSITY : idx[0] = the atoms of the (flattened) selection, ascending; needs mdgpu_system_desc_t.atom_radius. Per frame, value_range [0, 1]:
 *              0 when the frame's cell is triclinic or the selection is empty (as the reference, which logs an error there). Otherwise
 *              xyzr = (x, y, z, radius) of the selected atoms in index order; com = md_util_com_compute_vec4(xyzr, 0, n, cell) (the trigonometric
 *              centre of mass weighted by the radii: serial float sums in index order); md_util_deperiodize_vec4 about com; bmin / bmax = min(p - r) /
 *              max(p + r) per axis; ext = max(bmax - bmin, 1.0f), t = max(ext) / 512 (exact), dim = max(1, (int)(ext / t)) (the longest axis gets
 *              512), d = ext / (float)dim. A sphere covers the voxels of the index box (int)floorf(((p -+ r) - bmin) / d) clamped to [0, dim - 1] whose
 *              centre c = bmin + ((float)i + 0.5f) * d passes fmaf(dx, dx, fmaf(dy, dy, dz * dz)) <= r * r with d* = c - p; those two fmaf are the only
 *              fused operations, everything else rounds separately. With `set` occupied voxels out of N = dim0 * dim1 * dim2, the value is 0 if
 *              set == 0, else (float)(((double)N - set) / (double)N). mdgpu_plan_property_frame_rows gives set (which = 0) and N (which = 1) per
 *              frame as u64, zero for frames not evaluated. Values equal the reference's wherever it is defined: the reference weights the centre of
 *              mass and pads the box with rad[atom index] from an array that holds only the radii of atoms 0 .. n-1 (md_atom_extract_radii(rad, 0,
 *              count) :5906, read through extract_xyzw_vec4 :5912), which is correct only when the selection is a prefix of the atoms (all,
 *              atom(1:k), residue(1:k)) and reads past the array otherwise; the library uses each selected atom's own radius, as the reference's voxel
 *              loop does (:5946). N <= 2^23 makes the float value determine `set` uniquely; larger grids can share a value between counts.
 *   DISTANCE/ANGLE/DIHEDRAL: idx[k] = the atoms of argument k (0-based). A single integer index is that atom's position; an
 *              argument that was a selection (bit k of com_args set, or more than one index) is its centre of mass as
 *              coordinate_extract_com evaluates it (:1717 -> md_util_com_compute md_util.c:8163: periodic cells use the
 *              trigonometric centre of mass _com_pbc_iw :7850, 8-lane float accumulation as in the AVX2 build).
 *              dihedral (and BACKBONE_ANGLES) bring each bond vector to its minimum image with the reference's subtract / add loop
 *              (min_image_ortho md_util.c:8424, the zone reduction of min_image_triclinic :8360), uncapped: a bond vector of any number of box
 *              lengths gives the reference's value. Where the reference's loop never ends (a step leaves the component unchanged: an infinite
 *              component, or one so large that x - box == x) the loop stops and the frame's value is NaN. */
/* A dynamic selection as an argument: within([radius_min:]radius_max, selection) [and static_selection] (_within_expl_flt / _frng
 * md_script_functions.inl:2485-2720, `and` :1975), evaluated per frame on the device over the system-wide cell list (get_spatial_acc :734).
 * For argument k of a property, idx[k] holds the atoms of the within() selection and dyn[k] the rest.
 *
 * An argument can instead be a coordinate range: see mdgpu_range_arg_t below. */
typedef struct mdgpu_dynamic_arg_t {
    float radius_min, radius_max;   /* radius_max > 0 switches the argument to dynamic */
    const int32_t* and_idx;         /* the static side of `selection and within(...)`, or NULL */
    size_t and_count;
    uint32_t has_and;               /* 1: and_idx is meaningful even when empty (`nothing and within(...)` selects nothing) */
} mdgpu_dynamic_arg_t;

typedef struct mdgpu_property_desc_t {
    const char* name;
    uint32_t op;
    const int32_t* idx[4];
    size_t idx_count[4];
    size_t num_structures;
    size_t structure_size;
    float cutoff_min;
    float cutoff_max;
    const uint32_t* structure_offsets;   /* optional CSR offsets into idx[0] for groups of different sizes (rdf) */
    uint32_t com_args;                   /* distance/angle/dihedral: bit k = argument k is a selection (centre of mass even for one atom); WITHIN_COUNT:
                                          * bit 0 = idx[2] is a static `and` side, bit 1 = count over the groups of idx[1] (see above) */
    float ref_within_radius;             /* rdf: > 0 -> the reference argument was within(radius, idx[0]): the dynamic selection is evaluated per frame */
    float ref_within_min;                /* ... within(min:radius, idx[0]) (_within_expl_frng :2609); 0 for the plain form */
    const uint32_t* structure_offsets_b; /* distance_pair: CSR groups of argument 1 when it was an array of selections (argument 0 uses structure_offsets);
                                          * rdf: the TARGET was an array of num_structures_b selections (idx[1] back to back): their centres of mass are the
                                          * target points (compute_rdf md_script_functions.inl:5293-5302); contact_count: the exclusion CSR */
    size_t num_structures_b;
    mdgpu_dynamic_arg_t dyn[4];          /* per argument: a dynamic selection (see above). Consumers: rdf reference and / or target, sdf target, density_x/_y/_z,
                                          * distance / angle / dihedral / com (the centre of mass of the frame's selection), distance_min / _max, count().
                                          * ref_within_radius (+ com_args bit 0 / idx[2]) is the round-1 spelling of dyn[0] for rdf and still honoured. */
    const uint32_t* arg_offsets[4];      /* distance / angle / dihedral / com: argument k was an ARRAY of arg_parts[k] >= 2 selections. idx[k] holds them back to */
    uint32_t arg_parts[4];               /* back, arg_offsets[k] their arg_parts[k] + 1 CSR offsets. Its position is the centre of the selections' centres:
                                          * md_util_com_compute per selection, then md_util_com_compute_vec4 over those with weight 1
                                          * (coordinate_extract_com md_script_functions.inl:1826-1842). 0 or 1: idx[k] is one selection. */
} mdgpu_property_desc_t;

/* Result view: the fields of md_script_property_data_t (md_script.h:73-92) that the evaluation fills. */
typedef struct mdgpu_property_data_t {
    int32_t dim[4];
    size_t  num_values;
    float*  values;       /* owned by the plan, stable for its lifetime (as in the reference, md_script.c:6497-6504) */
    float*  weights;      /* distributions only: values + dim[2] */
    float   min_value, max_value;
    float   min_range[2], max_range[2];
    uint64_t frames_accumulated;
} mdgpu_property_data_t;

typedef struct mdgpu_plan mdgpu_plan;

typedef struct mdgpu_plan_options_t {
    int      device;              /* CUDA device ordinal */
    uint32_t batch_frames;        /* frames per launch batch; 0 = default (one per SM) */
    uint32_t num_streams;         /* CUDA streams (slots) the frame loop is dispatched onto; 0 = default (6), at most 8 */
    uint32_t keep_frame_results;  /* 1: retain raw per-frame integer bins of distributions (parity tests) */
    uint32_t cell_capacity;       /* cells per frame the cell lists are sized for; 0 = 2x the grid of the first evaluation's first frame, at least
                                   * 2^16. A non-periodic axis (no cell, or a cell without PBC on it) gets its grid from the atoms' bounding box:
                                   * mdgpu_eval_host_frames fits it to all frames of that call; device-resident, XTC and trajectory frames are not
                                   * seen then and get 2^16. A frame that needs more cells fails its batch with MDGPU_ERR_CAPACITY; raise this */
    uint32_t rdf_variant;         /* rdf pair-kernel variant, all bit-identical in their results: 0 = default (register-pair targets, 4 CTAs/SM), 1 = scalar kernel
                                   * without candidate lists, 2 = 3 CTAs/SM with a longer hit queue, 4 = reference chunks staged by the TMA unit
                                   * (cp.async.bulk + mbarrier; kept as an alternative) */
    uint32_t ingest_mode;         /* host ingest (mdgpu_eval_host_frames / _trajectory): 0 = copy only the atoms the properties read when they are
                                   * less than 3/4 of the system (gathered into pinned staging by the ingest threads), 1 = always whole frames */
    uint32_t ingest_threads;      /* host threads that gather frames into pinned staging; 0 = default (min(16, cores / 2)) */
    uint32_t num_devices;         /* > 1: ONE process drives several GPUs (VIAMD is one process): contiguous frame blocks per device, accumulators
                                   * merged onto devices[0] by one NCCL reduce at mdgpu_plan_sync (SURVEY.md 8(e)); `device` is then ignored */
    int32_t  devices[16];         /* CUDA ordinals when num_devices > 1 */
} mdgpu_plan_options_t;

const char* mdgpu_last_error(void);
int mdgpu_device_count(void);

/* Plan lifetime. num_frames is the trajectory length (rows of temporal properties; md_script_eval_create :6506). */
mdgpu_plan* mdgpu_plan_create(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props,
                              size_t num_frames, const mdgpu_plan_options_t* opts);

/* A coordinate range as argument `arg` of property `prop`: within_x(a:b) / within_y(a:b) / within_z(a:b) / within_xyz(a:b, c:d, e:f)
 * [and static_selection] (procedures md_script_functions.inl:668-671, coordinate_range :2394-2476), evaluated per frame on the device.
 * Atom i of the frame is selected iff lo[0] <= x[i] <= hi[0] and the same for y and z: the frame's coordinates as loaded (no wrapping, no cell,
 * orthorhombic or triclinic: atoms of unwrapped trajectories outside the cell count by their raw coordinates), both ends inclusive. An axis the
 * call does not constrain is [-FLT_MAX, FLT_MAX]; it is still compared, so an atom with a NaN or +-inf coordinate on any axis is never selected.
 * Integer bounds arrive as the frange the front end casts them to. Unlike within(), no atom is removed afterwards; `selection and within_*(...)`
 * is the intersection: the static side is dyn[arg].and_idx / and_count / has_and of the property, whose radius_* stay 0; idx[arg] stays empty.
 * A range is evaluated over all atoms of the system (:2414-2424); the form inside an `in` context (:2401-2412, only the context's atoms) is not
 * lowered. Consumers: those of within() (see mdgpu_property_desc_t.dyn); count(<range expression>) is MDGPU_OP_WITHIN_COUNT with the range as
 * argument 0 (cutoff_min = cutoff_max = 0).
 * The ranges travel beside the property descriptors, not in them, so that the layout of mdgpu_property_desc_t stays that of hosts compiled
 * before ranges existed. */
typedef struct mdgpu_range_arg_t {
    uint32_t prop;                  /* index into props */
    uint32_t arg;                   /* argument 0..3 of that property */
    float lo[3], hi[3];             /* x, y, z bounds, inclusive */
} mdgpu_range_arg_t;
/* mdgpu_plan_create with coordinate-range arguments. Fails with MDGPU_ERR_INVALID_ARG for a range whose prop / arg is out of range or listed twice,
 * an argument with both a radius and a range, and a range with lo > hi or a NaN bound; with MDGPU_ERR_UNSUPPORTED where the procedure takes no
 * dynamic selection. mdgpu_plan_create(...) is this function with no ranges. */
mdgpu_plan* mdgpu_plan_create_with_ranges(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props,
                                          size_t num_frames, const mdgpu_plan_options_t* opts, const mdgpu_range_arg_t* ranges, size_t num_ranges);

/* A temporal expression: the value of an MDGPU_OP_EXPRESSION property, evaluated per frame on the device after the procedure properties of the
 * frame (operators md_script_functions.inl:505-571, functions :576-603). The program is postfix: CONST pushes `value`, PROP pushes the row of
 * property `prop` (a temporal of the plan, not the expression itself), every other node pops its operands and pushes its result. A value is a
 * float or an array of n floats; `+ - * /` take two floats, an array and a float (either order) or two arrays of equal length, element-wise;
 * NEG, ABS, FLOOR and CEIL take a float or an array; every other function takes floats only (the reference registers no array form of it).
 * The property is [F, n] (n = 1 for a float result) with the per-frame aggregates of a multi-valued temporal.
 * Numerical contract: + - * / NEG ABS FLOOR CEIL MIN MAX SQRT are IEEE float32 operations (MIN / MAX as fminf / fmaxf), bit-equal to the
 * reference's; the other functions are evaluated in double and rounded to float once (the reference calls glibc's float functions; the two
 * differ by at most 1 ulp on the reference data, DESIGN.md section 3).
 * The reference applies `scalar op array` as `array op scalar` (its FLAG_SYMMETRIC_ARGS swaps the operands: `2 - a` is a - 2); a host lowering
 * from the reference's syntax tree sees the operands already swapped. */
enum {
    MDGPU_EXPR_CONST = 0, MDGPU_EXPR_PROP = 1,
    MDGPU_EXPR_NEG = 2, MDGPU_EXPR_ADD = 3, MDGPU_EXPR_SUB = 4, MDGPU_EXPR_MUL = 5, MDGPU_EXPR_DIV = 6,
    MDGPU_EXPR_SQRT = 7, MDGPU_EXPR_CBRT = 8, MDGPU_EXPR_ABS = 9, MDGPU_EXPR_FLOOR = 10, MDGPU_EXPR_CEIL = 11, MDGPU_EXPR_COS = 12,
    MDGPU_EXPR_SIN = 13, MDGPU_EXPR_ASIN = 14, MDGPU_EXPR_ACOS = 15, MDGPU_EXPR_ATAN = 16, MDGPU_EXPR_LOG = 17, MDGPU_EXPR_EXP = 18,
    MDGPU_EXPR_LOG2 = 19, MDGPU_EXPR_EXP2 = 20, MDGPU_EXPR_LOG10 = 21,
    MDGPU_EXPR_ATAN2 = 22, MDGPU_EXPR_POW = 23, MDGPU_EXPR_MIN = 24, MDGPU_EXPR_MAX = 25,   /* two operands: atan(y, x) = atan2(y, x) */
};
#define MDGPU_EXPR_MAX_DEPTH 16   /* operand stack depth of a program */
typedef struct mdgpu_expr_node_t {
    uint32_t kind;                  /* MDGPU_EXPR_* */
    float value;                    /* CONST */
    uint32_t prop;                  /* PROP: index into props */
} mdgpu_expr_node_t;
typedef struct mdgpu_expr_t {
    uint32_t prop;                  /* the MDGPU_OP_EXPRESSION property this program computes */
    const mdgpu_expr_node_t* nodes; /* postfix order */
    size_t num_nodes;
} mdgpu_expr_t;
/* mdgpu_plan_create_with_ranges with temporal expressions beside the descriptors (their layout stays that of earlier hosts). Fails with
 * MDGPU_ERR_INVALID_ARG for: an EXPRESSION property without exactly one program or a program naming a property that is not an EXPRESSION;
 * a PROP that names no property, a non-temporal one or the expression itself; expressions that depend on each other in a cycle; a program
 * that pops an empty stack, holds more than MDGPU_EXPR_MAX_DEPTH operands or does not end with exactly one; two arrays of different lengths;
 * an array given to a function that takes floats only; an unknown kind. Expressions of expressions are evaluated in dependency order.
 * mdgpu_plan_create_with_ranges(...) is this function with no expressions. */
mdgpu_plan* mdgpu_plan_create_ex(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props, size_t num_frames,
                                 const mdgpu_plan_options_t* opts, const mdgpu_range_arg_t* ranges, size_t num_ranges,
                                 const mdgpu_expr_t* exprs, size_t num_exprs);
void mdgpu_plan_destroy(mdgpu_plan* plan);

/* Frame 0 of the trajectory ("initial configuration", md_script.c:5808): reference structure of sdf() and rmsd(), reference cell of density_*(). */
int mdgpu_plan_set_initial_frame(mdgpu_plan* plan, const float* x, const float* y, const float* z, const mdgpu_unitcell_t* cell);

/* md_script_eval_clear_data (md_script.c:6563): zero accumulators, frame mask, interrupt flag. */
int mdgpu_plan_clear(mdgpu_plan* plan);

/* XTC input (SURVEY.md section 8(f)1; reference: md_xtc.c:747-931 decode, :947-993 reader, :436-570 frame offsets): `h_blob` holds
 * whole XTC frames as they are in the file, frame i spanning bytes [frame_offsets[i], frame_offsets[i+1]) (offsets are multiples of 4, as
 * XDR guarantees). The compressed bytes cross PCIe and are expanded on the device with the reader's arithmetic (coordinates in
 * Angstrom = int * (10 / precision), unit cell from the box matrix * 10); results are those of evaluating the decoded frames. */
int mdgpu_eval_xtc_frames(mdgpu_plan* plan, const uint8_t* h_blob, const uint64_t* frame_offsets, uint32_t frame_beg, uint32_t count);
/* The same from a file: reads `path` into pinned memory, finds the frame starts, takes frame 0 as the initial configuration if none was set
 * (md_script.c:5808), evaluates frames [frame_beg, frame_end) and waits for them. */
int mdgpu_eval_xtc_file(mdgpu_plan* plan, const char* path, uint32_t frame_beg, uint32_t frame_end);
/* Frame starts of an XTC file image: offsets[0..n] (offsets[n] = end of the last complete frame), n and the atom count returned. */
int mdgpu_xtc_frame_offsets(const uint8_t* file, size_t nbytes, uint64_t* offsets, size_t capacity, size_t* num_frames, size_t* num_atoms);
/* The same decode without a plan: h_xyz[count][3][num_atoms], optional cells / steps / times per frame. */
int mdgpu_xtc_decode_frames(int device, const uint8_t* h_blob, const uint64_t* frame_offsets, uint32_t count, size_t num_atoms,
                            float* h_xyz, mdgpu_unitcell_t* h_cells, int32_t* h_steps, float* h_times);

/* The frame loop. Frames [frame_beg, frame_beg+count) are evaluated and accumulated.
 *  _device: coordinates already in HBM; frame i has x at d_xyz + i*frame_stride, y at + axis_stride, z at + 2*axis_stride (floats).
 *  _host  : same layout in host memory (pinned or pageable); copied host->device batch by batch inside the call — when it returns the
 *            buffer has been read and may be refilled (the kernels may still be running: mdgpu_plan_sync waits for them). When the
 *            properties read less than 3/4 of the atoms, only those atoms cross PCIe (options.ingest_mode).
 *  _trajectory: pulls frames through the md_trajectory_i-compatible interface with `loader_threads` readers
 *               (md_script_eval_frame_range semantics, md_script.c:6573-6612). */
int mdgpu_eval_device_frames(mdgpu_plan* plan, const float* d_xyz, size_t frame_stride, size_t axis_stride,
                             const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count);
int mdgpu_eval_host_frames(mdgpu_plan* plan, const float* h_xyz, size_t frame_stride, size_t axis_stride,
                           const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count);
int mdgpu_eval_trajectory(mdgpu_plan* plan, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads);

/* Wait for all enqueued batches and fold device accumulators into the host-visible property data. */
int mdgpu_plan_sync(mdgpu_plan* plan);

/* Threading (md_script_eval_frame_range is re-entrant on one eval from many threads with disjoint ranges, src/task_system.cpp:73-87,
 * mdlib/unittest/test_script.c:1352-1417): mdgpu_eval_trajectory / _host_frames / _device_frames and mdgpu_plan_sync may be called
 * concurrently on one plan with disjoint frame ranges. Each call takes stream slots as they become free; results do not depend on the
 * interleaving (integer accumulators, disjoint temporal rows).
 *
 * Result storage: by default the plan owns `values`. mdgpu_plan_bind_property_storage makes it write a property's values (and the per-frame
 * aggregate arrays of a multi-valued temporal: mean[F], variance[F], extent[F][2]; may be NULL) into the caller's arrays instead — the
 * md_script shim binds md_script_property_data_t::values (md_script.h:73-92), which VIAMD reads directly (src/main.cpp:1286-1303, 1524).
 *
 * Progress: with a callback installed, every completed batch publishes at once — its temporal rows are copied to the host values, running
 * means of distributions / volumes are refreshed at most every 100 ms — and the callback is invoked (from the thread that retired the batch)
 * with the batch's frame range; the shim sets md_script_eval_t::frame_mask bits there (md_script.c:5962-5964), so the UI sees partial
 * results while the evaluation runs (src/main.cpp:1513-1524). */
typedef void (*mdgpu_progress_fn)(void* user, uint32_t frame_beg, uint32_t frame_count);
int mdgpu_plan_bind_property_storage(mdgpu_plan* plan, size_t prop, float* values, size_t num_values, float* agg_mean, float* agg_var, float* agg_ext);
int mdgpu_plan_set_progress_callback(mdgpu_plan* plan, mdgpu_progress_fn fn, void* user);

/* Pin the calling thread (and the threads it creates afterwards) to the CPUs next to `device` (sysfs local_cpulist of its PCI function), so
 * that pinned staging it allocates and the ingest threads sit on the GPU's NUMA node. Returns the number of CPUs, or a negative status. */
int mdgpu_bind_host_to_device(int device);

/* Multi-device plans: milliseconds the last exchange step (NCCL reduce onto devices[0]) took on the root device, and how many ran. */
int mdgpu_plan_exchange_stats(mdgpu_plan* plan, double* last_ms, uint64_t* count);
/* Host-ingest facts of a plan: atoms copied per frame (= num_atoms unless the compact ingest is active) and the ingest thread count. */
int mdgpu_plan_ingest_info(mdgpu_plan* plan, size_t* atoms_per_frame, uint32_t* threads);
void mdgpu_plan_interrupt(mdgpu_plan* plan);   /* md_script_eval_interrupt :6663 */

size_t mdgpu_plan_property_count(const mdgpu_plan* plan);
int mdgpu_plan_property_index(const mdgpu_plan* plan, const char* name);
int mdgpu_plan_property_data(mdgpu_plan* plan, size_t prop, mdgpu_property_data_t* out);   /* implies mdgpu_plan_sync */
int mdgpu_plan_property_peek(mdgpu_plan* plan, size_t prop, mdgpu_property_data_t* out);   /* as last folded, waits for nothing (for progress callbacks) */

/* Per-frame aggregates of a temporal with several values per frame (md_script_aggregate_t md_script.h:63-70, filled at md_script.c:5886-5890):
 * out_mean[num_frames], out_var[num_frames] (population variance), out_ext[num_frames][2] (min, max); any may be NULL. Implies mdgpu_plan_sync. */
int mdgpu_plan_property_aggregate(mdgpu_plan* plan, size_t prop, float* out_mean, float* out_var, float* out_ext, size_t num_frames);

/* Histogram of a temporal property over the evaluated frames, on the device: VIAMD's compute_histogram_masked (src/main.cpp:172-226, called from
 * :1513 for every temporal display property whenever its fingerprint changes). The [F, dim] values stay in HBM; out_bins[(aggregate ? 1 : dim)][num_bins]
 * receives counts scaled by 1 / (bin width x samples of the row), out_min_max (optional) the smallest / largest scaled bin. Implies mdgpu_plan_sync. */
int mdgpu_plan_property_histogram(mdgpu_plan* plan, size_t prop, uint32_t num_bins, float range_min, float range_max, int aggregate, float* out_bins, float* out_min_max);

/* VIAMD's Ramachandran density (src/components/ramachandran/ramachandran.cpp:1277-1370, rama_rep_compute_density) from the (phi, psi) rows of an
 * MDGPU_OP_BACKBONE_ANGLES property, on the device. Class c (0 general, 1 glycine, 2 proline, 3 pre-proline: segment.rama_type as
 * md_util_backbone_ramachandran_classify fills it) holds the segments segments[class_offsets[c] .. class_offsets[c+1]). Every frame of
 * [frame_beg, frame_end) that has been evaluated (frame-mask bit set) and every listed segment whose angles are not (0, 0) adds 1 to texel (x, y)
 * of channel c, then the map is blurred by three box passes per axis with the radii of boxes_for_gauss(., 3, sigma) (blur_density_gaussian :368-387).
 * out_tex[512][512][4] receives the map in VIAMD's density_tex layout (texel y * 512 + x, RGBA = the four classes), out_sum[c] the samples of class c.
 * sigma must lie in VIAMD's slider range [0.1, 10]. Implies mdgpu_plan_sync; runs on devices[0] of a multi-device plan.
 * Numerical contract (against the reference built with -fno-fast-math -ffp-contract=off): u = phi * s + 0.5f and v = psi * s + 0.5f with
 * s = (float)(1 / 2pi) and two roundings each, x = ((uint32_t)(u * 512.0f)) & 511 truncating toward zero (phi = -pi lands in texel 0, phi = pi wraps
 * to 0), the same for y; a texel's value is min(samples, 2^24), the exact result of adding 1.0f per sample in float; the box passes add and subtract
 * in the reference's order, so the map equals the reference's value for value (only the sign of a zero may differ); out_sum[c] = (float)(double)n. */
int mdgpu_plan_rama_density(mdgpu_plan* plan, size_t prop, const uint32_t* segments, const uint32_t class_offsets[5], uint32_t frame_beg, uint32_t frame_end,
                            float sigma, float* out_tex, float out_sum[4]);

/* The secondary structure of frames [frame_beg, frame_end) of an MDGPU_OP_SECONDARY_STRUCTURE property: out[(f - frame_beg) * S + i] = the
 * md_secondary_structure_t of segment i (4 bytes each), ready to be copied into VIAMD's trajectory_data.secondary_structure at stride S per frame.
 * Frames not evaluated yet hold 0 (MD_SECONDARY_STRUCTURE_UNKNOWN). Implies mdgpu_plan_sync; runs on devices[0] of a multi-device plan. */
int mdgpu_plan_secondary_structure(mdgpu_plan* plan, size_t prop, uint32_t frame_beg, uint32_t frame_end, int32_t* out);

/* Exact integer results (what parity is asserted on).
 *  _counts: accumulated counts over all evaluated frames: RDF 1024 x u64 bins; SDF 128^3 x u64 voxels (widened from u32);
 *           DENSITY 1024 x u64 fixed-point mass sums (unit 2^-24 Da).
 *  _frame_counts: raw bins of one frame (needs keep_frame_results), RDF: u32[1024] plus the frame's pair total; SDF: the frame's hit total
 *           (the voxel increments of all its structures) only, out_bins must be NULL. */
int mdgpu_plan_property_counts(mdgpu_plan* plan, size_t prop, uint64_t* out, size_t out_len);
int mdgpu_plan_property_frame_counts(mdgpu_plan* plan, size_t prop, uint32_t frame, uint32_t* out_bins, uint64_t* out_total);

/* Completed-frame bitmask (md_script_eval_frame_mask :6655): 1 bit per frame, little-endian u64 words. */
int mdgpu_plan_frame_mask(mdgpu_plan* plan, uint64_t* out_words, size_t num_words);

/* Multi-GPU: device pointer + byte size of a property's accumulator (u64 bins, u32 voxels, f32 temporal rows) so the caller's communicator
 * (NCCL via torch.distributed in bench.py) can all-reduce it in place; then mdgpu_plan_set_frames_accumulated. */
int mdgpu_plan_property_accum_ptr(mdgpu_plan* plan, size_t prop, void** d_ptr, size_t* bytes, uint32_t* elem_bytes);
/* Temporals shard by rows: accum_ptr returns their float32 [num_frames][len] buffer (rows of frames this plan did not evaluate are zero, so a
 * SUM all-reduce merges the shards exactly); afterwards the frames the other ranks evaluated are declared done, so that min/max, ranges and
 * the per-frame aggregates cover them. */
int mdgpu_plan_mark_frames_done(mdgpu_plan* plan, uint32_t frame_beg, uint32_t count);
/* Per-frame integer rows of a distribution / volume property — which = 0: pair / hit total per frame (rdf weights come from the last frame's),
 * 1 / 2: smallest / largest bin of the frame (min_value / max_value). [num_frames] entries of elem_bytes each, zero where this plan did not
 * evaluate, so the same SUM all-reduce merges them when every rank's plan spans the global frame range. d_ptr = NULL if the property has none. */
int mdgpu_plan_property_frame_rows(mdgpu_plan* plan, size_t prop, uint32_t which, void** d_ptr, size_t* bytes, uint32_t* elem_bytes);
int mdgpu_plan_set_frames_accumulated(mdgpu_plan* plan, size_t prop, uint64_t frames);

/* Kernel bookkeeping for bench.py: launches issued by this library since the counter was last reset, and
 * CUDA-event time (ms, summed over launches) measured on the launching stream when timing is enabled; `kernel` selects
 * "k_rdf_pairs" (the pair kernel alone), "k_rdf_cull" (its candidate-list pre-pass), "k_sdf" (fit + scatter kernels of an sdf) or "k_density"
 * (binning + finalize). The spans are exact only when one stream is in flight (a plan with num_streams = 1): with several slots the events
 * also see the kernels of the other streams. */
uint64_t mdgpu_launch_count(bool reset);
int mdgpu_plan_enable_kernel_timing(mdgpu_plan* plan, int enable);
/* Device-side stopwatch over everything the plan enqueues: _begin drains the device and records a CUDA event; _end records
 * one event per plan stream, waits, and returns the largest elapsed time (ms) — i.e. device time of the whole frame loop. */
int mdgpu_plan_timer_begin(mdgpu_plan* plan);
int mdgpu_plan_timer_end(mdgpu_plan* plan, double* elapsed_ms);
int mdgpu_plan_kernel_time_ms(mdgpu_plan* plan, const char* kernel, double* total_ms, uint64_t* launches);
/* Device-side counters of the pair kernel, accumulated while kernel timing is enabled: which = 0 pair tests executed (padding lanes of the
 * last chunk / reference group included: they occupy FP32 lanes), 1 = tests between a real reference point and a real listed target. */
int mdgpu_plan_kernel_counter(mdgpu_plan* plan, uint32_t which, uint64_t* value);

/* Host evaluation of the per-frame cell-grid geometry (the same code the device runs, one thread per frame); used by the
 * CPU-side tests and for sizing. out_i[13] = cdim[3], ncell[3], hlo[3], hdim[3], valid; out_f[7] = G00,G11,G22,H01,H02,H12,r2. */
int mdgpu_debug_frame_geom(const mdgpu_unitcell_t* cell, double cell_ext, double cutoff, const float* aabb_min_max /* 6 floats or NULL */,
                           int32_t* out_i, float* out_f);

/* Host fold of one frame of a multi-valued temporal, as mdgpu_plan_sync applies it (no device needed): out4 = min, max, mean, variance. */
int mdgpu_debug_aggregate(const float* values, size_t count, float* out4);

/* Self-check of the branch-free correctly-rounded sqrt used when binning RDF hits: compares it with the IEEE sqrt for every
 * float whose bit pattern lies in [lo_bits, hi_bits) and returns the number of mismatches (must be 0 in the normal range). */
int mdgpu_debug_sqrt_sweep(int device, uint32_t lo_bits, uint32_t hi_bits, uint64_t* mismatches);

/* The rdf candidate cull this process runs (no device needed): "full8" / "full6" / "full4" (full-warp cull at that register target, the
 * default is full8), "half" (half-warp cull) or "flat6" / "flat8" / "flat4" (flattened cull). MDGPU_CULL and MDGPU_CULL_OCC are read once, at
 * the first rdf launch or the first call of this function, whichever comes first; later changes of the environment have no effect.
 * Writes a NUL-terminated name into out[n]. */
int mdgpu_debug_rdf_config(char* out, size_t n);

/* Synthetic workloads (viamd_b200/csrc/synth.h), used by bench.py and the tests. */
int mdgpu_synth_water_desc(uint32_t n, uint32_t seed, uint32_t* num_atoms, float* L);
int mdgpu_synth_water_base(uint32_t n, uint32_t seed, float* base_xyz /* [3][num_atoms] wrapped */, float* whole_xyz /* optional */);
int mdgpu_synth_water_frames_host(uint32_t n, uint32_t seed, const float* base_xyz, uint32_t frame_beg, uint32_t count,
                                  float* out_xyz, size_t frame_stride, size_t axis_stride);
int mdgpu_synth_water_frames_device(int device, uint32_t n, uint32_t seed, const float* d_base_xyz, uint32_t frame_beg, uint32_t count,
                                    float* d_out_xyz, size_t frame_stride, size_t axis_stride);

/* membrane workload of BASELINE config 4 (coarse-grained bilayer + solvent beads, viamd_b200/csrc/synth.h) */
int mdgpu_synth_membrane_desc(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, uint32_t* num_atoms, uint32_t* num_lipids, float* L3);
int mdgpu_synth_membrane_base(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, float* base_xyz, float* whole_xyz, uint32_t* mol_id);
int mdgpu_synth_membrane_frames_host(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, const float* base_xyz, const uint32_t* mol_id,
                                     uint32_t frame_beg, uint32_t count, float* out_xyz, size_t frame_stride, size_t axis_stride);
int mdgpu_synth_membrane_frames_device(int device, uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, const float* d_base_xyz, const uint32_t* d_mol_id,
                                       uint32_t frame_beg, uint32_t count, float* d_out_xyz, size_t frame_stride, size_t axis_stride);

/* Thin device-memory helpers so C hosts need no CUDA headers. */
int mdgpu_device_alloc(int device, size_t bytes, void** out);
int mdgpu_device_free(int device, void* p);
int mdgpu_host_alloc_pinned(size_t bytes, void** out);
int mdgpu_host_free_pinned(void* p);
int mdgpu_memcpy_h2d(int device, void* dst, const void* src, size_t bytes);
int mdgpu_memcpy_d2h(int device, void* dst, const void* src, size_t bytes);
int mdgpu_device_synchronize(int device);

#ifdef __cplusplus
}
#endif
#endif /* MDGPU_H */
