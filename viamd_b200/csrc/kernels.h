// kernels.h — host-callable launchers of the per-batch kernels (defined in cells.cu, rdf.cu, sdf.cu, props.cu, porosity.cu, expr.cu, dssp.cu, synth.cu)
#pragma once
#include "common.cuh"

namespace mdg {

// cells.cu
void host_frame_geom(FrameGeom* g, const mdgpu_unitcell_t* uc, double cell_ext, double cutoff, const float* aabb, uint32_t cap);
void launch_geom(const mdgpu_unitcell_t* d_cells, const float* d_aabb, FrameGeom* d_geom, double cell_ext, double cutoff, uint32_t cap,
                 int B, int* d_err, cudaStream_t s);
void launch_aabb(const BatchFrames& fr, const int32_t* d_idx, uint32_t n, float* d_aabb, cudaStream_t s, DynSel dyn = DynSel{ nullptr, nullptr, 0 }, const float* d_aos = nullptr);
void launch_cell_list(int mode, const BatchFrames& fr, const int32_t* d_idx, const float* d_aos, uint32_t n, const FrameGeom* d_geom,
                      const CellList& cl, int store_linear_idx, cudaStream_t s, DynSel dyn = DynSel{ nullptr, nullptr, 0 });

// rdf.cu
struct RdfArgs {
    const FrameGeom* geom;
    CellList trg, ref;
    float min_cutoff, inv_cutoff_range, min_r2;
    uint32_t* frame_bins;        // [B][1024] + [B] work counters, zeroed by the launcher
    const uint32_t* excl_off;    // structure -> atoms CSR (rdf_cb_excl_mask), or null
    const int32_t* excl_idx;
    uint32_t frame0;             // global index of the batch's first frame
    int symmetric;               // reference selection == target selection
    // contact_count (scalar kernel only): reference points carry their position in the concatenated set list; ref_set maps it to the set, whose
    // exclusion list is excl_off / excl_idx[set] and whose pair count goes to "bin" set of the frame's row
    const uint32_t* ref_set; int count_mode;
    // candidate lists (k_rdf_cull -> k_rdf_pairs_v2): per frame `list_stride` entries (target position | image code << 26), per home cell a
    // header {first entry, entries of class 0, 1, 2}; one cursor per frame (zeroed by the launcher); err receives MDGPU_ERR_CAPACITY on overflow
    uint32_t* pair_list; uint4* list_hdr; uint32_t* list_cursor; size_t list_stride; size_t hdr_stride; int* err;
    // measurement only (null unless kernel timing is enabled): [0] pair tests the pair kernel executed, padding lanes included,
    // [1] of those, tests between a real reference point and a real listed target
    unsigned long long* counters;
    // finalize
    unsigned long long* acc;     // [1024] accumulated bins
    unsigned long long* frame_total;  // [num_frames]
    uint32_t* frame_min;         // [num_frames]
    uint32_t* frame_max;
    uint32_t* keep;              // [num_frames][1024] or null
};
void launch_group_com(const BatchFrames& fr, const int32_t* d_idx, const uint32_t* d_off, uint32_t n_groups, const float* d_mass, float* d_out, cudaStream_t s);
void launch_rdf(const RdfArgs& a, int B, bool tri, int variant, int sm_count, cudaStream_t s, cudaEvent_t* ev4 /* null, or events recorded {before cull, after cull, before pairs, after pairs} */);
// the candidate cull launch_rdf runs (MDGPU_CULL / MDGPU_CULL_OCC, read once per process)
enum RdfCullKind { RDF_CULL_FULL = 0, RDF_CULL_HALF = 1, RDF_CULL_FLAT = 2 };
struct RdfCullConfig { int kind; int occ; };   // occ: resident CTAs / SM the register allocation aims for (8, 6 or 4; 0 for the half-warp cull)
RdfCullConfig rdf_cull_config();

void launch_contact_rows(const uint32_t* d_frame_bins, uint32_t n_sets, float* d_out, uint32_t frame0, int B, cudaStream_t s);   // running totals over the sets -> temporal row
unsigned long long run_sqrt_sweep(uint32_t lo_bits, uint32_t hi_bits);

// sdf.cu
struct SdfArgs {
    const FrameGeom* geom;
    CellList trg;
    BatchFrames frames;
    const mdgpu_unitcell_t* cells;   // [B]
    const float* init_xyz;           // [3][num_atoms] initial configuration (device)
    size_t init_axis_stride;
    const float* mass;
    const int32_t* struct_idx;       // [n_struct][struct_size]
    uint32_t n_struct, struct_size;
    const int2* unwrap_pairs;        // (child, parent) local indices in BFS order
    uint32_t n_unwrap;
    float cutoff;
    float4* scratch_xyzw;            // [B][n_struct+1][struct_size]
    float* ref0;                     // [B][20]: VA(16) com0(3) pad
    float* matrices;                 // [B][n_struct][32]: M[16] com[3] pad lo[3] hi[3] cmin[3] cmax[3] (ints)
    uint32_t* vol;                   // [128^3] accumulated voxels
    unsigned long long* frame_total; // [num_frames]
    uint32_t frame0;
};
void launch_sdf(const SdfArgs& a, int B, bool tri, cudaStream_t s);

struct ShapeArgs {                   // shape weights of n_struct structures per frame (VIAMD shape space / _shape_weights)
    BatchFrames frames;
    const mdgpu_unitcell_t* cells;   // [B]
    const float* mass; int use_mass; // weights: atom masses or 1
    const int32_t* idx; const uint32_t* soff; uint32_t n_struct, n_atoms_total;   // CSR: structure s = idx[soff[s] .. soff[s+1])
    float4* scratch_xyzw;            // [B][n_atoms_total]
    float* out;                      // [num_frames][n_struct][3]
    uint32_t frame0;
};
void launch_shape_weights(const ShapeArgs& a, int B, cudaStream_t s);
// an ARRAY of selections as one position argument (coordinate_extract_com :1826-1842): centre of every selection -> d_parts [B][n_parts] (xyz, w = 1),
// then md_util_com_compute_vec4 over them -> d_out[f][arg]
void launch_arg_com_parts(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_idx, const uint32_t* d_off, uint32_t n_parts, const float* d_mass, float4* d_parts, cudaStream_t s);
void launch_arg_combine(const float4* d_parts, uint32_t n_parts, const mdgpu_unitcell_t* d_cells, float* d_out, int arg, int B, cudaStream_t s);

struct RmsdArgs {                    // rmsd(selection) against the initial frame, one value per frame
    BatchFrames frames;
    const mdgpu_unitcell_t* cells;   // [B]
    const float* init_xyz; size_t init_axis_stride;
    const float* mass;
    const int32_t* idx; uint32_t n;  // the selection's atoms, ascending
    const float* pos;                // plane() of an ARRAY of selections: [B][n][3] centres of mass, the n positions (idx unused); else null
    const int2* unwrap_pairs; uint32_t n_unwrap;
    float4* scratch_xyzw;            // [B][2][n]
    float* out;                      // [num_frames], or [num_frames][n_groups] for groups
    uint32_t frame0;
    // rmsd(selection) in <contexts>: n_groups groups of idx[0] (CSR soff); group g walks the n pairs unwrap_pairs[first ..) of group_pairs[g] = (first, n)
    const uint32_t* soff; const uint2* group_pairs; uint32_t n_groups;
};
void launch_rmsd(const RmsdArgs& a, int B, cudaStream_t s);
void launch_rmsd_groups(const RmsdArgs& a, int B, cudaStream_t s);   // one value per group and frame (k_rmsd_groups)
void launch_plane(const RmsdArgs& a, int B, cudaStream_t s);   // plane(selection): out is [num_frames][4], scratch [B][n], init_xyz unused

// within.cu — count(within(radius, selection))
struct WithinArgs {
    const FrameGeom* geom;           // grid of ALL atoms: cell extent ceil(radius/6)*6, cutoff = radius (get_spatial_acc)
    CellList trg, ref;               // all atoms (clamped cells) / the selection's atoms (home grid)
    const int32_t* sel; uint32_t n_sel;
    float min_r2;                    // within(min:max, ...): a pair counts from d2 >= min * min on; 0 for within(radius, ...)
    const uint8_t* and_mask;         // `selection and within(...)` (_and md_script_functions.inl:1975): [num_atoms] bytes, or null
    uint32_t num_atoms;
    uint8_t* flags;                  // [B][num_atoms], zeroed by the launcher
    float* out;                      // [num_frames]
    uint32_t frame0;
};
void launch_within_count(const WithinArgs& a, int B, bool tri, int sm_count, cudaStream_t s);
// the same marks as a per-frame ascending index list (dyn_idx [B][num_atoms], dyn_n [B]); consumers take it as a DynSel
void launch_within_list(const WithinArgs& a, int B, bool tri, int sm_count, int32_t* d_dyn_idx, uint32_t* d_dyn_n, cudaStream_t s);
// within_x / _y / _z / _xyz(...) [and static] (coordinate_range md_script_functions.inl:2394): marks -> the same per-frame list / count
struct RangeArgs {
    BatchFrames frames;
    float lo[3], hi[3];              // inclusive bounds per axis; unconstrained axes are [-FLT_MAX, FLT_MAX]
    uint32_t has_and;                // 1: `selection and within_*(...)`: only the static side's atoms and_idx[0 .. n_and) are tested; 0: every atom
    const int32_t* and_idx; uint32_t n_and;
    uint32_t num_atoms;
    uint8_t* flags;                  // [B][num_atoms]
};
void launch_range_list(const RangeArgs& a, int B, int sm_count, int32_t* d_dyn_idx, uint32_t* d_dyn_n, cudaStream_t s);
void launch_range_count(const RangeArgs& a, int B, int sm_count, float* d_out, uint32_t frame0, cudaStream_t s);
void launch_scan_home_cells(const FrameGeom* d_geom, const CellList& cl, int B, cudaStream_t s);   // cells.cu: k_scan_cells<1> alone

// props.cu
struct DensityArgs {
    BatchFrames frames; const int32_t* idx; uint32_t n; const float* mass; int axis;
    DynSel dyn;                            // density of a dynamic selection: per-frame list instead of idx / n
    float rc, re, inv_ext, min_point;      // reference point / extent / 1/extent / lower bound along the axis (initial cell)
    unsigned long long* acc;               // [1024] fixed-point mass sums (2^-24 Da)
    unsigned long long* frame_bins;        // [B][1024] scratch, zeroed by launcher
    unsigned long long* frame_min; unsigned long long* frame_max;   // [num_frames]
    unsigned long long* keep;              // [num_frames][1024] or null
    uint32_t frame0;
};
void launch_density(const DensityArgs& a, int B, cudaStream_t s);

struct TemporalArgs {
    BatchFrames frames; const mdgpu_unitcell_t* cells; int op; int atom[4]; float* out; uint32_t frame0;
    const float* pos; uint32_t com_mask;   // [B][4][3] centres of mass (k_arg_com) for the arguments whose bit is set
    const int32_t* ctx_idx[4]; uint32_t n_ctx;   // `expr in contexts`: per-context atom of each argument (k_temporal_ctx), out is [num_frames][n_ctx]
    const float4* ctx_pos[4];                    // ... or, for an argument that is a selection, [B][n_ctx] centres of mass of (selection AND context) (k_arg_com_parts); null: the atom
};
void launch_temporal_ctx(const TemporalArgs& a, int B, cudaStream_t s);
void launch_arg_com(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_idx, uint32_t count, const float* d_mass, float* d_out, int arg, cudaStream_t s, DynSel dyn = DynSel{ nullptr, nullptr, 0 });
void launch_temporal(const TemporalArgs& a, int B, cudaStream_t s);
void launch_com_rows(const TemporalArgs& a, int B, cudaStream_t s);   // com(x): row (frame0 + f) of a [num_frames][3] temporal = position of argument 0
void launch_min_distance(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb, float* d_out, uint32_t frame0, cudaStream_t s,
                         DynSel da = DynSel{ nullptr, nullptr, 0 }, DynSel db = DynSel{ nullptr, nullptr, 0 });
void launch_min_distance_pos(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb,
                             const float* d_posa, const float* d_posb, float* d_out, uint32_t frame0, cudaStream_t s);   // an argument that was an array of selections: its groups' centres of mass
void launch_coord_rows_pos(const float* d_pos, uint32_t n, int axis, float* d_out, uint32_t frame0, int B, cudaStream_t s);
void launch_distance_pair(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb,
                          const float* d_posa, const float* d_posb, float* d_out, uint32_t frame0, cudaStream_t s);   // d_pos*: [B][n][3] group centres or null (atoms)
void launch_coord_rows(const BatchFrames& fr, const int32_t* d_idx, uint32_t n, int axis, float* d_out, uint32_t frame0, cudaStream_t s);   // coord_x/_y/_z
void launch_temporal_histogram(const float* d_values, const unsigned long long* d_mask, uint32_t num_frames, uint32_t dim, float range_min, float range_max, float inv_range,
                               uint32_t num_bins, int aggregate, uint32_t* d_counts, uint32_t* d_totals, cudaStream_t s);
void launch_mean_u32(const uint32_t* d_in, float* d_out, size_t count, unsigned long long n, cudaStream_t s);

// expr.cu — temporal expressions (MDGPU_OP_EXPRESSION): one launch per dependency level of a batch, one block row per expression
struct ExprNode { uint32_t kind; float value; const float* src; uint32_t src_len; };   // PROP: src = [num_frames][src_len] rows of the operand
struct ExprProg { uint32_t first_node, num_nodes; float* out; uint32_t len; };         // out = [num_frames][len] rows of the expression
void launch_temporal_expr(const ExprProg* d_progs, uint32_t n_progs, const ExprNode* d_nodes, uint32_t max_len, uint32_t frame0, int B, cudaStream_t s);

// rama.cu — VIAMD's Ramachandran density maps from the (phi, psi) rows of a backbone-angles temporal
struct RamaArgs {
    const float* angles; uint32_t n_seg;         // [num_frames][n_seg][2]
    const uint32_t* seg; uint32_t n_entries;      // the class lists back to back: segment index per entry
    uint32_t class_end[3];                        // entries [0, class_end[0]) are class 0, ... [class_end[2], n_entries) class 3
    uint32_t frame_beg, frame_count; const unsigned long long* mask;   // frames [beg, beg + count) whose mask bit is set
    float scale;                                  // (float)(1 / 2pi): angle -> texture coordinate
    unsigned long long* counts;                   // [512][512][4] scratch (element (x, y, c) at (x * 512 + y) * 4 + c)
    unsigned long long* samples;                  // [4] samples per class
    float* buf[3];                                // [512][512][4] float scratch each; the blurred map ends in buf[1] as [y][x][c]
    int box[3];                                   // box radii of the three passes per axis (boxes_for_gauss)
    int sm_count;
};
void launch_rama_density(const RamaArgs& a, cudaStream_t s);

// porosity.cu — porosity(selection): the unoccupied fraction of a 512-voxel bit grid over the selection's van der Waals spheres, per frame
constexpr uint32_t PORO_FRAMES = 8;                         // frames per sub-batch: one grid each, per stream slot
constexpr size_t PORO_GRID_WORDS = (size_t)8 * 512 * 512;   // the largest grid: ceil(512 / 64) words per row x 512 x 512 rows (16 MiB)
struct PorosityHdr {                 // per frame, written by k_porosity_prepare
    float bmin[3], d[3];             // box minimum, voxel size per axis
    int dim[3];                      // voxels per axis; the longest axis has 512
    uint32_t row_words;              // 64-bit words per grid row, ceil(dim[0] / 64)
    uint32_t valid;                  // 0: triclinic cell or empty selection, the value is 0
};
struct PorosityArgs {
    BatchFrames frames;              // the sub-batch: at most PORO_FRAMES frames
    const mdgpu_unitcell_t* cells;   // [frames.count]
    const int32_t* idx; uint32_t n;  // the selection's atoms, ascending
    const float* radius;             // [atoms] van der Waals radii in the frames' atom space
    float4* xyzr;                    // [PORO_FRAMES][n] scratch
    PorosityHdr* hdr;                // [PORO_FRAMES]
    unsigned long long* grid;        // [PORO_FRAMES][PORO_GRID_WORDS], all zero between calls
    unsigned long long* count;       // [PORO_FRAMES], all zero between calls
    unsigned long long* frame_set;   // [num_frames] occupied voxels
    unsigned long long* frame_n;     // [num_frames] voxels of the grid (N)
    float* out;                      // [num_frames]
    uint32_t frame0;                 // global index of the sub-batch's first frame
};
void launch_porosity(const PorosityArgs& a, int nf, cudaStream_t s);

// dssp.cu — secondary structure of every backbone segment per frame (md_util_backbone_secondary_structure_infer)
constexpr uint32_t SS_RES_FLOATS = 20;   // per (frame, segment): N, CA, C, O, H (xyz each), the CA's cell-grid coordinates (3) and packed cell
struct SsArgs {
    BatchFrames frames;
    const int32_t* atoms;            // [S][5] N, CA, C, O, HN (-1: estimated) in the frames' atom space
    const uint32_t* seg;             // [S][3] range id, range begin, range end of each segment
    uint32_t S;
    const FrameGeom* geom;           // [B] the candidate walk's grid (cell extent and cutoff 9 A) of each frame
    float* res;                      // [B][S][SS_RES_FLOATS] scratch
    float4* hb;                      // [B][S] per donor: the two lowest energies <= -0.5 (acceptor bits, energy, acceptor bits, energy)
    uint32_t* bits;                  // [B][2][S] scratch: turn / bend bits, then the structure flags
    float* out;                      // [num_frames][S] codes as floats
    uint32_t frame0;
    int* err;                        // MDGPU_ERR_UNSUPPORTED: a frame's grid cannot visit each candidate pair once
};
void launch_secondary_structure(const SsArgs& a, int B, bool tri, cudaStream_t s);

// xtc.cu — compressed trajectory frames expanded on the device
struct XtcFrameInfo {   // written by k_xtc_scan, one per frame
    int status;                 // 0 ok, otherwise the frame is malformed
    uint32_t ngroups, data_off; // groups found by the scan; byte offset of the bit stream inside the frame
    uint32_t bitsize, bitsizeint[3], sizeint[3]; int minint[3]; float precision;
    uint32_t rounds, restages;  // scan statistics (diagnostics)
};
void launch_xtc_decode(const uint8_t* d_blob, const unsigned long long* d_frame_off, uint32_t num_atoms, int B, XtcFrameInfo* d_info,
                       uint2* d_rec, uint16_t* d_rec_state, size_t rec_stride, float* d_out, size_t frame_stride, size_t axis_stride, int* d_err, cudaStream_t s);

void launch_xtc_scan(const uint8_t* d_blob, const unsigned long long* d_frame_off, uint32_t num_atoms, int nframes, XtcFrameInfo* d_info,
                     uint2* d_rec, uint16_t* d_rec_state, size_t rec_stride, cudaStream_t s);
void launch_xtc_expand(const uint8_t* d_blob, const unsigned long long* d_frame_off, uint32_t num_atoms, int nframes, const XtcFrameInfo* d_info,
                       const uint2* d_rec, const uint16_t* d_rec_state, size_t rec_stride, float* d_out, size_t frame_stride, size_t axis_stride, int* d_err, cudaStream_t s);

// synth.cu
void launch_synth_frames(uint32_t seed, float Lx, float Ly, float Lz, uint32_t num_atoms, const float* d_base, size_t base_axis_stride,
                         const uint32_t* d_mol_id, uint32_t frame_beg, uint32_t count, float* d_out, size_t frame_stride, size_t axis_stride, cudaStream_t s);

}  // namespace mdg
