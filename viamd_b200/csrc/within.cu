// within.cu — dynamic selections: within(radius, selection) and the coordinate ranges within_x / _y / _z / _xyz, evaluated per frame.
//
// Replaces _within_expl_flt + within_float_cb (reference md_script_functions.inl:2478-2533) over the system-wide cell list of
// get_spatial_acc (:734-760: every atom of the system, cell extent ceil(radius / 6) * 6), and _count (:2868) on the result:
// the atoms of the system within `radius` of any atom of the selection, the selection's own atoms excluded (:2521-2525); the min:max form
// (_within_expl_frng :2609) queries at max and accepts a pair from d2 >= min * min on.
//
// The cell lists come from cells.cu exactly as for rdf(): targets = all atoms (clamped cells), references = the selection's atoms in
// the home grid. The pair enumeration is the reference's (core/md_spatial_acc.c:1649-1803 / :1498-1647): (2n+1)^3 neighbour offsets of
// the reference point's cell, wrapped once, the reference point shifted by the periodic image, wraps on non-periodic axes skipped;
// d2 = fma(G00, dx*dx, fma(G11, dy*dy, G22*dz*dz)) (+ cross terms, triclinic) compared with calc_r2(radius) (:541-544). A pair within
// the radius sets the target atom's flag; flags are idempotent, so no ordering between warps matters.
#include "common.cuh"
#include "kernels.h"
#include "cellmath.cuh"

namespace mdg {

constexpr int WITHIN_WARPS = 4;

// One warp per home cell (grid-stride): for every neighbour cell the lanes take its target points 32 at a time and test them against
// the home cell's reference points until one is within the radius.
template <bool TRI>
__global__ void __launch_bounds__(WITHIN_WARPS * 32) k_within_mark(WithinArgs a) {
    const int f = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const FrameGeom& g = a.geom[f];
    if (g.valid <= 0) return;
    const float4* __restrict__ trg = a.trg.sorted + (size_t)f * a.trg.max_points;
    const uint32_t* __restrict__ trg_off = a.trg.cell_cnt + (size_t)f * (a.trg.cap + 1);
    const float4* __restrict__ ref = a.ref.sorted + (size_t)f * a.ref.max_points;
    const uint32_t* __restrict__ ref_off = a.ref.cell_cnt + (size_t)f * (a.ref.cap + 1);
    uint8_t* __restrict__ flags = a.flags + (size_t)f * a.num_atoms;
    const CellWalk w = cell_walk(g);
    const int nn = walk_size(w);
    const float r2 = g.r2, min_r2 = a.min_r2;
    for (uint32_t h = blockIdx.x * WITHIN_WARPS + warp; h < g.num_home; h += gridDim.x * WITHIN_WARPS) {
        const uint32_t rb = ref_off[h], re = ref_off[h + 1];
        if (rb == re) continue;
        const int3 c = home_cell(g, h);
        for (int n = 0; n < nn; ++n) {
            const Neighbour nb = neighbour_cell<TRI>(w, c, n);
            if (!nb.ok) continue;
            const uint32_t start = trg_off[nb.cj], len = trg_off[nb.cj + 1] - start;
            const float3 sh = image_shift(nb.code);
            for (uint32_t j = lane; j < len; j += 32) {
                const float4 t = trg[start + j];
                const uint32_t tj = __float_as_uint(t.w);
                if (flags[tj]) continue;   // already marked (by this or another warp): nothing to add
                bool hit = false;
                for (uint32_t i = rb; i < re && !hit; ++i) {
                    const float4 rf = ref[i];
                    const float fx = __fadd_rn(rf.x, sh.x), fy = __fadd_rn(rf.y, sh.y), fz = __fadd_rn(rf.z, sh.z);   // f + image shift (:1755)
                    const float d2 = pair_d2<TRI>(__fsub_rn(fx, t.x), __fsub_rn(fy, t.y), __fsub_rn(fz, t.z), g);
                    hit = d2 <= r2 && d2 >= min_r2;   // within_frng_cb (:2599-2607); min_r2 = 0 for the plain form
                }
                if (hit) flags[tj] = 1;
            }
        }
    }
}

// The selection's own atoms leave the result (md_bitfield_andnot_inplace :2524), then _count (:2868): one CTA per frame.
__global__ void __launch_bounds__(256) k_within_count(WithinArgs a) {
    const int f = blockIdx.x;
    uint8_t* __restrict__ flags = a.flags + (size_t)f * a.num_atoms;
    for (uint32_t k = threadIdx.x; k < a.n_sel; k += blockDim.x) flags[a.sel[k]] = 0;
    __syncthreads();
    uint32_t c = 0;
    for (uint32_t i = threadIdx.x; i < a.num_atoms; i += blockDim.x) c += (flags[i] != 0 && (!a.and_mask || a.and_mask[i] != 0)) ? 1u : 0u;
    __shared__ uint32_t total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    if (c) atomicAdd(&total, c);
    __syncthreads();
    if (threadIdx.x == 0) a.out[a.frame0 + f] = (float)total;
}

// count(x, 'residue' | 'chain' | 'structure') (_count_with_arg -> internal_count md_script_functions.inl:5465-5531): per frame the number of
// groups that hold at least one atom of the selection k_within_count counts. One CTA per frame in three phases, separated by barriers:
//   1. the frame's hit bytes are zeroed and the within() selection's own atoms leave the marks (:2524);
//   2. every marked atom that passes the static `and` side sets the hit byte of its group (idempotent: the stores' order does not matter);
//   3. the set hit bytes are counted.
// O(atoms + groups) per frame whatever the groups' layout; the count is an exact integer.
constexpr int GROUP_THREADS = 1024;
__global__ void __launch_bounds__(GROUP_THREADS) k_group_count(WithinArgs a) {
    const int f = blockIdx.x;
    uint8_t* __restrict__ flags = a.flags + (size_t)f * a.num_atoms;
    uint8_t* __restrict__ hits = a.grp.hits + (size_t)f * a.grp.n_groups;
    const int32_t* __restrict__ group_of = a.grp.group_of;
    __shared__ uint32_t total;
    if (threadIdx.x == 0) total = 0;
    for (uint32_t g = threadIdx.x; g < a.grp.n_groups; g += blockDim.x) hits[g] = 0;
    for (uint32_t k = threadIdx.x; k < a.n_sel; k += blockDim.x) flags[a.sel[k]] = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < a.num_atoms; i += blockDim.x) {
        if (!flags[i] || (a.and_mask && !a.and_mask[i])) continue;
        const int32_t g = group_of[i];
        if (g >= 0) hits[g] = 1;
    }
    __syncthreads();
    uint32_t c = 0;
    for (uint32_t g = threadIdx.x; g < a.grp.n_groups; g += blockDim.x) c += hits[g];
    if (c) atomicAdd(&total, c);
    __syncthreads();
    if (threadIdx.x == 0) a.out[a.frame0 + f] = (float)total;
}

// the per-frame count of the marks: of the atoms, or of the groups they fall in
static void launch_count(const WithinArgs& a, int B, cudaStream_t s) {
    if (a.grp.group_of) {
        k_group_count<<<B, GROUP_THREADS, 0, s>>>(a);
        note_launch("k_group_count", s);
    } else {
        k_within_count<<<B, 256, 0, s>>>(a);
        note_launch("k_within_count", s);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The dynamic selection as the REFERENCE set of an rdf(): rdf(within(radius, selection), targets, cutoff). The marked atoms (selection
// removed) become a per-frame index list; its reference cell list is built like cells.cu builds a static one, but with the frame's own
// list and count (coordinate_extract on a single bitfield: the atoms' positions, ascending index; compute_rdf :5281-5290).
// ---------------------------------------------------------------------------------------------------------------
// flags -> ascending index list, one CTA per frame: 256 atoms per step, ballot prefix inside the warps, running offset across steps
__global__ void __launch_bounds__(256) k_within_compact(WithinArgs a, int32_t* __restrict__ dyn_idx, uint32_t* __restrict__ dyn_n) {
    const int f = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* __restrict__ flags = a.flags + (size_t)f * a.num_atoms;
    for (uint32_t k = threadIdx.x; k < a.n_sel; k += blockDim.x) flags[a.sel[k]] = 0;   // md_bitfield_andnot_inplace (:2524)
    __shared__ uint32_t s_warp[8]; __shared__ uint32_t s_base;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    int32_t* out = dyn_idx + (size_t)f * a.num_atoms;
    for (uint32_t i0 = 0; i0 < a.num_atoms; i0 += 256u) {
        const uint32_t i = i0 + threadIdx.x;
        const bool on = i < a.num_atoms && flags[i] != 0 && (!a.and_mask || a.and_mask[i] != 0);
        const uint32_t m = __ballot_sync(0xffffffffu, on);
        if (lane == 0) s_warp[warp] = (uint32_t)__popc(m);
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (int w = 0; w < 8; ++w) { const uint32_t c = s_warp[w]; before += (w < warp) ? c : 0u; total += c; }
        const uint32_t base = s_base;
        if (on) out[base + before + (uint32_t)__popc(m & ((1u << lane) - 1u))] = (int32_t)i;
        __syncthreads();
        if (threadIdx.x == 0) s_base = base + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) dyn_n[f] = s_base;
}

// zero the flags, mark: a few CTAs per frame, enough to fill the SMs across the batch
static void launch_mark(const WithinArgs& a, int B, bool tri, int sm_count, cudaStream_t s) {
    cudaMemsetAsync(a.flags, 0, (size_t)B * a.num_atoms, s);
    if (!a.n_sel) return;
    const dim3 grid((unsigned)max(1, (4 * sm_count) / max(B, 1) + 1), (unsigned)B);
    if (tri) k_within_mark<true><<<grid, WITHIN_WARPS * 32, 0, s>>>(a); else k_within_mark<false><<<grid, WITHIN_WARPS * 32, 0, s>>>(a);
    note_launch("k_within_mark", s);
}

// within() marks -> per-frame reference list (dyn_idx [B][num_atoms], dyn_n [B])
void launch_within_list(const WithinArgs& a, int B, bool tri, int sm_count, int32_t* d_dyn_idx, uint32_t* d_dyn_n, cudaStream_t s) {
    if (B <= 0) return;
    launch_mark(a, B, tri, sm_count, s);
    k_within_compact<<<B, 256, 0, s>>>(a, d_dyn_idx, d_dyn_n);
    note_launch("k_within_compact", s);
}

void launch_within_count(const WithinArgs& a, int B, bool tri, int sm_count, cudaStream_t s) {
    if (B <= 0) return;
    launch_mark(a, B, tri, sm_count, s);
    launch_count(a, B, s);
}

// ---------------------------------------------------------------------------------------------------------------
// Coordinate ranges within_x / _y / _z / _xyz(...) (coordinate_range md_script_functions.inl:2394-2476, the form outside an `in` context):
// atom i is selected iff lo <= p[i] <= hi on all three axes, on the frame's raw coordinates. Unconstrained axes come as [-FLT_MAX, FLT_MAX] and
// are compared like the others, so a NaN or infinite coordinate is never selected. No atom is removed afterwards: the compaction and the count
// run with n_sel = 0. One frame per block row; with a static `and` side only its atoms are tested (the flags were zeroed first), otherwise
// every atom's flag is written.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_range_mark(RangeArgs a) {
    const int f = blockIdx.y;
    const float* __restrict__ x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    const float* __restrict__ y = x + a.frames.axis_stride;
    const float* __restrict__ z = y + a.frames.axis_stride;
    uint8_t* __restrict__ flags = a.flags + (size_t)f * a.num_atoms;
    const uint32_t n = a.has_and ? a.n_and : a.num_atoms;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = a.has_and ? (uint32_t)a.and_idx[j] : j;
        const float px = x[i], py = y[i], pz = z[i];
        const bool in = a.lo[0] <= px && px <= a.hi[0] && a.lo[1] <= py && py <= a.hi[1] && a.lo[2] <= pz && pz <= a.hi[2];
        if (!a.has_and) flags[i] = in ? 1 : 0;
        else if (in) flags[i] = 1;
    }
}

// the marks of a batch, and the WithinArgs under which k_within_compact / k_within_count read them
static WithinArgs range_mark(const RangeArgs& a, int B, int sm_count, cudaStream_t s) {
    const uint32_t n = a.has_and ? a.n_and : a.num_atoms;
    if (a.has_and) cudaMemsetAsync(a.flags, 0, (size_t)B * a.num_atoms, s);
    if (n) {
        const unsigned per_frame = (unsigned)min((n + 255u) / 256u, (uint32_t)max(1, (8 * sm_count) / max(B, 1)));
        k_range_mark<<<dim3(per_frame, (unsigned)B), 256, 0, s>>>(a);
        note_launch("k_range_mark", s);
    }
    WithinArgs w{};
    w.num_atoms = a.num_atoms; w.flags = a.flags;   // n_sel = 0, no and_mask: the marks are the selection
    return w;
}

void launch_range_list(const RangeArgs& a, int B, int sm_count, int32_t* d_dyn_idx, uint32_t* d_dyn_n, cudaStream_t s) {
    if (B <= 0) return;
    const WithinArgs w = range_mark(a, B, sm_count, s);
    k_within_compact<<<B, 256, 0, s>>>(w, d_dyn_idx, d_dyn_n);
    note_launch("k_within_compact", s);
}

void launch_range_count(const RangeArgs& a, const GroupArgs& g, int B, int sm_count, float* d_out, uint32_t frame0, cudaStream_t s) {
    if (B <= 0) return;
    WithinArgs w = range_mark(a, B, sm_count, s);
    w.out = d_out; w.frame0 = frame0; w.grp = g;
    launch_count(w, B, s);
}

}  // namespace mdg
