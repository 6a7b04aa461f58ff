// cells.cu — K1: per-frame cell-list build for a batch of frames.
//
// Replaces md_spatial_acc_init (reference core/md_spatial_acc.c:155-438): fractional coordinates
// s = (r - origin) * I, wrap of periodic axes with s - floor(s), cell = clamp(floor(s * dim)), counting sort.
// The geometry (metric G, inverse basis I, grid dims, neighbour reach) is derived on the device in double precision,
// one thread per frame, with the reference's exact expression order, so NPT trajectories (cell changes every frame)
// cost nothing extra on the host.
//
// Order of points inside a cell is arbitrary here (atomic ranks) whereas the reference keeps input order; every
// consumer on the path (histogram / voxel increments) is order independent.
#include "common.cuh"
#include "kernels.h"
#include "cellmath.cuh"
#include "pbcmath.cuh"

namespace mdg {

// ---------------------------------------------------------------------------------------------------------------
// Geometry, mirrors core/md_spatial_acc.c:179-300 and :1650-1659 (ext-pair neighbour reach) and :541-544 (calc_r2)
// ---------------------------------------------------------------------------------------------------------------
MDG_HD void compute_frame_geom(FrameGeom& g, const mdgpu_unitcell_t& uc, double in_cell_ext, double cutoff,
                               const float* aabb /* min[3], max[3] of the points incl. the origin, or nullptr */, uint32_t cell_cap) {
    if (in_cell_ext <= 0.0) in_cell_ext = 6.0;
    const double CELL_EXT = in_cell_ext > 3.0 ? in_cell_ext : 3.0;
    double A[3][3] = { { 1, 0, 0 }, { 0, 1, 0 }, { 0, 0, 1 } }, I[3][3] = { { 1, 0, 0 }, { 0, 1, 0 }, { 0, 0, 1 } };
    const uint32_t flags = uc.flags;
    // md_unitcell_A_extract_double / md_unitcell_I_extract_double (md_unitcell.inl:129-175)
    A[0][0] = uc.x;  A[0][1] = 0;     A[0][2] = 0;
    A[1][0] = uc.xy; A[1][1] = uc.y;  A[1][2] = 0;
    A[2][0] = uc.xz; A[2][1] = uc.yz; A[2][2] = uc.z;
    if (!flags) {
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) I[i][j] = 0.0;
    } else cell_inverse(uc, I);
    float origin[3] = { 0.f, 0.f, 0.f };
    if ((flags & MDGPU_CELL_PBC_ALL) != MDGPU_CELL_PBC_ALL && aabb) {
        for (int k = 0; k < 3; ++k) {
            const float mn = aabb[k], mx = aabb[3 + k];
            float ext = mx - mn;
            ext = ceilf(ext / (float)CELL_EXT) * (float)CELL_EXT;
            const float cen = (mn + mx) * 0.5f;
            const float lo = cen - ext * 0.5f;
            if ((flags & (MDGPU_CELL_PBC_X << k)) == 0) {
                origin[k] = lo;
                if (ext > 0.0f) { A[k][k] = ext; I[k][k] = 1.0 / ext; }
            }
        }
    }
    const double a0 = A[0][0], a1 = A[0][1], a2 = A[0][2];
    const double b0 = A[1][0], b1 = A[1][1], b2 = A[1][2];
    const double c0 = A[2][0], c1 = A[2][1], c2 = A[2][2];
    const double G00 = a0 * a0 + a1 * a1 + a2 * a2;
    const double G11 = b0 * b0 + b1 * b1 + b2 * b2;
    const double G22 = c0 * c0 + c1 * c1 + c2 * c2;
    const double G01 = a0 * b0 + a1 * b1 + a2 * b2;
    const double G02 = a0 * c0 + a1 * c1 + a2 * c2;
    const double G12 = b0 * c0 + b1 * c1 + b2 * c2;
    double H01 = 0.0, H02 = 0.0, H12 = 0.0;
    const double na = sqrt(G00), nb = sqrt(G11), nc = sqrt(G22);
    g.inv_cell_ext[0] = (float)(na > 0.0 ? 1.0 / na : 0.0);
    g.inv_cell_ext[1] = (float)(nb > 0.0 ? 1.0 / nb : 0.0);
    g.inv_cell_ext[2] = (float)(nc > 0.0 ? 1.0 / nc : 0.0);
    g.valid = 1;
    if (flags & MDGPU_CELL_TRICLINIC) {
        H01 = 2.0 * G01; H02 = 2.0 * G02; H12 = 2.0 * G12;
        const double det = G00 * (G11 * G22 - G12 * G12) - G01 * (G01 * G22 - G12 * G02) + G02 * (G01 * G12 - G11 * G02);
        if (det < DBL_EPSILON) g.valid = 0;
        g.inv_cell_ext[0] = (float)sqrt((G11 * G22 - G12 * G12) / det);
        g.inv_cell_ext[1] = (float)sqrt((G00 * G22 - G02 * G02) / det);
        g.inv_cell_ext[2] = (float)sqrt((G00 * G11 - G01 * G01) / det);
    }
    uint32_t cd[3] = { (uint32_t)(na / CELL_EXT), (uint32_t)(nb / CELL_EXT), (uint32_t)(nc / CELL_EXT) };
    for (int k = 0; k < 3; ++k) { cd[k] = cd[k] < 1u ? 1u : (cd[k] > 1024u ? 1024u : cd[k]); g.cdim[k] = (int)cd[k]; }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { g.A[i][j] = (float)A[i][j]; g.I[i][j] = (float)I[i][j]; }
    for (int k = 0; k < 3; ++k) g.origin[k] = origin[k];
    g.G00 = (float)G00; g.G11 = (float)G11; g.G22 = (float)G22;
    g.H01 = (float)H01; g.H02 = (float)H02; g.H12 = (float)H12;
    g.flags = flags;
    const uint64_t ncells = (uint64_t)cd[0] * cd[1] * cd[2];
    g.num_cells = (uint32_t)(ncells > 0xffffffffull ? 0xffffffffull : ncells);
    // neighbour reach of for_each_external_pair_within_cutoff_* (:1650-1659)
    for (int k = 0; k < 3; ++k) {
        g.ncell[k] = (int)ceil(cutoff * (double)g.inv_cell_ext[k] * (double)cd[k]);
        if (2 * g.ncell[k] + 1 > 5) g.valid = 0;   // reference logs "cutoff too large for cell size" and returns no pairs
        const int reach = g.ncell[k] < 0 ? 0 : (g.ncell[k] > 2 ? 2 : g.ncell[k]);
        // Home grid = range of unclamped reference cell coordinates that can still reach a valid cell after the
        // reference's single wrap. Ortho wraps the reference point first (coordinate in [0,cdim]); the triclinic query
        // does not (:1565), so a point up to one period outside the cell is still served by the single wrap.
        const int extra = (flags & MDGPU_CELL_TRICLINIC) ? (int)cd[k] : 0;
        g.hlo[k] = -extra - reach - 1;
        g.hdim[k] = (int)cd[k] + 2 * extra + 2 * reach + 2;
    }
    g.num_home = (uint32_t)((uint64_t)g.hdim[0] * g.hdim[1] * g.hdim[2]);
    g.sym_ok = 1;
    for (int k = 0; k < 3; ++k) if ((flags & (MDGPU_CELL_PBC_X << k)) && (int)cd[k] < 2 * g.ncell[k] + 1) g.sym_ok = 0;
    {   // calc_r2: (float)(cutoff^2) rounded up by one ulp
        const float r2 = (float)(cutoff * cutoff);
        g.r2 = nextafterf(r2, r2 + 1.0f);
    }
    if (ncells + 1 > cell_cap || (uint64_t)g.num_home + 1 > cell_cap) g.valid = -1;   // capacity error, reported by the host
}

void host_frame_geom(FrameGeom* g, const mdgpu_unitcell_t* uc, double cell_ext, double cutoff, const float* aabb, uint32_t cap) {
    compute_frame_geom(*g, *uc, cell_ext, cutoff, aabb, cap);
}

__global__ void k_frame_geom(const mdgpu_unitcell_t* __restrict__ cells, const float* __restrict__ aabb, FrameGeom* __restrict__ out,
                             double cell_ext, double cutoff, uint32_t cap, int B, int* __restrict__ err) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= B) return;
    FrameGeom g;
    compute_frame_geom(g, cells[f], cell_ext, cutoff, aabb ? aabb + 6 * f : nullptr, cap);
    out[f] = g;
    if (g.valid < 0) atomicExch(err, MDGPU_ERR_CAPACITY);
}

// AABB of the target points (only when an axis is non-periodic, :201-243). The box starts at the origin ({0} init).
MDG_D void atomic_min_f(float* addr, float v) {
    int* ia = (int*)addr; int old = *ia;
    while (__int_as_float(old) > v) { const int assumed = old; old = atomicCAS(ia, assumed, __float_as_int(v)); if (old == assumed) break; }
}
MDG_D void atomic_max_f(float* addr, float v) {
    int* ia = (int*)addr; int old = *ia;
    while (__int_as_float(old) < v) { const int assumed = old; old = atomicCAS(ia, assumed, __float_as_int(v)); if (old == assumed) break; }
}

__global__ void k_aabb(BatchFrames fr, const int32_t* __restrict__ idx_, uint32_t n_, float* __restrict__ aabb /* [B][6], zero-initialised */, DynSel dyn,
                       const float* __restrict__ aos = nullptr /* [B][n][3]: positions given directly (centres of mass of groups) instead of atoms */) {
    const int f = blockIdx.y;
    const int32_t* __restrict__ idx = sel_list(idx_, dyn, f); const uint32_t n = sel_count(n_, dyn, f);
    const float* x = fr.xyz + (size_t)f * fr.frame_stride; const float* y = x + fr.axis_stride; const float* z = y + fr.axis_stride;
    float mn[3] = { 0.f, 0.f, 0.f }, mx[3] = { 0.f, 0.f, 0.f };
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float r[3];
        if (aos) { const float* q = aos + ((size_t)f * n + i) * 3; r[0] = q[0]; r[1] = q[1]; r[2] = q[2]; }
        else { const int a = idx ? idx[i] : (int)i; r[0] = x[a]; r[1] = y[a]; r[2] = z[a]; }
        for (int k = 0; k < 3; ++k) { mn[k] = fminf(mn[k], r[k]); mx[k] = fmaxf(mx[k], r[k]); }
    }
    for (int k = 0; k < 3; ++k) {
        for (int o = 16; o > 0; o >>= 1) { mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o)); mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o)); }
    }
    if ((threadIdx.x & 31) == 0) for (int k = 0; k < 3; ++k) { atomic_min_f(aabb + 6 * f + k, mn[k]); atomic_max_f(aabb + 6 * f + 3 + k, mx[k]); }
}

// MODE 0: internal (target) points -> clamped cell index (:341-371)
// MODE 1: external (reference) points -> unclamped home cell (:1713-1719 ortho wraps periodic axes, :1561-1566 triclinic does not)
template <int MODE>
__global__ void k_bin_points(BatchFrames fr, const int32_t* __restrict__ idx_, const float* __restrict__ aos /* [B][n][3] or null */, uint32_t n_,
                             const FrameGeom* __restrict__ geom, CellList cl, int store_linear_idx, DynSel dyn) {
    const int f = blockIdx.y;
    const int32_t* __restrict__ idx = sel_list(idx_, dyn, f); const uint32_t n = sel_count(n_, dyn, f);   // per-frame list of a dynamic selection, or the static one
    __shared__ FrameGeom g;
    for (int k = threadIdx.x; k < (int)(sizeof(FrameGeom) / 4); k += blockDim.x) ((uint32_t*)&g)[k] = ((const uint32_t*)&geom[f])[k];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float r[3]; uint32_t tag;
    if (aos) {
        const float* p = aos + ((size_t)f * n + i) * 3;
        r[0] = p[0]; r[1] = p[1]; r[2] = p[2]; tag = i;
    } else {
        const int a = idx ? idx[i] : (int)i;
        const float* x = fr.xyz + (size_t)f * fr.frame_stride;
        r[0] = x[a]; r[1] = x[fr.axis_stride + a]; r[2] = x[2 * fr.axis_stride + a];
        tag = store_linear_idx ? i : (uint32_t)a;
    }
    float s[3]; cart_to_fract(s, r, g);
    const bool tri = (g.flags & MDGPU_CELL_TRICLINIC) != 0;
    uint32_t cell;
    if (MODE == 0) {
        int cc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (g.flags & (MDGPU_CELL_PBC_X << k)) s[k] = __fsub_rn(s[k], floorf(s[k]));
            int ic = (int)floorf(__fmul_rn(s[k], (float)g.cdim[k]));
            ic = max(0, min(ic, g.cdim[k] - 1));
            cc[k] = ic;
        }
        cell = ((uint32_t)cc[2] * (uint32_t)g.cdim[1] + (uint32_t)cc[1]) * (uint32_t)g.cdim[0] + (uint32_t)cc[0];
    } else {
        int hc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (!tri && (g.flags & (MDGPU_CELL_PBC_X << k))) s[k] = __fsub_rn(s[k], floorf(s[k]));
            const float cf = floorf(__fmul_rn(s[k], (float)g.cdim[k]));
            // keep the unclamped reference cell coordinate; anything beyond the neighbour reach collapses onto the
            // sentinel planes hlo / hlo+hdim-1, which have no valid neighbours
            const float lo = (float)g.hlo[k], hi = (float)(g.hlo[k] + g.hdim[k] - 1);
            const float cl_ = fminf(fmaxf(cf, lo), hi);
            hc[k] = (int)cl_ - g.hlo[k];
            if (!(cf == cf)) hc[k] = 0;   // NaN coordinate: park on the sentinel plane
            if (!(cf >= 0.0f && cf < (float)g.cdim[k])) cl.oob[f] = 1u;   // e.g. fract() rounded up to 1.0: home cell != target cell of the same atom
        }
        cell = ((uint32_t)hc[2] * (uint32_t)g.hdim[1] + (uint32_t)hc[1]) * (uint32_t)g.hdim[0] + (uint32_t)hc[0];
    }
    if (g.valid <= 0) cell = 0;
    const size_t o = (size_t)f * cl.max_points + i;
    cl.scratch[o] = make_float4(s[0], s[1], s[2], __uint_as_float(tag));
    cl.cell_of[o] = cell;
    cl.rank[o] = atomicAdd(&cl.cell_cnt[(size_t)f * (cl.cap + 1) + cell], 1u);
}

// exclusive scan of the per-cell counts, one CTA per frame; writes offsets in place, total at [num]
template <int MODE>
__global__ void k_scan_cells(const FrameGeom* __restrict__ geom, CellList cl) {
    const int f = blockIdx.x;
    const uint32_t num = (MODE == 0) ? geom[f].num_cells : geom[f].num_home;
    uint32_t* cnt = cl.cell_cnt + (size_t)f * (cl.cap + 1);
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (uint32_t base = 0; base < num + 1; base += blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = (i < num) ? cnt[i] : 0u;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = (lane < nwarps) ? warp_sums[lane] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
            warp_sums[lane] = w;   // inclusive over warps
        }
        __syncthreads();
        const uint32_t warp_off = warp ? warp_sums[warp - 1] : 0u;
        const uint32_t c = carry;
        if (i <= num) cnt[i] = c + warp_off + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = c + warp_off + incl;
        __syncthreads();
    }
}

__global__ void k_scatter_points(uint32_t n, CellList cl, const uint32_t* __restrict__ dyn_n) {
    const int f = blockIdx.y;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (dyn_n ? dyn_n[f] : n)) return;
    const size_t o = (size_t)f * cl.max_points + i;
    const uint32_t dst = cl.cell_cnt[(size_t)f * (cl.cap + 1) + cl.cell_of[o]] + cl.rank[o];
    cl.sorted[(size_t)f * cl.max_points + dst] = cl.scratch[o];
}

// ---------------------------------------------------------------------------------------------------------------
// Host-side launch sequence for one cell list
// ---------------------------------------------------------------------------------------------------------------
void launch_geom(const mdgpu_unitcell_t* d_cells, const float* d_aabb, FrameGeom* d_geom, double cell_ext, double cutoff, uint32_t cap,
                 int B, int* d_err, cudaStream_t s) {
    k_frame_geom<<<(B + 63) / 64, 64, 0, s>>>(d_cells, d_aabb, d_geom, cell_ext, cutoff, cap, B, d_err);
    note_launch("k_frame_geom", s);
}

void launch_aabb(const BatchFrames& fr, const int32_t* d_idx, uint32_t n, float* d_aabb, cudaStream_t s, DynSel dyn, const float* d_aos) {
    cudaMemsetAsync(d_aabb, 0, sizeof(float) * 6 * fr.count, s);
    if (dyn.n) n = dyn.stride;   // upper bound of a per-frame list
    if (!n) return;
    dim3 grid(min((n + 255u) / 256u, 64u), fr.count);
    k_aabb<<<grid, 256, 0, s>>>(fr, d_idx, n, d_aabb, dyn, d_aos);
    note_launch("k_aabb", s);
}

void launch_scan_home_cells(const FrameGeom* d_geom, const CellList& cl, int B, cudaStream_t s) {
    k_scan_cells<1><<<B, 1024, 0, s>>>(d_geom, cl);
    note_launch("k_scan_cells", s);
}

void launch_cell_list(int mode, const BatchFrames& fr, const int32_t* d_idx, const float* d_aos, uint32_t n, const FrameGeom* d_geom,
                      const CellList& cl, int store_linear_idx, cudaStream_t s, DynSel dyn) {
    cudaMemsetAsync(cl.cell_cnt, 0, sizeof(uint32_t) * (size_t)fr.count * (cl.cap + 1), s);
    cudaMemsetAsync(cl.oob, 0, sizeof(uint32_t) * fr.count, s);
    if (dyn.n) n = dyn.stride;   // grid for the longest possible per-frame list; each frame stops at its own count
    if (n) {
        dim3 grid((n + 255u) / 256u, fr.count);
        if (mode == 0) k_bin_points<0><<<grid, 256, 0, s>>>(fr, d_idx, d_aos, n, d_geom, cl, store_linear_idx, dyn);
        else           k_bin_points<1><<<grid, 256, 0, s>>>(fr, d_idx, d_aos, n, d_geom, cl, store_linear_idx, dyn);
        note_launch("k_bin_points", s);
    }
    if (mode == 0) k_scan_cells<0><<<fr.count, 1024, 0, s>>>(d_geom, cl);
    else           k_scan_cells<1><<<fr.count, 1024, 0, s>>>(d_geom, cl);
    note_launch("k_scan_cells", s);
    if (n) {
        dim3 grid((n + 255u) / 256u, fr.count);
        k_scatter_points<<<grid, 256, 0, s>>>(n, cl, dyn.n);
        note_launch("k_scatter_points", s);
    }
}

}  // namespace mdg
