// porosity.cu — porosity(selection) per frame (_porosity, md_script_functions.inl:5858-6003): the selection's van der Waals spheres are
// voxelised into a bit grid over their bounding box, whose longest axis has 512 voxels, and the value is the grid's unoccupied fraction.
//
// Per sub-batch of at most PORO_FRAMES frames:
//   k_porosity_prepare  : one block per frame. Gather (x, y, z, radius) of the selected atoms, md_util_com_compute_vec4 on one thread (index order,
//                         pbcmath.cuh), md_util_deperiodize_vec4 about it, the box min(p - r) / max(p + r), then the grid header.
//   k_porosity_voxelise : one warp per sphere, the lanes over the rows (iy, iz) of its voxel box. A lane tests the voxels of its row run word by
//                         word into a 64-bit mask and issues one atomicOr per non-zero word. Rows are padded to whole words.
//   k_porosity_count    : popcount of every used word of a frame's grid, which it zeroes again, so a grid is all zero between sub-batches.
//   k_porosity_finalize : occupied voxels and N per frame into the u64 rows, (float)((N - set) / N) in double into the temporal row.
//
// Every float operation keeps the reference's operands and rounding; the two fmaf of the voxel test are the only fused operations.
#include "common.cuh"
#include "kernels.h"
#include "pbcmath.cuh"

namespace mdg {

constexpr int PORO_PREP_THREADS = 256;
constexpr int PORO_VOX_WARPS = 8;
constexpr int PORO_COUNT_THREADS = 256;
constexpr int PORO_COUNT_BLOCKS = 64;   // blocks per frame of the count pass

__global__ void __launch_bounds__(PORO_PREP_THREADS) k_porosity_prepare(PorosityArgs a) {
    const int f = blockIdx.x, tid = threadIdx.x;
    const mdgpu_unitcell_t uc = a.cells[f];
    PorosityHdr* h = a.hdr + f;
    // a triclinic cell of the current frame, or an empty selection: the value is 0 (:5876-5880, :5896-5899)
    if ((uc.flags & MDGPU_CELL_TRICLINIC) || a.n == 0) { if (tid == 0) *h = PorosityHdr{}; return; }
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    const float* y = x + a.frames.axis_stride; const float* z = y + a.frames.axis_stride;
    float4* p = a.xyzr + (size_t)f * a.n;
    for (uint32_t k = tid; k < a.n; k += blockDim.x) { const int at = a.idx[k]; p[k] = make_float4(x[at], y[at], z[at], a.radius[at]); }
    __syncthreads();
    __shared__ float s_com[3];
    if (tid == 0) { float com[3]; com_compute_vec4(p, a.n, uc, com); s_com[0] = com[0]; s_com[1] = com[1]; s_com[2] = com[2]; }
    __syncthreads();
    const bool ortho = (uc.flags & MDGPU_CELL_ORTHO) != 0;
    const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
    float lo[3] = { FLT_MAX, FLT_MAX, FLT_MAX }, hi[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
    for (uint32_t k = tid; k < a.n; k += blockDim.x) {
        float4 v = p[k];
        if (ortho) { v.x = deperiodize1(v.x, s_com[0], ext[0]); v.y = deperiodize1(v.y, s_com[1], ext[1]); v.z = deperiodize1(v.z, s_com[2], ext[2]); p[k] = v; }
        lo[0] = fminf(lo[0], __fsub_rn(v.x, v.w)); lo[1] = fminf(lo[1], __fsub_rn(v.y, v.w)); lo[2] = fminf(lo[2], __fsub_rn(v.z, v.w));   // md_util_aabb_compute_vec4
        hi[0] = fmaxf(hi[0], __fadd_rn(v.x, v.w)); hi[1] = fmaxf(hi[1], __fadd_rn(v.y, v.w)); hi[2] = fmaxf(hi[2], __fadd_rn(v.z, v.w));
    }
    __shared__ float s_red[6][PORO_PREP_THREADS / 32];
    for (int c = 0; c < 3; ++c) for (int o = 16; o > 0; o >>= 1) { lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o)); hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o)); }
    if ((tid & 31) == 0) for (int c = 0; c < 3; ++c) { s_red[c][tid >> 5] = lo[c]; s_red[3 + c][tid >> 5] = hi[c]; }
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) for (int c = 0; c < 3; ++c) { lo[c] = fminf(lo[c], s_red[c][w]); hi[c] = fmaxf(hi[c], s_red[3 + c][w]); }
    PorosityHdr r{};
    float e[3];
    for (int c = 0; c < 3; ++c) e[c] = fmaxf(__fsub_rn(hi[c], lo[c]), 1.0f);   // vec3_max(bmax - bmin, 1)
    const float max_ext = fmaxf(e[0], fmaxf(e[1], e[2]));
    const float t = __fdiv_rn(max_ext, 512.0f);                                  // a power-of-two scaling: the longest axis gets exactly 512 voxels
    for (int c = 0; c < 3; ++c) {
        r.bmin[c] = lo[c];
        r.dim[c] = max(1, __float2int_rz(__fdiv_rn(e[c], t)));
        r.d[c] = __fdiv_rn(e[c], (float)r.dim[c]);
    }
    r.row_words = (uint32_t)(r.dim[0] + 63) >> 6;
    r.valid = 1;
    *h = r;
}

MDG_D int poro_cell(float q, int dim) { return min(dim - 1, max(0, __float2int_rz(floorf(q)))); }

__global__ void __launch_bounds__(PORO_VOX_WARPS * 32) k_porosity_voxelise(PorosityArgs a) {
    const int f = blockIdx.y, lane = threadIdx.x & 31;
    const PorosityHdr h = a.hdr[f];
    if (!h.valid) return;
    const float4* p = a.xyzr + (size_t)f * a.n;
    unsigned long long* grid = a.grid + (size_t)f * PORO_GRID_WORDS;
    for (uint32_t i = blockIdx.x * PORO_VOX_WARPS + (threadIdx.x >> 5); i < a.n; i += gridDim.x * PORO_VOX_WARPS) {
        const float4 v = p[i];
        const float r = v.w, r2 = __fmul_rn(r, r);
        // (int)floorf(((p - r) - bmin) / d) and (int)floorf(((p + r) - bmin) / d), clamped to the grid
        const int x0 = poro_cell(__fdiv_rn(__fsub_rn(__fsub_rn(v.x, r), h.bmin[0]), h.d[0]), h.dim[0]), x1 = poro_cell(__fdiv_rn(__fsub_rn(__fadd_rn(v.x, r), h.bmin[0]), h.d[0]), h.dim[0]);
        const int y0 = poro_cell(__fdiv_rn(__fsub_rn(__fsub_rn(v.y, r), h.bmin[1]), h.d[1]), h.dim[1]), y1 = poro_cell(__fdiv_rn(__fsub_rn(__fadd_rn(v.y, r), h.bmin[1]), h.d[1]), h.dim[1]);
        const int z0 = poro_cell(__fdiv_rn(__fsub_rn(__fsub_rn(v.z, r), h.bmin[2]), h.d[2]), h.dim[2]), z1 = poro_cell(__fdiv_rn(__fsub_rn(__fadd_rn(v.z, r), h.bmin[2]), h.d[2]), h.dim[2]);
        const int ny = y1 - y0 + 1, nrows = ny * (z1 - z0 + 1);
        for (int row = lane; row < nrows; row += 32) {
            const int iy = y0 + row % ny, iz = z0 + row / ny;
            const float dzv = __fsub_rn(__fadd_rn(h.bmin[2], __fmul_rn(__fadd_rn((float)iz, 0.5f), h.d[2])), v.z);
            const float dyv = __fsub_rn(__fadd_rn(h.bmin[1], __fmul_rn(__fadd_rn((float)iy, 0.5f), h.d[1])), v.y);
            const float yz = __fmaf_rn(dyv, dyv, __fmul_rn(dzv, dzv));
            unsigned long long* row_words = grid + ((size_t)iz * h.dim[1] + iy) * h.row_words;
            for (int w = x0 >> 6; w <= (x1 >> 6); ++w) {
                const int b0 = max(x0, w << 6), b1 = min(x1, (w << 6) + 63);
                unsigned long long m = 0ull;
                for (int ix = b0; ix <= b1; ++ix) {
                    const float dxv = __fsub_rn(__fadd_rn(h.bmin[0], __fmul_rn(__fadd_rn((float)ix, 0.5f), h.d[0])), v.x);
                    if (__fmaf_rn(dxv, dxv, yz) <= r2) m |= 1ull << (ix & 63);
                }
                if (m) atomicOr(row_words + w, m);
            }
        }
    }
}

__global__ void __launch_bounds__(PORO_COUNT_THREADS) k_porosity_count(PorosityArgs a) {
    const int f = blockIdx.y, tid = threadIdx.x;
    const PorosityHdr h = a.hdr[f];
    if (!h.valid) return;
    const size_t words = (size_t)h.row_words * h.dim[1] * h.dim[2];
    unsigned long long* grid = a.grid + (size_t)f * PORO_GRID_WORDS;
    unsigned long long c = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + tid; i < words; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned long long w = grid[i];
        if (w) { c += (unsigned long long)__popcll(w); grid[i] = 0ull; }
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    __shared__ unsigned long long s_sum[PORO_COUNT_THREADS / 32];
    if ((tid & 31) == 0) s_sum[tid >> 5] = c;
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) c += s_sum[w];
    if (c) atomicAdd(a.count + f, c);
}

__global__ void k_porosity_finalize(PorosityArgs a, int nf) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nf) return;
    const PorosityHdr h = a.hdr[f];
    const unsigned long long set = a.count[f];
    a.count[f] = 0ull;
    const unsigned long long N = h.valid ? (unsigned long long)h.dim[0] * (unsigned long long)h.dim[1] * (unsigned long long)h.dim[2] : 0ull;
    const size_t g = (size_t)a.frame0 + f;
    a.frame_set[g] = set; a.frame_n[g] = N;
    a.out[g] = set ? (float)(((double)N - (double)set) / (double)N) : 0.0f;   // no occupied voxel: 0, as the reference reports
}

void launch_porosity(const PorosityArgs& a, int nf, cudaStream_t s) {
    if (nf <= 0) return;
    k_porosity_prepare<<<nf, PORO_PREP_THREADS, 0, s>>>(a);
    note_launch("k_porosity_prepare", s);
    if (a.n) {
        const unsigned gx = (a.n + PORO_VOX_WARPS - 1) / PORO_VOX_WARPS < 4096u ? (a.n + PORO_VOX_WARPS - 1) / PORO_VOX_WARPS : 4096u;
        k_porosity_voxelise<<<dim3(gx, (unsigned)nf), PORO_VOX_WARPS * 32, 0, s>>>(a);
        note_launch("k_porosity_voxelise", s);
        k_porosity_count<<<dim3(PORO_COUNT_BLOCKS, (unsigned)nf), PORO_COUNT_THREADS, 0, s>>>(a);
        note_launch("k_porosity_count", s);
    }
    k_porosity_finalize<<<(nf + 63) / 64, 64, 0, s>>>(a, nf);
    note_launch("k_porosity_finalize", s);
}

}  // namespace mdg
