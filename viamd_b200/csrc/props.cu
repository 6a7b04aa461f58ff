// props.cu — K5 (density_x/_y/_z streaming histogram) and K6 (distance / angle / dihedral, batched over frames).
//
// K5 replaces _internal_density (reference md_script_functions.inl:4825-4947): deperiodise about the centre of the
// INITIAL frame's cell, bin = clamp((int)(fc*1024)), bins[bin] += mass. The reference sums masses in float in atom order;
// here masses are accumulated exactly as 64-bit fixed point (unit 2^-24 Da, exact for every float mass >= 1 Da), which is
// order independent and therefore deterministic; the float result agrees with the reference to its own rounding drift.
// K6 replaces _distance / _angle / _dihedral for single-atom arguments (:3851-3890, :4099-4114, :4171-4196).
#include "common.cuh"
#include "kernels.h"
#include "pbcmath.cuh"

namespace mdg {

// Per-CTA histogram in two 32-bit limbs: a 64-bit shared atomicAdd is a CAS loop (64 cyc/warp, more under contention), a 32-bit one is native.
// The low limb takes the low word of the 2^-24 fixed-point mass; the carry out of each individual add (old + lo wraps) goes to the
// high limb together with the high word, which for masses < 256 u happens for mass/256 of the atoms only.
__global__ void __launch_bounds__(256) k_density(DensityArgs a) {
    const int f = blockIdx.y;
    __shared__ uint32_t hist_lo[MDGPU_DIST_BINS], hist_hi[MDGPU_DIST_BINS];
    for (int b = threadIdx.x; b < MDGPU_DIST_BINS; b += blockDim.x) { hist_lo[b] = 0u; hist_hi[b] = 0u; }
    __syncthreads();
    const float* src = a.frames.xyz + (size_t)f * a.frames.frame_stride + (size_t)a.axis * a.frames.axis_stride;
    const int32_t* __restrict__ idx = sel_list(a.idx, a.dyn, f); const uint32_t n = sel_count(a.n, a.dyn, f);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int at = idx[i];
        const float v = deperiodize1(src[at], a.rc, a.re);
        const float fc = __fmul_rn(__fsub_rn(v, a.min_point), a.inv_ext);
        const int b = max(0, min(__float2int_rz(__fmul_rn(fc, (float)MDGPU_DIST_BINS)), MDGPU_DIST_BINS - 1));
        const unsigned long long m = __float2ull_rn(__fmul_rn(a.mass[at], 16777216.0f));
        const uint32_t lo = (uint32_t)m;
        const uint32_t old = atomicAdd(&hist_lo[b], lo);
        const uint32_t hi = (uint32_t)(m >> 32) + ((old + lo) < old ? 1u : 0u);
        if (hi) atomicAdd(&hist_hi[b], hi);
    }
    __syncthreads();
    unsigned long long* out = a.frame_bins + (size_t)f * MDGPU_DIST_BINS;
    for (int b = threadIdx.x; b < MDGPU_DIST_BINS; b += blockDim.x) {
        const unsigned long long v = ((unsigned long long)hist_hi[b] << 32) + hist_lo[b];
        if (v) atomicAdd(&out[b], v);
    }
}

__global__ void k_density_finalize(DensityArgs a) {
    const int f = blockIdx.x, t = threadIdx.x;
    const unsigned long long v = a.frame_bins[(size_t)f * MDGPU_DIST_BINS + t];
    const uint32_t gf = a.frame0 + f;
    if (v) atomicAdd(&a.acc[t], v);
    if (a.keep) a.keep[(size_t)gf * MDGPU_DIST_BINS + t] = v;
    unsigned long long mn = v, mx = v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long m1 = __shfl_xor_sync(0xffffffffu, mn, o), m2 = __shfl_xor_sync(0xffffffffu, mx, o);
        mn = m1 < mn ? m1 : mn; mx = m2 > mx ? m2 : mx;
    }
    __shared__ unsigned long long s_mn[32], s_mx[32];
    if ((t & 31) == 0) { s_mn[t >> 5] = mn; s_mx[t >> 5] = mx; }
    __syncthreads();
    if (t < 32) {
        mn = s_mn[t]; mx = s_mx[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long m1 = __shfl_xor_sync(0xffffffffu, mn, o), m2 = __shfl_xor_sync(0xffffffffu, mx, o);
            mn = m1 < mn ? m1 : mn; mx = m2 > mx ? m2 : mx;
        }
        if (t == 0) { a.frame_min[gf] = mn; a.frame_max[gf] = mx; }
    }
}

void launch_density(const DensityArgs& a, int B, cudaStream_t s) {
    cudaMemsetAsync(a.frame_bins, 0, sizeof(unsigned long long) * (size_t)B * MDGPU_DIST_BINS, s);
    const uint32_t nmax = a.dyn.n ? a.dyn.stride : a.n;
    if (nmax) {
        const uint32_t blocks = min((nmax + 256u * 8u - 1u) / (256u * 8u), 64u);   // ~8 atoms per thread, <=64 CTAs per frame
        dim3 grid(blocks ? blocks : 1u, B);
        k_density<<<grid, 256, 0, s>>>(a);
        note_launch("k_density", s);
    }
    k_density_finalize<<<B, MDGPU_DIST_BINS, 0, s>>>(a);
    note_launch("k_density_finalize", s);
}

// ---------------------------------------------------------------------------------------------------------------
// Centres of mass of atom groups, as coordinate_extract() produces them for an array of bitfields
// (md_script_functions.inl:1496-1507 -> extract_com :857-874): NO periodic treatment, one sequential float pass in ascending atom
// order, sum += (x*w, y*w, z*w, 1*w), then xyz / w (w == 0 -> 1). One thread per (group, frame): the order of the float additions
// is the result.
__global__ void k_group_com(BatchFrames fr, const int32_t* __restrict__ idx, const uint32_t* __restrict__ off, uint32_t n_groups,
                            const float* __restrict__ mass, float* __restrict__ out /* [B][n_groups][3] */) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = blockIdx.y;
    if (g >= n_groups) return;
    const float* x = fr.xyz + (size_t)f * fr.frame_stride; const float* y = x + fr.axis_stride; const float* z = y + fr.axis_stride;
    float sx = 0.f, sy = 0.f, sz = 0.f, sw = 0.f;
    for (uint32_t k = off[g]; k < off[g + 1]; ++k) {
        const int a = idx[k]; const float w = mass[a];
        sx = __fadd_rn(sx, __fmul_rn(x[a], w)); sy = __fadd_rn(sy, __fmul_rn(y[a], w)); sz = __fadd_rn(sz, __fmul_rn(z[a], w));
        sw = __fadd_rn(sw, __fmul_rn(1.0f, w));
    }
    if (sw == 0.0f) sw = 1.0f;
    float* o = out + ((size_t)f * n_groups + g) * 3;
    o[0] = __fdiv_rn(sx, sw); o[1] = __fdiv_rn(sy, sw); o[2] = __fdiv_rn(sz, sw);
}

void launch_group_com(const BatchFrames& fr, const int32_t* d_idx, const uint32_t* d_off, uint32_t n_groups, const float* d_mass, float* d_out, cudaStream_t s) {
    if (!n_groups || !fr.count) return;
    dim3 grid((n_groups + 127u) / 128u, fr.count);
    k_group_com<<<grid, 128, 0, s>>>(fr, d_idx, d_off, n_groups, d_mass, d_out);
    note_launch("k_group_com", s);
}

// ---------------------------------------------------------------------------------------------------------------
// md_mm256_reduce_add_ps (core/md_simd.h:691, :678) over the 8 emulated lanes held by threads 0..7 of the warp
MDG_D float reduce8(float v) {
    v = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, 4));    // (l0+l4, l1+l5, l2+l6, l3+l7)
    const float a = __fadd_rn(v, __shfl_down_sync(0xffffffffu, v, 1));   // lane0: (l0+l4)+(l1+l5), lane2: (l2+l6)+(l3+l7)
    return __fadd_rn(a, __shfl_down_sync(0xffffffffu, a, 2));
}

// Position of one argument of distance/angle/dihedral that is a selection: md_util_com_compute (md_util.c:8163) as the reference's
// AVX2 build evaluates it — threads 0..7 of the warp are the 8 SIMD lanes (element i goes to lane i % 8, sequential per lane), the
// count % 8 tail and the final atan2 step run in double on thread 0. No cell (flags == 0): com() :7139; otherwise the trigonometric
// periodic centre of mass com_pbc :8019 -> _com_pbc_iw :7850. One warp per (argument, frame).
MDG_D void periodic_com_warp(const float* const src[3], const mdgpu_unitcell_t& uc, const int32_t* __restrict__ idx, uint32_t count,
                             const float* __restrict__ mass, float* __restrict__ o, int lane) {
    const uint32_t simd_count = count & ~7u;
    if (uc.flags == 0) {
        float v[4] = { 0.f, 0.f, 0.f, 0.f };
        if (lane < 8) for (uint32_t i = lane; i < simd_count; i += 8) {
            const int a = idx[i]; const float w = mass[a];
            v[0] = __fadd_rn(v[0], __fmul_rn(src[0][a], w)); v[1] = __fadd_rn(v[1], __fmul_rn(src[1][a], w));
            v[2] = __fadd_rn(v[2], __fmul_rn(src[2][a], w)); v[3] = __fadd_rn(v[3], w);
        }
        double acc[4];
        for (int k = 0; k < 4; ++k) acc[k] = (double)reduce8(v[k]);
        if (lane == 0) {
            for (uint32_t i = simd_count; i < count; ++i) {
                const int a = idx[i]; const float w = mass[a];
                acc[0] += (double)__fmul_rn(src[0][a], w); acc[1] += (double)__fmul_rn(src[1][a], w); acc[2] += (double)__fmul_rn(src[2][a], w); acc[3] += (double)w;
            }
            for (int k = 0; k < 3; ++k) o[k] = (float)(acc[k] / acc[3]);
        }
        return;
    }
    float A[3][3], M[3][3], I[3][3]; cell_box(uc, A);
    {   // the double inverse cast to float; M = 2pi * Ai, I = A / 2pi element-wise (com_pbc :8027-8030)
        double Id[3][3]; cell_inverse(uc, Id);
        const float tp = (float)6.283185307179586, itp = (float)(1.0 / 6.283185307179586);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { M[r][c] = __fmul_rn(tp, (float)Id[r][c]); I[r][c] = __fmul_rn(A[r][c], itp); }
    }
    float vs[3] = { 0.f, 0.f, 0.f }, vc[3] = { 0.f, 0.f, 0.f }, vw = 0.f;
    if (lane < 8) for (uint32_t i = lane; i < simd_count; i += 8) {
        const int a = idx[i]; const float w = mass[a];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float p = src[k][a];
            const float t = __fmaf_rn(p, M[k][0], __fmaf_rn(p, M[k][1], __fmul_rn(p, M[k][2])));
            float sn, cs; sincos_cephes(t, SINCOS_DP3_PS256, sn, cs);   // one lane of the 8-lane md_mm256_sincos_ps (core/md_simd.h:1177-1258)
            vs[k] = __fmaf_rn(sn, w, vs[k]); vc[k] = __fmaf_rn(cs, w, vc[k]);
        }
        vw = __fadd_rn(vw, w);
    }
    double acc_s[3], acc_c[3], acc_w = (double)reduce8(vw);
    for (int k = 0; k < 3; ++k) { acc_s[k] = (double)reduce8(vs[k]); acc_c[k] = (double)reduce8(vc[k]); }
    if (lane == 0) {
        for (uint32_t i = simd_count; i < count; ++i) {   // scalar remainder in double (:7988-8003)
            const int a = idx[i]; const double w = (double)mass[a];
            for (int k = 0; k < 3; ++k) {
                const double p = (double)src[k][a];
                const double t = __dadd_rn(__dadd_rn(__dmul_rn(p, (double)M[k][0]), __dmul_rn(p, (double)M[k][1])), __dmul_rn(p, (double)M[k][2]));
                acc_c[k] = __dadd_rn(acc_c[k], __dmul_rn(w, cos(t))); acc_s[k] = __dadd_rn(acc_s[k], __dmul_rn(w, sin(t)));
            }
            acc_w += w;
        }
        const double inv_w = 1.0 / acc_w;
        for (int k = 0; k < 3; ++k) {
            double theta = 3.14159265358979323846;
            const double px = __dmul_rn(acc_c[k], inv_w), py = __dmul_rn(acc_s[k], inv_w);
            if (__dadd_rn(__dmul_rn(px, px), __dmul_rn(py, py)) > 1.0e-8) theta += atan2(-py, -px);
            o[k] = (float)__dadd_rn(__dadd_rn(__dmul_rn(theta, (double)I[k][0]), __dmul_rn(theta, (double)I[k][1])), __dmul_rn(theta, (double)I[k][2]));
        }
    }
}

__global__ void k_arg_com(BatchFrames fr, const mdgpu_unitcell_t* __restrict__ cells, const int32_t* __restrict__ idx_, uint32_t count_,
                          const float* __restrict__ mass, float* __restrict__ out /* [B][4][3] */, int arg, DynSel dyn) {
    const int f = blockIdx.x, lane = threadIdx.x;
    const int32_t* __restrict__ idx = sel_list(idx_, dyn, f); const uint32_t count = sel_count(count_, dyn, f);
    if (count == 0) { if (lane < 3) out[((size_t)f * 4 + arg) * 3 + lane] = 0.0f; return; }   // md_util_com_compute: count == 0 -> (0, 0, 0) (md_util.c:8168)
    const float* x = fr.xyz + (size_t)f * fr.frame_stride;
    const float* src[3] = { x, x + fr.axis_stride, x + 2 * fr.axis_stride };
    periodic_com_warp(src, cells[f], idx, count, mass, out + ((size_t)f * 4 + arg) * 3, lane);
}

void launch_arg_com(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_idx, uint32_t count, const float* d_mass, float* d_out, int arg, cudaStream_t s, DynSel dyn) {
    if (!fr.count || (!count && !dyn.n)) return;   // a coordinate range has no static list: its per-frame list is all there is
    k_arg_com<<<fr.count, 32, 0, s>>>(fr, d_cells, d_idx, count, d_mass, d_out, arg, dyn);
    note_launch("k_arg_com", s);
}

// One warp per (frame, selection of an array argument): md_util_com_compute of that selection, stored as xyzw with w = 1 for k_arg_combine.
__global__ void k_arg_com_parts(BatchFrames fr, const mdgpu_unitcell_t* __restrict__ cells, const int32_t* __restrict__ idx, const uint32_t* __restrict__ off, uint32_t n_parts,
                                const float* __restrict__ mass, float4* __restrict__ parts /* [B][n_parts] */) {
    const int f = blockIdx.x, lane = threadIdx.x; const uint32_t part = blockIdx.y;
    float* o = (float*)(parts + (size_t)f * n_parts + part);
    const uint32_t beg = off[part], count = off[part + 1] - beg;
    if (lane == 0) o[3] = 1.0f;                                                         // vec4_from_vec3(com, 1.0f) :1840
    if (count == 0) { if (lane < 3) o[lane] = 0.0f; return; }                           // md_util_com_compute: count == 0 -> (0, 0, 0) (md_util.c:8168)
    const float* x = fr.xyz + (size_t)f * fr.frame_stride;
    const float* src[3] = { x, x + fr.axis_stride, x + 2 * fr.axis_stride };
    periodic_com_warp(src, cells[f], idx + beg, count, mass, o, lane);
}

void launch_arg_com_parts(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_idx, const uint32_t* d_off, uint32_t n_parts, const float* d_mass, float4* d_parts, cudaStream_t s) {
    if (!fr.count || !n_parts) return;
    k_arg_com_parts<<<dim3(fr.count, n_parts), 32, 0, s>>>(fr, d_cells, d_idx, d_off, n_parts, d_mass, d_parts);
    note_launch("k_arg_com_parts", s);
}

// One subtract / add loop of min_image_ortho (md_util.c:8424-8436) or of min_image_triclinic's zone reduction (:8360-8423): while
// d[i] > half subtract row `step` (components 0..i), then while d[i] <= -half add it, every step rounded as the reference rounds it.
// There is no iteration cap, so every input on which the reference's loop ends gives its result, however many box lengths d[i] spans.
// The reference never ends when a step leaves d[i] unchanged (d[i] infinite, or so large that d[i] - step[i] == d[i]); here the loop stops
// there and returns false, and the caller makes the frame's value NaN. NaN input skips both loops, as in the reference.
MDG_D bool min_image_loop(float* d, const float* step, int i, float half) {
    while (d[i] > half) {
        const float next = __fsub_rn(d[i], step[i]);
        if (next == d[i]) return false;
        for (int j = i; j >= 0; --j) d[j] = __fsub_rn(d[j], step[j]);
    }
    while (d[i] <= -half) {
        const float next = __fadd_rn(d[i], step[i]);
        if (next == d[i]) return false;
        for (int j = i; j >= 0; --j) d[j] = __fadd_rn(d[j], step[j]);
    }
    return true;
}

// distance / angle / dihedral on the argument positions: an atom's coordinates (single index, coordinate_extract_com :1755) or the
// centre of mass k_arg_com left in a.pos
// distance (:3851-3890) / angle (:4099-4114) / dihedral (:4171-4196) of up to four positions in one cell
MDG_D float temporal_value(int op, const float P[4][3], const mdgpu_unitcell_t& uc) {
    const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
    float out = 0.0f;
    if (op == MDGPU_OP_DISTANCE) {
        const float* pa = P[0]; float pb[3] = { P[1][0], P[1][1], P[1][2] };
        if (uc.flags & MDGPU_CELL_ORTHO) for (int k = 0; k < 3; ++k) pb[k] = deperiodize1(pb[k], pa[k], ext[k]);   // md_util_deperiodize_vec4 md_util.c:8971
        const float d[3] = { pa[0] - pb[0], pa[1] - pb[1], pa[2] - pb[2] };
        out = __fsqrt_rn(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    } else if (op == MDGPU_OP_ANGLE) {
        float v0[3] = { P[0][0] - P[1][0], P[0][1] - P[1][1], P[0][2] - P[1][2] }, v1[3] = { P[2][0] - P[1][0], P[2][1] - P[1][1], P[2][2] - P[1][2] };
        normalize3(v0); normalize3(v1);
        out = acosf(v0[0] * v1[0] + v0[1] * v1[1] + v0[2] * v1[2]);
    } else if (op == MDGPU_OP_DIHEDRAL) {
        float dx[3][3];
        for (int k = 0; k < 3; ++k) for (int i = 0; i < 3; ++i) dx[k][i] = P[k + 1][i] - P[k][i];
        if (uc.flags & MDGPU_CELL_ORTHO) {   // min_image_ortho md_util.c:8424-8436
            for (int k = 0; k < 3; ++k) for (int i = 0; i < 3; ++i) {
                if (ext[i] > 0.0f) {
                    float d = dx[k][i];
                    if (!min_image_loop(&d, &ext[i], 0, __fmul_rn(ext[i], 0.5f))) return __int_as_float(0x7fffffff);
                    dx[k][i] = d;
                }
            }
        }
        else if (uc.flags & MDGPU_CELL_TRICLINIC) {   // min_image_triclinic with the half diagonal (md_util.c:8360-8423): zone reduction along c, b, a, then the 27 images
            float box[3][3]; cell_box(uc, box);
            const float half3[3] = { box[0][0] * 0.5f, box[1][1] * 0.5f, box[2][2] * 0.5f };
            for (int k = 0; k < 3; ++k) {
                for (int i = 2; i >= 0; --i)
                    if (half3[i] > 0.0f && !min_image_loop(dx[k], box[i], i, half3[i])) return __int_as_float(0x7fffffff);
                min_image_triclinic(dx[k], box);
            }
        }
        const float* d1 = dx[0]; const float* d2 = dx[1]; const float* d3 = dx[2];   // vec3_dihedral_angle core/md_vec_math.h:558-567
        const float v1[3] = { d1[1] * d2[2] - d1[2] * d2[1], d1[2] * d2[0] - d1[0] * d2[2], d1[0] * d2[1] - d1[1] * d2[0] };
        const float v2[3] = { d2[1] * d3[2] - d2[2] * d3[1], d2[2] * d3[0] - d2[0] * d3[2], d2[0] * d3[1] - d2[1] * d3[0] };
        const float w[3] = { v1[1] * v2[2] - v1[2] * v2[1], v1[2] * v2[0] - v1[0] * v2[2], v1[0] * v2[1] - v1[1] * v2[0] };
        const float wl = __fsqrt_rn(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        const float sdot = v1[0] * v2[0] + v1[1] * v2[1] + v1[2] * v2[2];
        float angle = atan2f(wl, sdot);
        const float dot = d1[0] * v2[0] + d1[1] * v2[1] + d1[2] * v2[2];
        if (dot < 0.0f) angle = -angle;
        out = angle;
    }
    return out;
}

__global__ void k_temporal(TemporalArgs a, int B) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= B) return;
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride; const float* y = x + a.frames.axis_stride; const float* z = y + a.frames.axis_stride;
    const mdgpu_unitcell_t uc = a.cells[f];
    const int nargs = a.op == MDGPU_OP_DISTANCE ? 2 : (a.op == MDGPU_OP_ANGLE ? 3 : 4);
    float P[4][3];
    for (int k = 0; k < nargs; ++k) {
        if (a.com_mask & (1u << k)) { const float* p = a.pos + ((size_t)f * 4 + k) * 3; P[k][0] = p[0]; P[k][1] = p[1]; P[k][2] = p[2]; }
        else { const int at = a.atom[k]; P[k][0] = x[at]; P[k][1] = y[at]; P[k][2] = z[at]; }
    }
    a.out[a.frame0 + f] = temporal_value(a.op, P, uc);
}

// the same expression evaluated `in` n contexts (evaluate_context md_script.c:3418: the integer arguments are relative to each context's
// first atom, remap_index_to_context): ctx_idx[k][c] is argument k's atom in context c; row (frame0 + f) holds the n values
__global__ void k_temporal_ctx(TemporalArgs a, int B) {
    const int f = blockIdx.y;
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_ctx) return;
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride; const float* y = x + a.frames.axis_stride; const float* z = y + a.frames.axis_stride;
    const int nargs = a.op == MDGPU_OP_DISTANCE ? 2 : (a.op == MDGPU_OP_ANGLE ? 3 : 4);
    float P[4][3]; bool defined = true;
    for (int k = 0; k < nargs; ++k) {
        if (a.ctx_pos[k]) { const float4 q = a.ctx_pos[k][(size_t)f * a.n_ctx + c]; P[k][0] = q.x; P[k][1] = q.y; P[k][2] = q.z; continue; }   // selection AND context: its centre of mass (coordinate_extract_com with ctx->mol_ctx, :1812-1823)
        const int at = a.ctx_idx[k][c];
        if (at < 0) { defined = false; break; }   // backbone angles: the end segments of a chain have no phi / psi and stay 0 (md_util.c:2576, :2592)
        P[k][0] = x[at]; P[k][1] = y[at]; P[k][2] = z[at];
    }
    a.out[(size_t)(a.frame0 + f) * a.n_ctx + c] = defined ? temporal_value(a.op, P, a.cells[f]) : 0.0f;
}

// Histogram of a temporal's values over the frames of `mask` — the counting half of VIAMD's compute_histogram_masked (src/main.cpp:172-226):
// values outside [range_min, range_max] are skipped, bin = clamp((int)(((v - min) * inv_range) * num_bins)). counts: [dim or 1][num_bins],
// totals: [dim or 1] samples that landed in a bin.
__global__ void k_temporal_histogram(const float* __restrict__ values, const unsigned long long* __restrict__ mask, uint32_t num_frames, uint32_t dim, float range_min, float range_max,
                                     float inv_range, uint32_t num_bins, int aggregate, uint32_t* __restrict__ counts, uint32_t* __restrict__ totals) {
    const size_t n = (size_t)num_frames * dim;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t f = (uint32_t)(i / dim), c = (uint32_t)(i % dim);
        if (!((mask[f >> 6] >> (f & 63)) & 1ull)) continue;
        const float v = values[i];
        if (v < range_min || range_max < v) continue;
        int b = __float2int_rz(__fmul_rn(__fmul_rn(__fsub_rn(v, range_min), inv_range), (float)num_bins));
        b = max(0, min(b, (int)num_bins - 1));
        const uint32_t row = aggregate ? 0u : c;
        atomicAdd(&counts[(size_t)row * num_bins + (uint32_t)b], 1u);
        atomicAdd(&totals[row], 1u);
    }
}
void launch_temporal_histogram(const float* d_values, const unsigned long long* d_mask, uint32_t num_frames, uint32_t dim, float range_min, float range_max, float inv_range,
                               uint32_t num_bins, int aggregate, uint32_t* d_counts, uint32_t* d_totals, cudaStream_t s) {
    const size_t n = (size_t)num_frames * dim; if (!n) return;
    const size_t want = (n + 255) / 256; const unsigned blocks = (unsigned)(want < 1184 ? want : 1184);
    k_temporal_histogram<<<blocks, 256, 0, s>>>(d_values, d_mask, num_frames, dim, range_min, range_max, inv_range, num_bins, aggregate, d_counts, d_totals);
    note_launch("k_temporal_histogram", s);
}

// com(x) (_com md_script_functions.inl:4726): the position coordinate_extract_com yields for the argument — an atom's coordinates or the
// centre of mass k_arg_com left in a.pos — stored as the frame's 3 values.
__global__ void k_com_rows(TemporalArgs a, int B) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= B) return;
    float* o = a.out + (size_t)(a.frame0 + f) * 3;
    if (a.com_mask & 1u) { const float* p = a.pos + (size_t)f * 4 * 3; o[0] = p[0]; o[1] = p[1]; o[2] = p[2]; }
    else {
        const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride; const int at = a.atom[0];
        o[0] = x[at]; o[1] = x[a.frames.axis_stride + at]; o[2] = x[2 * a.frames.axis_stride + at];
    }
}

// coord_x / coord_y / coord_z(selection) (_coordinate_x/_y/_z md_script_functions.inl:5077-5169): the atoms' coordinates along one axis, row
// (frame0 + f) of a [num_frames][n] temporal
__global__ void k_coord_rows(BatchFrames fr, const int32_t* __restrict__ idx, uint32_t n, int axis, float* __restrict__ out, uint32_t frame0) {
    const int f = blockIdx.y;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    out[(size_t)(frame0 + f) * n + k] = fr.xyz[(size_t)f * fr.frame_stride + (size_t)axis * fr.axis_stride + idx[k]];
}

// One pair of md_util_min_distance / md_util_distance_array (md_util.c:8210-8297): no cell -> vec3_distance; orthorhombic ->
// vec4_periodic_distance (core/md_vec_math.h:1268-1273, vec4_dot sums (x+y)+(z+w)); triclinic -> the 27-image minimum + vec3_length.
MDG_D float pair_distance(float ax, float ay, float az, float bx, float by, float bz, uint32_t flags, const float ext[3], const float box[3][3]) {
    float d[3] = { __fsub_rn(ax, bx), __fsub_rn(ay, by), __fsub_rn(az, bz) };
    if (flags == 0) return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
    if (flags & MDGPU_CELL_ORTHO) {
        for (int k = 0; k < 3; ++k) if (ext[k] != 0.0f) d[k] = __fsub_rn(d[k], __fmul_rn(rintf(__fdiv_rn(d[k], ext[k])), ext[k]));
        return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fadd_rn(__fmul_rn(d[2], d[2]), 0.0f)));
    }
    min_image_triclinic(d, box);
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
}

// Minimum of `best` over the 256 threads of the block (8 warps), stored by thread 0
MDG_D void block_min_store(float best, float* out) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = fminf(best, __shfl_xor_sync(0xffffffffu, best, o));
    __shared__ float s_best[8];
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) { for (int w = 1; w < 8; ++w) best = fminf(best, s_best[w]); *out = best; }
}

// Element i of a position argument in frame f: row i of pos ([B][n][3], the centres of mass of an ARRAY of selections) or atom idx[i]
MDG_D void load_pos(const float* __restrict__ pos, const int32_t* __restrict__ idx, uint32_t i, int f, uint32_t n,
                    const float* x, const float* y, const float* z, float out[3]) {
    if (pos) { const float* q = pos + ((size_t)f * n + i) * 3; out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; }
    else { const int a = idx[i]; out[0] = x[a]; out[1] = y[a]; out[2] = z[a]; }
}

// distance_min / distance_max (both md_util_min_distance, md_util.c:8242-8297): all pairs of two selections, one CTA per frame.
// The minimum of floats is order independent, so the pairs are spread over the threads and reduced.
__global__ void __launch_bounds__(256) k_min_distance(BatchFrames fr, const mdgpu_unitcell_t* __restrict__ cells, const int32_t* __restrict__ ia_, uint32_t na_,
                                                      const int32_t* __restrict__ ib_, uint32_t nb_, float* __restrict__ out, uint32_t frame0, DynSel da, DynSel db) {
    const int f = blockIdx.x;
    const int32_t* __restrict__ ia = sel_list(ia_, da, f); const uint32_t na = sel_count(na_, da, f);
    const int32_t* __restrict__ ib = sel_list(ib_, db, f); const uint32_t nb = sel_count(nb_, db, f);
    const float* x = fr.xyz + (size_t)f * fr.frame_stride; const float* y = x + fr.axis_stride; const float* z = y + fr.axis_stride;
    const mdgpu_unitcell_t uc = cells[f];
    const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
    float box[3][3]; cell_box(uc, box);
    float best = 3.402823466e+38f;
    const unsigned long long npairs = (unsigned long long)na * nb;
    for (unsigned long long p = threadIdx.x; p < npairs; p += blockDim.x) {
        const int a = ia[p / nb], b = ib[p % nb];
        best = fminf(best, pair_distance(x[a], y[a], z[a], x[b], y[b], z[b], uc.flags, ext, box));
    }
    block_min_store(best, out + frame0 + f);
}

// distance_pair(a, b) (_distance_pair md_script_functions.inl:3972 -> md_util_distance_array md_util.c:8210): the na x nb matrix of a frame,
// row (frame0 + f) of a [num_frames][na*nb] temporal; one thread per pair.
// posa / posb (may be null): [B][na][3] / [B][nb][3] centres of mass when the argument was an ARRAY of selections (k_group_com: extract_com, no periodic treatment)
__global__ void __launch_bounds__(256) k_distance_pair(BatchFrames fr, const mdgpu_unitcell_t* __restrict__ cells, const int32_t* __restrict__ ia, uint32_t na,
                                                       const int32_t* __restrict__ ib, uint32_t nb, const float* __restrict__ posa, const float* __restrict__ posb,
                                                       float* __restrict__ out, uint32_t frame0) {
    const int f = blockIdx.y;
    const unsigned long long npairs = (unsigned long long)na * nb, p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    const float* x = fr.xyz + (size_t)f * fr.frame_stride; const float* y = x + fr.axis_stride; const float* z = y + fr.axis_stride;
    const mdgpu_unitcell_t uc = cells[f];
    const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
    float box[3][3]; cell_box(uc, box);
    const uint32_t i = (uint32_t)(p / nb), j = (uint32_t)(p % nb);
    float pa[3], pb[3];
    load_pos(posa, ia, i, f, na, x, y, z, pa); load_pos(posb, ib, j, f, nb, x, y, z, pb);
    out[(size_t)(frame0 + f) * npairs + p] = pair_distance(pa[0], pa[1], pa[2], pb[0], pb[1], pb[2], uc.flags, ext, box);
}

// distance_min / distance_max when an argument was an ARRAY of selections: that argument's positions are the selections' centres of mass
// (coordinate_extract md_script_functions.inl:1503 -> extract_com :857; posa / posb as for k_distance_pair), then md_util_min_distance (md_util.c:8242)
__global__ void __launch_bounds__(256) k_min_distance_pos(BatchFrames fr, const mdgpu_unitcell_t* __restrict__ cells, const int32_t* __restrict__ ia, uint32_t na,
                                                          const int32_t* __restrict__ ib, uint32_t nb, const float* __restrict__ posa, const float* __restrict__ posb,
                                                          float* __restrict__ out, uint32_t frame0) {
    const int f = blockIdx.x;
    const float* x = fr.xyz + (size_t)f * fr.frame_stride; const float* y = x + fr.axis_stride; const float* z = y + fr.axis_stride;
    const mdgpu_unitcell_t uc = cells[f];
    const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
    float box[3][3]; cell_box(uc, box);
    float best = 3.402823466e+38f;
    const unsigned long long npairs = (unsigned long long)na * nb;
    for (unsigned long long p = threadIdx.x; p < npairs; p += blockDim.x) {
        const uint32_t i = (uint32_t)(p / nb), j = (uint32_t)(p % nb);
        float pa[3], pb[3];
        load_pos(posa, ia, i, f, na, x, y, z, pa); load_pos(posb, ib, j, f, nb, x, y, z, pb);
        best = fminf(best, pair_distance(pa[0], pa[1], pa[2], pb[0], pb[1], pb[2], uc.flags, ext, box));
    }
    block_min_store(best, out + frame0 + f);
}

void launch_min_distance_pos(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb,
                             const float* d_posa, const float* d_posb, float* d_out, uint32_t frame0, cudaStream_t s) {
    if (!fr.count) return;
    k_min_distance_pos<<<fr.count, 256, 0, s>>>(fr, d_cells, d_ia, na, d_ib, nb, d_posa, d_posb, d_out, frame0);
    note_launch("k_min_distance_pos", s);
}

// coord_x / _y / _z of an ARRAY of selections: one coordinate per selection, of its centre of mass (coordinate_extract :1503); pos [B][n][3]
__global__ void k_coord_rows_pos(const float* __restrict__ pos, uint32_t n, int axis, float* __restrict__ out, uint32_t frame0) {
    const int f = blockIdx.y;
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    out[(size_t)(frame0 + f) * n + k] = pos[((size_t)f * n + k) * 3 + axis];
}

void launch_coord_rows_pos(const float* d_pos, uint32_t n, int axis, float* d_out, uint32_t frame0, int B, cudaStream_t s) {
    if (!n || B <= 0) return;
    k_coord_rows_pos<<<dim3((n + 255u) / 256u, (unsigned)B), 256, 0, s>>>(d_pos, n, axis, d_out, frame0);
    note_launch("k_coord_rows_pos", s);
}

void launch_min_distance(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb, float* d_out, uint32_t frame0, cudaStream_t s, DynSel da, DynSel db) {
    if (!fr.count) return;
    k_min_distance<<<fr.count, 256, 0, s>>>(fr, d_cells, d_ia, na, d_ib, nb, d_out, frame0, da, db);
    note_launch("k_min_distance", s);
}

void launch_distance_pair(const BatchFrames& fr, const mdgpu_unitcell_t* d_cells, const int32_t* d_ia, uint32_t na, const int32_t* d_ib, uint32_t nb,
                          const float* d_posa, const float* d_posb, float* d_out, uint32_t frame0, cudaStream_t s) {
    const unsigned long long npairs = (unsigned long long)na * nb;
    if (!fr.count || !npairs) return;
    k_distance_pair<<<dim3((unsigned)((npairs + 255) / 256), fr.count), 256, 0, s>>>(fr, d_cells, d_ia, na, d_ib, nb, d_posa, d_posb, d_out, frame0);
    note_launch("k_distance_pair", s);
}

// fold of an integer accumulator into the float mean the property data exposes: (float)((double)count / (double)n), IEEE on the device
__global__ void k_mean_u32(const uint32_t* __restrict__ in, float* __restrict__ out, size_t count, unsigned long long n) {
    const double dn = (double)n;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x)
        out[i] = n ? (float)((double)in[i] / dn) : 0.0f;
}
void launch_mean_u32(const uint32_t* d_in, float* d_out, size_t count, unsigned long long n, cudaStream_t s) {
    k_mean_u32<<<132 * 4, 256, 0, s>>>(d_in, d_out, count, n);
    note_launch("k_mean_u32", s);
}

void launch_coord_rows(const BatchFrames& fr, const int32_t* d_idx, uint32_t n, int axis, float* d_out, uint32_t frame0, cudaStream_t s) {
    if (!n || !fr.count) return;
    k_coord_rows<<<dim3((n + 255u) / 256u, fr.count), 256, 0, s>>>(fr, d_idx, n, axis, d_out, frame0);
    note_launch("k_coord_rows", s);
}

void launch_com_rows(const TemporalArgs& a, int B, cudaStream_t s) {
    k_com_rows<<<(B + 63) / 64, 64, 0, s>>>(a, B);
    note_launch("k_com_rows", s);
}

void launch_temporal_ctx(const TemporalArgs& a, int B, cudaStream_t s) {
    if (!a.n_ctx || B <= 0) return;
    k_temporal_ctx<<<dim3((a.n_ctx + 63u) / 64u, (unsigned)B), 64, 0, s>>>(a, B);
    note_launch("k_temporal_ctx", s);
}

void launch_temporal(const TemporalArgs& a, int B, cudaStream_t s) {
    k_temporal<<<(B + 63) / 64, 64, 0, s>>>(a, B);
    note_launch("k_temporal", s);
}

}  // namespace mdg
