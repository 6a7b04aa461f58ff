// dssp.cu — secondary structure of every backbone segment per frame: md_util_backbone_secondary_structure_infer -> dssp() (md_util.c:2047-2550).
//
// Three kernels per batch:
//   k_ss_gather   one thread per (frame, segment): N, CA, C, O and the given or estimated H (estimate_HN / estimate_HN_term :1974-1989), and the
//                 CA's fractional coordinates and cell in the candidate walk's grid (md_spatial_acc_init over the CA positions, cell extent 9 A).
//   k_ss_hbonds   one thread per (frame, donor): the acceptors in ascending order, 128 at a time through shared memory; a pair is evaluated when the
//                 reference's internal pair walk reports it (md_spatial_acc_for_each_internal_pair_within_cutoff(.., 9.0) :2150) and the two
//                 residues are not neighbours of one range. Keeps the two lowest energies <= -0.5 with strict `<` (calc_hbond_energy :1910-1972).
//   k_ss_assign   one CTA per frame: turns, helices and bends per range (:2155-2227); bridges (:2248-2316) from the <= 2S recorded bonds, each
//                 one a sheet candidate as the reference requires; ladders (:2390-2453) grown from every bridge; priority (:2523-2547).
//
// The candidate walk visits a home cell's own pairs and its forward neighbours. When every periodic axis has at least 2n + 1 cells (n the
// neighbour reach), each pair of cells is joined by exactly one offset, so whether the walk reports a pair, and which of the two residues is the
// home point that carries the periodic shift, follows from the two cells alone: ss_candidate restates that. Grids with fewer cells on a
// periodic axis can report a pair more than once; such frames fail with MDGPU_ERR_UNSUPPORTED.
//
// Ladders: the reference grows a ladder from a seed bridge by exact-key lookup of the next bridge at either end, whatever `used` says, until
// neither end grows. The ladder is therefore the maximal run of same-type, same-chain-pair bridges through the seed, whichever bridge of the run
// seeds it; marking the run of every bridge gives the reference's sheet marks in any order.
#include "common.cuh"
#include "kernels.h"
#include "cellmath.cuh"

namespace mdg {

constexpr uint32_t SSF_TURN = 1, SSF_BEND = 2, SSF_H310 = 4, SSF_HALPHA = 8, SSF_HPI = 16, SSF_SHEET = 32, SSF_BRIDGE = 64;   // flags of :1997-2006
enum : uint32_t { SS_COIL = 1, SS_TURN = 2, SS_BEND = 3, SS_H310 = 4, SS_HALPHA = 5, SS_HPI = 6, SS_SHEET = 7, SS_BRIDGE = 8 };   // md_secondary_structure_t

// vec4 arithmetic with w = 0 (core/md_vec_math.h): dot = (x + y) + (z + w), normalize multiplies by 1 / sqrtf(mag2) above 1e-5
MDG_D float ss_dot(float3 a, float3 b) { return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fadd_rn(__fmul_rn(a.z, b.z), 0.0f)); }
MDG_D float3 ss_sub(float3 a, float3 b) { return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)); }
MDG_D float3 ss_add(float3 a, float3 b) { return make_float3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z)); }
MDG_D float3 ss_scale(float3 a, float s) { return make_float3(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s)); }
MDG_D float ss_dist2(float3 a, float3 b) { const float3 d = ss_sub(a, b); return ss_dot(d, d); }
MDG_D float3 ss_normalize(float3 v) {
    const float m2 = ss_dot(v, v);
    return m2 > 1.0e-5f ? ss_scale(v, __fdiv_rn(1.0f, __fsqrt_rn(m2))) : v;
}
MDG_D float3 ss_estimate_hn(float3 N, float3 CA, float3 Cp) {   // estimate_HN :1974-1979
    const float3 U = ss_normalize(ss_sub(N, CA)), V = ss_normalize(ss_sub(N, Cp));
    return ss_add(N, ss_scale(ss_normalize(ss_add(U, V)), 1.01f));
}
MDG_D float3 ld3(const float* p) { return make_float3(p[0], p[1], p[2]); }

// the energy of donor (N, H) and acceptor (C, O), or 0 when above -0.5; vec4_rsqrt is 1 / sqrt here (the reference's rsqrtps + Newton step
// depends on the host CPU)
MDG_D float ss_energy(float3 N, float3 H, float3 C, float3 O) {
    const float d0 = ss_dist2(N, O), d1 = ss_dist2(H, C), d2 = ss_dist2(N, C), d3 = ss_dist2(H, O);
    float e;
    if (d0 < 0.25f || d1 < 0.25f || d2 < 0.25f || d3 < 0.25f) e = -9.9f;
    else {
        const float r0 = __fdiv_rn(1.0f, __fsqrt_rn(d0)), r1 = __fdiv_rn(1.0f, __fsqrt_rn(d1)), r2 = __fdiv_rn(1.0f, __fsqrt_rn(d2)), r3 = __fdiv_rn(1.0f, __fsqrt_rn(d3));
        e = __fmul_rn(27.888f, __fadd_rn(__fadd_rn(r0, r1), __fadd_rn(-r2, -r3)));
    }
    if (e > -0.5f) return 0.0f;
    return e > -9.9f ? e : -9.9f;
}

MDG_D uint32_t pack_cell(int x, int y, int z) { return (uint32_t)x | ((uint32_t)y << 10) | ((uint32_t)z << 20); }
MDG_D int cell_coord(uint32_t c, int k) { return (int)((c >> (10 * k)) & 1023u); }

// Whether the internal pair walk reports the pair of CA positions with fractional coordinates si / sj in cells ci / cj (see the file comment).
template <bool TRI>
MDG_D bool ss_candidate(const FrameGeom& g, float3 si, uint32_t ci, float3 sj, uint32_t cj) {
    float dx, dy, dz;
    if (ci == cj) { dx = __fsub_rn(si.x, sj.x); dy = __fsub_rn(si.y, sj.y); dz = __fsub_rn(si.z, sj.z); }
    else {
        int off[3]; float sh[3];
        for (int k = 0; k < 3; ++k) {
            const int o = cell_coord(cj, k) - cell_coord(ci, k), n = g.ncell[k], cd = g.cdim[k];
            const bool periodic = TRI || (g.flags & (MDGPU_CELL_PBC_X << k));
            if (o >= -n && o <= n) { off[k] = o; sh[k] = 0.0f; }
            else if (periodic && o - cd >= -n && o - cd <= n) { off[k] = o - cd; sh[k] = 1.0f; }    // ci + off < 0: lower wrap, the home point moves +1
            else if (periodic && o + cd >= -n && o + cd <= n) { off[k] = o + cd; sh[k] = -1.0f; }   // upper wrap
            else return false;
        }
        const bool fwd = off[2] > 0 || (off[2] == 0 && (off[1] > 0 || (off[1] == 0 && off[0] > 0)));
        if (fwd) { dx = __fsub_rn(__fadd_rn(si.x, sh[0]), sj.x); dy = __fsub_rn(__fadd_rn(si.y, sh[1]), sj.y); dz = __fsub_rn(__fadd_rn(si.z, sh[2]), sj.z); }
        else     { dx = __fsub_rn(__fadd_rn(sj.x, -sh[0]), si.x); dy = __fsub_rn(__fadd_rn(sj.y, -sh[1]), si.y); dz = __fsub_rn(__fadd_rn(sj.z, -sh[2]), si.z); }
    }
    return pair_d2<TRI>(dx, dy, dz, g) <= g.r2;
}

// ---------------------------------------------------------------------------------------------------------------------------------- gather
__global__ void k_ss_gather(SsArgs a) {
    const int f = blockIdx.y; const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const FrameGeom& g = a.geom[f];
    if (i == 0 && (g.valid <= 0 || !g.sym_ok)) atomicExch(a.err, (int)MDGPU_ERR_UNSUPPORTED);
    if (i >= a.S) return;
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride; const float* y = x + a.frames.axis_stride; const float* z = y + a.frames.axis_stride;
    const int32_t* q = a.atoms + 5 * (size_t)i;
    auto P = [&](int32_t at) { return make_float3(x[at], y[at], z[at]); };
    const float3 N = P(q[0]), CA = P(q[1]), C = P(q[2]), O = P(q[3]);
    float3 H;
    if (q[4] >= 0) H = P(q[4]);
    else if (i > a.seg[3 * i + 1]) H = ss_estimate_hn(N, CA, P(a.atoms[5 * (size_t)(i - 1) + 2]));
    else H = ss_estimate_hn(N, CA, ss_add(N, ss_sub(CA, C)));   // estimate_HN_term: C_prev = N + (CA - C)
    float s[3]; const float r[3] = { CA.x, CA.y, CA.z };
    cart_to_fract(s, r, g);
    int cc[3];
    for (int k = 0; k < 3; ++k) {
        if (g.flags & (MDGPU_CELL_PBC_X << k)) s[k] = __fsub_rn(s[k], floorf(s[k]));
        const int ic = (int)floorf(__fmul_rn(s[k], (float)g.cdim[k]));
        cc[k] = max(0, min(ic, g.cdim[k] - 1));
    }
    float* o = a.res + ((size_t)f * a.S + i) * SS_RES_FLOATS;
    const float v[SS_RES_FLOATS] = { N.x, N.y, N.z, CA.x, CA.y, CA.z, C.x, C.y, C.z, O.x, O.y, O.z, H.x, H.y, H.z, s[0], s[1], s[2],
                                     __uint_as_float(pack_cell(cc[0], cc[1], cc[2])), 0.0f };
    for (int k = 0; k < (int)SS_RES_FLOATS; ++k) o[k] = v[k];
}

// ---------------------------------------------------------------------------------------------------------------------------------- H bonds
constexpr int SS_TILE = 128;

template <bool TRI>
__global__ void __launch_bounds__(SS_TILE) k_ss_hbonds(SsArgs a) {
    const int f = blockIdx.y; const uint32_t d = blockIdx.x * SS_TILE + threadIdx.x;
    __shared__ FrameGeom g;
    __shared__ float t_c[SS_TILE][3], t_o[SS_TILE][3], t_s[SS_TILE][3];
    __shared__ uint32_t t_cell[SS_TILE], t_rid[SS_TILE];
    if (threadIdx.x == 0) g = a.geom[f];
    const float* res = a.res + (size_t)f * a.S * SS_RES_FLOATS;
    const bool live = d < a.S;
    float3 N = make_float3(0, 0, 0), H = N, s = N; uint32_t cell = 0, rid = 0;
    if (live) {
        const float* p = res + (size_t)d * SS_RES_FLOATS;
        N = ld3(p); H = ld3(p + 12); s = ld3(p + 15); cell = __float_as_uint(p[18]); rid = a.seg[3 * d];
    }
    uint32_t i0 = 0, i1 = 0; float e0 = 0.0f, e1 = 0.0f;   // the reference starts from zeroed records (:2118)
    for (uint32_t base = 0; base < a.S; base += SS_TILE) {
        __syncthreads();
        const uint32_t j = base + threadIdx.x;
        if (j < a.S) {
            const float* p = res + (size_t)j * SS_RES_FLOATS;
            for (int k = 0; k < 3; ++k) { t_c[threadIdx.x][k] = p[6 + k]; t_o[threadIdx.x][k] = p[9 + k]; t_s[threadIdx.x][k] = p[15 + k]; }
            t_cell[threadIdx.x] = __float_as_uint(p[18]); t_rid[threadIdx.x] = a.seg[3 * j];
        }
        __syncthreads();
        if (!live) continue;
        const uint32_t n = min((uint32_t)SS_TILE, a.S - base);
        for (uint32_t t = 0; t < n; ++t) {
            const uint32_t acc = base + t;
            if (acc == d) continue;
            if (t_rid[t] == rid && (acc + 1 == d || d + 1 == acc)) continue;   // same range, |i - j| <= 1 (:2033)
            const float3 sa = make_float3(t_s[t][0], t_s[t][1], t_s[t][2]);
            const bool cand = d < acc ? ss_candidate<TRI>(g, s, cell, sa, t_cell[t]) : ss_candidate<TRI>(g, sa, t_cell[t], s, cell);
            if (!cand) continue;
            const float e = ss_energy(N, H, make_float3(t_c[t][0], t_c[t][1], t_c[t][2]), make_float3(t_o[t][0], t_o[t][1], t_o[t][2]));
            if (e == 0.0f) continue;
            if (e < e0) { i1 = i0; e1 = e0; i0 = acc; e0 = e; }
            else if (e < e1) { i1 = acc; e1 = e; }
        }
    }
    if (live) a.hb[(size_t)f * a.S + d] = make_float4(__uint_as_float(i0), e0, __uint_as_float(i1), e1);
}

// ---------------------------------------------------------------------------------------------------------------------------------- assign
struct SsFrame {
    const float4* hb; const float* res; const uint32_t* seg; uint32_t S;
    MDG_D bool bond(uint32_t acceptor, uint32_t donor) const {   // dssp_test_bond :1991-1995
        const float4 h = hb[donor];
        return (__float_as_uint(h.x) == acceptor && h.y < -0.5f) || (__float_as_uint(h.z) == acceptor && h.w < -0.5f);
    }
    MDG_D bool same(uint32_t a, uint32_t b) const { return seg[3 * a] == seg[3 * b]; }
    // 0: not a bridge; 1: antiparallel; 2: parallel (:2250-2290). The pair must be a sheet candidate: reported by the walk and not within two
    // residues of one range (:2039).
    template <bool TRI>
    MDG_D uint32_t bridge(const FrameGeom& g, uint32_t i, uint32_t j) const {
        if (i >= j || j >= S) return 0;
        if (same(i, j) && j - i <= 2) return 0;
        const float* pi = res + (size_t)i * SS_RES_FLOATS; const float* pj = res + (size_t)j * SS_RES_FLOATS;
        if (!ss_candidate<TRI>(g, ld3(pi + 15), __float_as_uint(pi[18]), ld3(pj + 15), __float_as_uint(pj[18]))) return 0;
        const bool im = i > 0 && same(i - 1, i), ip = i + 1 < S && same(i + 1, i), jm = j > 0 && same(j - 1, j), jp = j + 1 < S && same(j + 1, j);
        if (bond(i, j) && bond(j, i)) return 1;
        if (im && ip && jm && jp && bond(i - 1, j + 1) && bond(j - 1, i + 1)) return 1;
        if (im && ip && bond(i - 1, j) && bond(j, i + 1)) return 2;
        if (jm && jp && bond(j - 1, i) && bond(i, j + 1)) return 2;
        return 0;
    }
};

template <bool TRI>
__global__ void __launch_bounds__(256) k_ss_assign(SsArgs a) {
    const int f = blockIdx.x; const uint32_t S = a.S;
    __shared__ FrameGeom g;
    if (threadIdx.x == 0) g = a.geom[f];
    const SsFrame fr{ a.hb + (size_t)f * S, a.res + (size_t)f * S * SS_RES_FLOATS, a.seg, S };
    uint32_t* tb = a.bits + (size_t)f * 2 * S; uint32_t* fl = tb + S;
    // turn bits 1 / 2 / 4 (n = 3 / 4 / 5) and the bend bit 8 of each residue
    for (uint32_t i = threadIdx.x; i < S; i += blockDim.x) {
        const uint32_t beg = a.seg[3 * i + 1], end = a.seg[3 * i + 2];
        uint32_t t = 0;
        if (i + 3 < end && fr.bond(i, i + 3)) t |= 1;
        if (i + 4 < end && fr.bond(i, i + 4)) t |= 2;
        if (i + 5 < end && fr.bond(i, i + 5)) t |= 4;
        if (i >= beg + 2 && i + 2 < end) {   // vec4_angle(CA(i-2) - CA(i), CA(i+2) - CA(i)) < 70 degrees
            const float3 c = ld3(fr.res + (size_t)i * SS_RES_FLOATS + 3);
            const float3 v1 = ss_sub(ld3(fr.res + (size_t)(i - 2) * SS_RES_FLOATS + 3), c), v2 = ss_sub(ld3(fr.res + (size_t)(i + 2) * SS_RES_FLOATS + 3), c);
            const float3 w = make_float3(__fsub_rn(__fmul_rn(v1.y, v2.z), __fmul_rn(v1.z, v2.y)), __fsub_rn(__fmul_rn(v1.z, v2.x), __fmul_rn(v1.x, v2.z)),
                                         __fsub_rn(__fmul_rn(v1.x, v2.y), __fmul_rn(v1.y, v2.x)));
            const double angle = atan2f(__fsqrt_rn(ss_dot(w, w)), ss_dot(v1, v2));
            if (angle < 70.0 * (3.14159265358979323846 / 180.0)) t |= 8;
        }
        tb[i] = t;
    }
    __syncthreads();
    // helices and turns: residue r takes the marks of the turn pairs (i, i + 1) of its range with i + 1 <= r <= i + n; bends of i - 2 .. i + 2
    for (uint32_t r = threadIdx.x; r < S; r += blockDim.x) {
        const uint32_t beg = a.seg[3 * r + 1], end = a.seg[3 * r + 2];
        uint32_t m = 0;
        for (uint32_t i = (r >= beg + 5 ? r - 5 : beg); i < r; ++i) {
            const uint32_t x = tb[i] & 7u, y = tb[i + 1] & 7u;
            if ((x & 1) && (y & 1) && r <= i + 3) m |= SSF_H310;
            if ((x & 2) && (y & 2) && r <= i + 4) m |= SSF_HALPHA;
            if ((x & 4) && (y & 4) && r <= i + 5) m |= SSF_HPI;
            if (x && r <= i + ((x & 4) ? 5u : (x & 2) ? 4u : 3u)) m |= SSF_TURN;
        }
        for (uint32_t i = (r >= beg + 2 ? r - 2 : beg); i <= r + 2 && i < end; ++i) if (tb[i] & 8u) m |= SSF_BEND;
        fl[r] = m;
    }
    __syncthreads();
    // bridges: every bridge needs one of the bonds (i -> j), (i - 1 -> j + 1), (i - 1 -> j), (i -> j + 1) in some orientation, so the pairs
    // {a, d}, {a + 1, d - 1}, {a + 1, d}, {a, d - 1} of the recorded bonds (acceptor a, donor d) hold them all. Each bridge marks the ladder run
    // through it (see the file comment); a bridge met more than once marks the same run again.
    for (uint32_t w = threadIdx.x; w < 2 * S; w += blockDim.x) {
        const uint32_t d = w >> 1; const float4 h = fr.hb[d];
        const float e = (w & 1) ? h.w : h.y; const uint32_t acc = __float_as_uint((w & 1) ? h.z : h.x);
        if (!(e < -0.5f)) continue;
        const uint32_t ca[4] = { acc, acc + 1, acc + 1, acc }, cd[4] = { d, d - 1, d, d - 1 };
        for (int k = 0; k < 4; ++k) {
            const uint32_t i = min(ca[k], cd[k]), j = max(ca[k], cd[k]);
            const uint32_t type = fr.bridge<TRI>(g, i, j);
            if (!type) continue;
            atomicOr(&fl[i], SSF_BRIDGE); atomicOr(&fl[j], SSF_BRIDGE);
            const bool par = type == 2; const uint32_t rp = min(a.seg[3 * i], a.seg[3 * j]), rq = max(a.seg[3 * i], a.seg[3 * j]);
            auto found = [&](uint32_t bi, uint32_t bj) {   // the exact key (i, j, type, chain pair) of the reference's maps
                if (fr.bridge<TRI>(g, bi, bj) != type) return false;
                return min(a.seg[3 * bi], a.seg[3 * bj]) == rp && max(a.seg[3 * bi], a.seg[3 * bj]) == rq;
            };
            uint32_t i_min = i, i_max = i, j_min = j, j_max = j;
            for (bool grew = true; grew; ) {
                grew = false;
                const uint32_t n1i = i_max + 1, n1j = par ? j_max + 1 : j_min - 1, n2i = i_min - 1, n2j = par ? j_min - 1 : j_max + 1;
                uint32_t bi, bj;
                if (found(n1i, n1j)) { bi = n1i; bj = n1j; grew = true; }
                else if (found(n2i, n2j)) { bi = n2i; bj = n2j; grew = true; }
                if (grew) { i_min = min(i_min, bi); i_max = max(i_max, bi); j_min = min(j_min, bj); j_max = max(j_max, bj); }
            }
            if (i_max - i_min + 1 >= 3 || j_max - j_min + 1 >= 3) {
                for (uint32_t r = i_min; r <= i_max; ++r) atomicOr(&fl[r], SSF_SHEET);
                for (uint32_t r = j_min; r <= j_max; ++r) atomicOr(&fl[r], SSF_SHEET);
            }
        }
    }
    __syncthreads();
    float* out = a.out + (size_t)(a.frame0 + f) * S;
    for (uint32_t i = threadIdx.x; i < S; i += blockDim.x) {   // priority: HELIX (PI > 310 > ALPHA) > SHEET > BRIDGE > TURN > BEND > COIL
        const uint32_t m = fl[i];
        const uint32_t c = (m & SSF_HPI) ? SS_HPI : (m & SSF_HALPHA) ? SS_HALPHA : (m & SSF_H310) ? SS_H310 : (m & SSF_SHEET) ? SS_SHEET
                         : (m & SSF_BRIDGE) ? SS_BRIDGE : (m & SSF_TURN) ? SS_TURN : (m & SSF_BEND) ? SS_BEND : SS_COIL;
        out[i] = (float)c;
    }
}

void launch_secondary_structure(const SsArgs& a, int B, bool tri, cudaStream_t s) {
    if (!B || !a.S) return;
    const dim3 grid((a.S + SS_TILE - 1) / SS_TILE, B);
    k_ss_gather<<<grid, SS_TILE, 0, s>>>(a);
    note_launch("k_ss_gather", s);
    if (tri) k_ss_hbonds<true><<<grid, SS_TILE, 0, s>>>(a);
    else     k_ss_hbonds<false><<<grid, SS_TILE, 0, s>>>(a);
    note_launch("k_ss_hbonds", s);
    if (tri) k_ss_assign<true><<<B, 256, 0, s>>>(a);
    else     k_ss_assign<false><<<B, 256, 0, s>>>(a);
    note_launch("k_ss_assign", s);
}

}  // namespace mdg
