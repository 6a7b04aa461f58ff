// cellmath.cuh — per-point arithmetic of the cell lists shared by cells.cu (static index lists), within.cu (per-frame lists) and rdf.cu:
// point binning, the neighbour-cell walk of the pair query and the pair metric.
#pragma once
#include "common.cuh"

namespace mdg {

// ---------------------------------------------------------------------------------------------------------------
// Point binning. vec4_linear_combine_3(r - origin, I) (core/md_vec_math.h:1323): ((I0*a.x) + (I1*a.y)) + (I2*a.z).
// ---------------------------------------------------------------------------------------------------------------
MDG_D void cart_to_fract(float s[3], const float r[3], const FrameGeom& g) {
    const float ax = __fsub_rn(r[0], g.origin[0]), ay = __fsub_rn(r[1], g.origin[1]), az = __fsub_rn(r[2], g.origin[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float v = __fmul_rn(g.I[0][k], ax);
        v = __fadd_rn(v, __fmul_rn(g.I[1][k], ay));
        v = __fadd_rn(v, __fmul_rn(g.I[2][k], az));
        s[k] = v;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The neighbour walk of the pair query (core/md_spatial_acc.c:1719-1755). A home cell is the unclamped cell coordinate of a reference
// point; its neighbours are the (2n+1)^3 offsets of ncell, wrapped once into the grid, with the reference point shifted by the periodic
// image of the wrap. The image is coded (sx + 1) | (sy + 1) << 2 | (sz + 1) << 4; IMAGE_NONE is no shift.
// ---------------------------------------------------------------------------------------------------------------
constexpr uint32_t IMAGE_NONE = 0x15u;

struct CellWalk { int cd0, cd1, cd2, n0, n1, n2; uint32_t flags; };   // the grid as the walk reads it, hoisted out of FrameGeom once
MDG_D CellWalk cell_walk(const FrameGeom& g) { return CellWalk{ g.cdim[0], g.cdim[1], g.cdim[2], g.ncell[0], g.ncell[1], g.ncell[2], g.flags }; }
MDG_D int walk_size(const CellWalk& w) { return (2 * w.n0 + 1) * (2 * w.n1 + 1) * (2 * w.n2 + 1); }

MDG_D uint32_t cell_index(const CellWalk& w, int x, int y, int z) {
    return ((uint32_t)z * (uint32_t)w.cd1 + (uint32_t)y) * (uint32_t)w.cd0 + (uint32_t)x;
}

// unclamped cell coordinate of home cell h (h runs over the home grid hlo + [0, hdim))
MDG_D int3 home_cell(const FrameGeom& g, uint32_t h) {
    const uint32_t hd0 = (uint32_t)g.hdim[0], hd1 = (uint32_t)g.hdim[1];
    return make_int3((int)(h % hd0) + g.hlo[0], (int)((h / hd0) % hd1) + g.hlo[1], (int)(h / (hd0 * hd1)) + g.hlo[2]);
}

struct Neighbour { bool ok; uint32_t cj, code; };   // ok: the reference visits target cell cj, with image `code`

template <bool TRI>
MDG_D Neighbour neighbour_cell(const CellWalk& w, int3 c, int n) {
    const int cd0 = w.cd0, cd1 = w.cd1, cd2 = w.cd2, w0 = 2 * w.n0 + 1, w1 = 2 * w.n1 + 1;
    int nx = c.x + (n % w0 - w.n0), ny = c.y + ((n / w0) % w1 - w.n1), nz = c.z + (n / (w0 * w1) - w.n2);
    const bool upx = nx > cd0 - 1, lox = nx < 0, upy = ny > cd1 - 1, loy = ny < 0, upz = nz > cd2 - 1, loz = nz < 0;
    bool ok = true;
    if (!TRI) {   // wraps on non-periodic axes are skipped (:1733); triclinic cells are periodic in all axes (:1556-1557)
        if ((upx || lox) && !(w.flags & MDGPU_CELL_PBC_X)) ok = false;
        if ((upy || loy) && !(w.flags & MDGPU_CELL_PBC_Y)) ok = false;
        if ((upz || loz) && !(w.flags & MDGPU_CELL_PBC_Z)) ok = false;
    }
    nx += lox ? cd0 : 0; nx -= upx ? cd0 : 0;
    ny += loy ? cd1 : 0; ny -= upy ? cd1 : 0;
    nz += loz ? cd2 : 0; nz -= upz ? cd2 : 0;
    // the reference wraps once only; a coordinate still outside would index out of bounds there
    if (nx < 0 || nx >= cd0 || ny < 0 || ny >= cd1 || nz < 0 || nz >= cd2) ok = false;
    const int sx = (lox ? 1 : 0) - (upx ? 1 : 0), sy = (loy ? 1 : 0) - (upy ? 1 : 0), sz = (loz ? 1 : 0) - (upz ? 1 : 0);
    return Neighbour{ ok, cell_index(w, nx, ny, nz), (uint32_t)(sx + 1) | ((uint32_t)(sy + 1) << 2) | ((uint32_t)(sz + 1) << 4) };
}

MDG_D float3 image_shift(uint32_t code) {   // the shift added to the reference point (:1755)
    return make_float3((float)((int)(code & 3u) - 1), (float)((int)((code >> 2) & 3u) - 1), (float)((int)((code >> 4) & 3u) - 1));
}

// Symmetric mode (reference selection == target selection): a pair of atoms reached WITHOUT an image shift has a bit-identical d2 in both
// directions (s_i - s_j = -(s_j - s_i) exactly, squares equal), so of two different cells only the one with the smaller index evaluates it,
// and counts it twice; the home cell's own pairs count once. Shifted pairs round (f +- 1) before the subtraction and are not symmetric:
// both directions are evaluated. The values are the unshifted classes of the rdf candidate lists.
enum SymClass : uint32_t { SYM_TWICE = 0, SYM_HOME = 1, SYM_SKIP = 3 };
MDG_D uint32_t sym_class(uint32_t cj, uint32_t ch) { return cj > ch ? SYM_TWICE : (cj == ch ? SYM_HOME : SYM_SKIP); }

// d2 = fma(G00, dx*dx, fma(G11, dy*dy, G22*dz*dz)): distance_squared_ort_256 (:524-529); triclinic cells add the cross terms of
// distance_squared_tri_256 (:503-515)
template <bool TRI>
MDG_D float pair_d2(float dx, float dy, float dz, const FrameGeom& g) {
    const float dx2 = __fmul_rn(dx, dx), dy2 = __fmul_rn(dy, dy), dz2 = __fmul_rn(dz, dz);
    if (!TRI) return __fmaf_rn(g.G00, dx2, __fmaf_rn(g.G11, dy2, __fmul_rn(g.G22, dz2)));
    const float dxy = __fmul_rn(dx, dy), dxz = __fmul_rn(dx, dz), dyz = __fmul_rn(dy, dz);
    const float acc = __fmaf_rn(g.G00, dx2, __fmaf_rn(g.G11, dy2, __fmul_rn(g.G22, dz2)));
    return __fadd_rn(acc, __fmaf_rn(g.H01, dxy, __fmaf_rn(g.H02, dxz, __fmul_rn(g.H12, dyz))));
}

}  // namespace mdg
