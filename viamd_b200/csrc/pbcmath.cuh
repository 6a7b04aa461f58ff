// pbcmath.cuh — the reference's periodic-cell routines, each restated bit for bit once, for every file that needs one: cells.cu (inverse
// cell), sdf.cu (bond unwrap, rmsd, plane, shape weights, array-of-selections arguments), props.cu (density, distance / angle / dihedral,
// centres of mass, pair distances) and porosity.cu. The cell as float box and double inverse, the orthorhombic deperiodisation, the 27-image
// triclinic minimum, vec3_normalize, the Cephes sincos lane, and the centres of mass com_vec4 / md_util_com_compute_vec4.
#pragma once
#include "common.cuh"

namespace mdg {

// md_unitcell_A_extract_float (md_unitcell.inl:143): the basis as float box[col][row]
MDG_D void cell_box(const mdgpu_unitcell_t& uc, float box[3][3]) {
    box[0][0] = (float)uc.x;  box[0][1] = 0.f;          box[0][2] = 0.f;
    box[1][0] = (float)uc.xy; box[1][1] = (float)uc.y;  box[1][2] = 0.f;
    box[2][0] = (float)uc.xz; box[2][1] = (float)uc.yz; box[2][2] = (float)uc.z;
}

// md_unitcell_I_extract_double (md_unitcell.inl:158-176): the inverse basis I[col][row]
MDG_HD void cell_inverse(const mdgpu_unitcell_t& uc, double I[3][3]) {
    const double i11 = uc.x > 0.0 ? 1.0 / uc.x : 0.0;
    const double i22 = uc.y > 0.0 ? 1.0 / uc.y : 0.0;
    const double i33 = uc.z > 0.0 ? 1.0 / uc.z : 0.0;
    const double i12 = (uc.x * uc.y) > 0.0 ? -uc.xy / (uc.x * uc.y) : 0.0;
    const double i13 = (uc.x * uc.y * uc.z) > 0.0 ? (uc.xy * uc.yz - uc.xz * uc.y) / (uc.x * uc.y * uc.z) : 0.0;
    const double i23 = (uc.y * uc.z) > 0.0 ? -uc.yz / (uc.y * uc.z) : 0.0;
    I[0][0] = i11; I[0][1] = 0.0; I[0][2] = 0.0;
    I[1][0] = i12; I[1][1] = i22; I[1][2] = 0.0;
    I[2][0] = i13; I[2][1] = i23; I[2][2] = i33;
}

// vec4_deperiodize_ortho (core/md_vec_math.h:1242-1253): round = nearest-even
MDG_D float deperiodize1(float x, float r, float ext) {
    if (ext == 0.0f) return x;
    const float inv = __fdiv_rn(1.0f, ext);
    const float dx = __fmul_rn(__fsub_rn(x, r), inv);
    const float dxp = __fsub_rn(dx, rintf(dx));
    return __fadd_rn(r, __fmul_rn(dxp, ext));
}

// minimum_image_triclinic md_util.c:1677-1718: the 27 images, squared length compared in double, first minimum in loop order wins.
// The sums are mixed precision as written there: float products (box * int) and float sums where both operands are float.
MDG_D void min_image_triclinic(float dx[3], const float box[3][3]) {
    double m0 = 0.0, m1 = 0.0, m2 = 0.0, dsq_min = (double)3.402823466e+38f;
    for (int ix = -1; ix < 2; ++ix) {
        const double rx = (double)__fadd_rn(dx[0], __fmul_rn(box[0][0], (float)ix));
        for (int iy = -1; iy < 2; ++iy) {
            const double ry0 = __dadd_rn(rx, (double)__fmul_rn(box[1][0], (float)iy));
            const double ry1 = (double)__fadd_rn(dx[1], __fmul_rn(box[1][1], (float)iy));
            for (int iz = -1; iz < 2; ++iz) {
                const double rz0 = __dadd_rn(ry0, (double)__fmul_rn(box[2][0], (float)iz)), rz1 = __dadd_rn(ry1, (double)__fmul_rn(box[2][1], (float)iz));
                const double rz2 = (double)__fadd_rn(dx[2], __fmul_rn(box[2][2], (float)iz));
                const double dsq = __dadd_rn(__dadd_rn(__dmul_rn(rz0, rz0), __dmul_rn(rz1, rz1)), __dmul_rn(rz2, rz2));
                if (dsq < dsq_min) { dsq_min = dsq; m0 = rz0; m1 = rz1; m2 = rz2; }
            }
        }
    }
    dx[0] = (float)m0; dx[1] = (float)m1; dx[2] = (float)m2;
}

MDG_D void normalize3(float v[3]) {   // vec3_normalize core/md_vec_math.h:505-514 (threshold compared in double)
    const float len = __fsqrt_rn(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if ((double)len > 1.0e-5) { v[0] = v[0] / len; v[1] = v[1] / len; v[2] = v[2] / len; } else { v[0] = v[1] = v[2] = 0.0f; }
}

// One lane of the reference's sincos (core/md_simd.h, Cephes polynomials): every operation is an IEEE float op (explicit FMAs where the
// reference has fmadd intrinsics), so the GPU reproduces the SIMD build bit for bit. The 4-lane md_mm_sincos_ps (:1093-1176) and the 8-lane
// md_mm256_sincos_ps (:1177-1258) spell the third Cody-Waite constant differently, one float ulp apart (0xB32216A9, 0xB32216A8): dp3 is
// the spelling of the variant the caller reproduces.
constexpr float SINCOS_DP3_PS = -3.77489497744594108e-8f, SINCOS_DP3_PS256 = -3.77489470793079817668E-8f;
MDG_D void sincos_cephes(float x, float dp3, float& out_s, float& out_c) {
    uint32_t sign_bit_sin = __float_as_uint(x) & 0x80000000u;
    x = fabsf(x);
    float y = __fmul_rn(x, 1.27323954473516f);
    int imm2 = __float2int_rz(y);
    imm2 = (imm2 + 1) & ~1;
    y = (float)imm2;
    const uint32_t swap_sign_bit_sin = ((uint32_t)(imm2 & 4)) << 29;
    const bool poly_mask = (imm2 & 2) == 0;
    const uint32_t sign_bit_cos = ((uint32_t)(~(imm2 - 2) & 4)) << 29;
    sign_bit_sin ^= swap_sign_bit_sin;
    x = __fmaf_rn(y, -0.78515625f, x);
    x = __fmaf_rn(y, -2.4187564849853515625e-4f, x);
    x = __fmaf_rn(y, dp3, x);
    const float x2 = __fmul_rn(x, x), x3 = __fmul_rn(x2, x), x4 = __fmul_rn(x2, x2);
    y = __fmaf_rn(x2, __fmaf_rn(x2, 2.443315711809948E-005f, -1.388731625493765E-003f), 4.166664568298827E-002f);
    y = __fmaf_rn(x2, -0.5f, __fmul_rn(y, x4));
    y = __fadd_rn(y, 1.0f);
    float y2 = __fmaf_rn(x2, __fmaf_rn(x2, -1.9515295891E-4f, 8.3321608736E-3f), -1.6666654611E-1f);
    y2 = __fmaf_rn(y2, x3, x);
    const float ysin2 = poly_mask ? y2 : 0.0f, ysin1 = poly_mask ? 0.0f : y;
    y2 = __fsub_rn(y2, ysin2); y = __fsub_rn(y, ysin1);
    out_s = __uint_as_float(__float_as_uint(__fadd_rn(ysin1, ysin2)) ^ sign_bit_sin);
    out_c = __uint_as_float(__float_as_uint(__fadd_rn(y, y2)) ^ sign_bit_cos);
}

// com_vec4 (md_util.c:8048-8061): the plain weighted centre of n points xyzw, float sums in index order
MDG_D void com_vec4(const float4* p, uint32_t n, float com[3]) {
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    for (uint32_t k = 0; k < n; ++k) { const float4 v = p[k]; ax = ax + v.x * v.w; ay = ay + v.y * v.w; az = az + v.z * v.w; aw = aw + v.w * 1.0f; }
    com[0] = ax / aw; com[1] = ay / aw; com[2] = az / aw;
}

// md_util_com_compute_vec4 (md_util.c:8188-8201) of n points xyzw: com_pbc_vec4 (:8063-8162) in a cell — serial float sums of w*sin, w*cos
// per axis in index order, the 4-lane md_mm_sincos_ps, double atan2; the triclinic branch as written (in_idx == NULL: theta through the
// 1/2pi-scaled inverse, and the result through it again) — com_vec4 without one. One thread.
MDG_D void com_compute_vec4(const float4* p, uint32_t n, const mdgpu_unitcell_t& uc, float com[3]) {
    const double TWO_PI_D = 2.0 * 3.1415926535897932, PI_D = 3.1415926535897932;
    if (uc.flags & MDGPU_CELL_ORTHO) {
        const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
        const float tp = (float)TWO_PI_D;
        const float scl[4] = { tp / ext[0], tp / ext[1], tp / ext[2], tp / tp };
        float as[4] = { 0.f, 0.f, 0.f, 0.f }, ac[4] = { 0.f, 0.f, 0.f, 0.f }, ax[4] = { 0.f, 0.f, 0.f, 0.f };
        for (uint32_t k = 0; k < n; ++k) {
            const float4 v = p[k]; const float e[4] = { v.x, v.y, v.z, v.w }, www1[4] = { v.w, v.w, v.w, 1.0f };
            for (int c = 0; c < 4; ++c) {
                float sn, cs; sincos_cephes(e[c] * scl[c], SINCOS_DP3_PS, sn, cs);   // one lane of the 4-lane md_mm_sincos_ps (its constant: core/md_simd.h:1137)
                as[c] = as[c] + sn * www1[c]; ac[c] = ac[c] + cs * www1[c]; ax[c] = ax[c] + e[c] * www1[c];
            }
        }
        const float w = ax[3];
        for (int c = 0; c < 3; ++c) {
            const double yy = (double)(as[c] / w), xx = (double)(ac[c] / w), r2 = xx * xx + yy * yy;
            double theta = PI_D; if (r2 > 1.0e-15) theta += atan2(-yy, -xx);
            com[c] = (float)((theta / TWO_PI_D) * (double)ext[c]);
        }
    } else if (uc.flags & MDGPU_CELL_TRICLINIC) {
        double Id[3][3]; cell_inverse(uc, Id);
        float Ai[3][3];   // [col][row]
        for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) Ai[c][r] = (float)Id[c][r];
        const float inv_tp = 1.0f / (float)TWO_PI_D;
        float I[3][3];   // mat3_mul(mat3_scale(1/2pi), Ai) (core/md_vec_math.h:1631): the three products of MULT(col,row), two of them with a zero factor
        for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) {
            const float s0 = (r == 0) ? inv_tp : 0.0f, s1 = (r == 1) ? inv_tp : 0.0f, s2 = (r == 2) ? inv_tp : 0.0f;
            I[c][r] = (s0 * Ai[c][0] + s1 * Ai[c][1]) + s2 * Ai[c][2];
        }
        float as[4] = { 0.f, 0.f, 0.f, 0.f }, ac[4] = { 0.f, 0.f, 0.f, 0.f }, ax[4] = { 0.f, 0.f, 0.f, 0.f };
        for (uint32_t k = 0; k < n; ++k) {
            const float4 v = p[k]; const float e[4] = { v.x, v.y, v.z, v.w }, www1[4] = { v.w, v.w, v.w, 1.0f };
            float th[4];   // mat4x3_mul_vec4(I, xyzw), the in_idx == NULL branch (:8138)
            for (int c = 0; c < 3; ++c) th[c] = (v.x * I[0][c] + v.y * I[1][c]) + v.z * I[2][c];
            th[3] = (v.x * 0.0f + v.y * 0.0f) + v.z * 0.0f;
            for (int c = 0; c < 4; ++c) {
                float sn, cs; sincos_cephes(th[c], SINCOS_DP3_PS, sn, cs);   // md_mm_sincos_ps, as above
                as[c] = as[c] + sn * www1[c]; ac[c] = ac[c] + cs * www1[c]; ax[c] = ax[c] + e[c] * www1[c];
            }
        }
        for (int c = 0; c < 3; ++c) {
            const double yy = (double)(as[c] / ax[3]), xx = (double)(ac[c] / ax[3]), r2 = xx * xx + yy * yy;
            double theta = PI_D; if (r2 > 1.0e-8) theta += atan2(-yy, -xx);
            com[c] = (float)(theta * (double)I[c][0] + theta * (double)I[c][1] + theta * (double)I[c][2]);   // :8158, as written
        }
    } else com_vec4(p, n, com);   // no cell: nothing to deperiodize
}

}  // namespace mdg
