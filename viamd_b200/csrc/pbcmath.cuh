// pbcmath.cuh — periodic-cell helpers shared by sdf.cu (shape weights, array-of-selections arguments) and porosity.cu: the
// trigonometric centre of mass md_util_com_compute_vec4 and the orthorhombic deperiodisation, restated bit for bit.
#pragma once
#include "common.cuh"

namespace mdg {

// vec4_deperiodize_ortho (core/md_vec_math.h:1242-1253): round = nearest-even
MDG_D float deperiodize1(float x, float r, float ext) {
    if (ext == 0.0f) return x;
    const float inv = __fdiv_rn(1.0f, ext);
    const float dx = __fmul_rn(__fsub_rn(x, r), inv);
    const float dxp = __fsub_rn(dx, rintf(dx));
    return __fadd_rn(r, __fmul_rn(dxp, ext));
}

// One lane of the 4-lane md_mm_sincos_ps (core/md_simd.h:1093-1176): the Cephes sequence of props.cu's ref_sincosf with the third
// Cody-Waite constant as that variant spells it (:1137).
MDG_D void sincos_cephes4(float x, float& out_s, float& out_c) {
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
    x = __fmaf_rn(y, -3.77489497744594108e-8f, x);
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

// md_util_com_compute_vec4 (md_util.c:8188-8201) of n points xyzw: com_pbc_vec4 (:8063-8162) in a cell — serial float sums of w*sin, w*cos
// per axis in index order, 4-lane sincos, double atan2; the triclinic branch as written (in_idx == NULL: theta through the 1/2pi-scaled
// inverse, and the result through it again) — com_vec4 (:8048) without one. One thread.
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
                float sn, cs; sincos_cephes4(e[c] * scl[c], sn, cs);
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
        const double i11 = uc.x > 0.0 ? 1.0 / uc.x : 0.0, i22 = uc.y > 0.0 ? 1.0 / uc.y : 0.0, i33 = uc.z > 0.0 ? 1.0 / uc.z : 0.0;   // md_unitcell.inl:158-176
        const double i12 = (uc.x * uc.y) > 0.0 ? -uc.xy / (uc.x * uc.y) : 0.0;
        const double i13 = (uc.x * uc.y * uc.z) > 0.0 ? (uc.xy * uc.yz - uc.xz * uc.y) / (uc.x * uc.y * uc.z) : 0.0;
        const double i23 = (uc.y * uc.z) > 0.0 ? -uc.yz / (uc.y * uc.z) : 0.0;
        const float Ai[3][3] = { { (float)i11, 0.f, 0.f }, { (float)i12, (float)i22, 0.f }, { (float)i13, (float)i23, (float)i33 } };   // [col][row]
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
                float sn, cs; sincos_cephes4(th[c], sn, cs);
                as[c] = as[c] + sn * www1[c]; ac[c] = ac[c] + cs * www1[c]; ax[c] = ax[c] + e[c] * www1[c];
            }
        }
        for (int c = 0; c < 3; ++c) {
            const double yy = (double)(as[c] / ax[3]), xx = (double)(ac[c] / ax[3]), r2 = xx * xx + yy * yy;
            double theta = PI_D; if (r2 > 1.0e-8) theta += atan2(-yy, -xx);
            com[c] = (float)(theta * (double)I[c][0] + theta * (double)I[c][1] + theta * (double)I[c][2]);   // :8158, as written
        }
    } else {   // no cell: com_vec4, nothing to deperiodize
        float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
        for (uint32_t k = 0; k < n; ++k) { const float4 v = p[k]; ax = ax + v.x * v.w; ay = ay + v.y * v.w; az = az + v.z * v.w; aw = aw + v.w * 1.0f; }
        com[0] = ax / aw; com[1] = ay / aw; com[2] = az / aw;
    }
}

}  // namespace mdg
