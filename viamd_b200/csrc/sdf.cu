// sdf.cu — K3 (local reference-frame fit per structure) and K4 (AABB gather + transform + voxel scatter) for sdf().
//
// Replaces _sdf / sdf_cb (reference md_script_functions.inl:5643-5856), md_util_unwrap_vec4 (md_util.c:8738-8819,8938),
// mat3_covariance_matrix_vec4 / mat3_cross_covariance_matrix_vec4 / mat3_eigen / mat3_extract_rotation
// (core/md_vec_math.c:22-42,101-156,227-300), svd (ext/svd3/svd3.c) and md_spatial_acc_for_each_point_in_aabb
// (core/md_spatial_acc.c:1805-2007). The cell routines under them (deperiodisation, 27-image minimum, com_vec4) are pbcmath.cuh's.
//
// All float expressions keep the reference's association; double accumulators stay double; the library is built with
// --fmad=false so nothing is contracted. The only fused operations are the reference's explicit fmadd intrinsics.
#include "common.cuh"
#include "kernels.h"
#include "pbcmath.cuh"

namespace mdg {

constexpr int SDF_REC = 32;   // floats per structure record: M[16] com[3] pad lo[3] hi[3] cmin[3] cmax[3]

// ------------------------------------------------------------------------------------------------- 3x3 SVD (McAdams)
struct M3 { float e[3][3]; };   // e[col][row] as in the reference's mat3_t; the svd routine itself is row-major A[r][c]
struct M4 { float e[4][4]; };

MDG_D float inv_sqrtf_(float v) { return __fdiv_rn(1.0f, __fsqrt_rn(v)); }
MDG_D void cond_swap(bool c, float& X, float& Y) { const float Z = X; X = c ? Y : X; Y = c ? Z : Y; }
MDG_D void cond_neg_swap(bool c, float& X, float& Y) { const float Z = -X; X = c ? Y : X; Y = c ? Z : Y; }

MDG_D void approx_givens(float a11, float a12, float a22, float& ch, float& sh) {
    ch = 2.0f * (a11 - a22);
    sh = a12;
    // _gamma is a double literal in svd3.c: the comparison is evaluated in double
    const bool b = 5.828427124746190097 * (double)sh * (double)sh < (double)(ch * ch);
    const float w = inv_sqrtf_(ch * ch + sh * sh);
    ch = b ? w * ch : (float)0.923879532511286756;
    sh = b ? w * sh : (float)0.382683432365089771;
}

MDG_D void jacobi_conj(const int x, const int y, const int z, float S[3][3], float q[4]) {
    float ch, sh; approx_givens(S[0][0], S[1][0], S[1][1], ch, sh);
    const float scale = ch * ch + sh * sh;
    const float a = (ch * ch - sh * sh) / scale;
    const float b = (2.0f * sh * ch) / scale;
    const float s00 = S[0][0], s10 = S[1][0], s11 = S[1][1], s20 = S[2][0], s21 = S[2][1], s22 = S[2][2];
    const float n00 = a * (a * s00 + b * s10) + b * (a * s10 + b * s11);
    const float n10 = a * (-b * s00 + a * s10) + b * (-b * s10 + a * s11);
    const float n11 = -b * (-b * s00 + a * s10) + a * (-b * s10 + a * s11);
    const float n20 = a * s20 + b * s21;
    const float n21 = -b * s20 + a * s21;
    const float n22 = s22;
    const float tmp0 = q[0] * sh, tmp1 = q[1] * sh, tmp2 = q[2] * sh;
    const float tmp[3] = { tmp0, tmp1, tmp2 };
    sh *= q[3];
    q[0] *= ch; q[1] *= ch; q[2] *= ch; q[3] *= ch;
    q[z] += sh; q[3] -= tmp[z]; q[x] += tmp[y]; q[y] -= tmp[x];
    S[0][0] = n11; S[1][0] = n21; S[1][1] = n22; S[2][0] = n10; S[2][1] = n20; S[2][2] = n00;
}

MDG_D float dist2_(float a, float b, float c) { return a * a + b * b + c * c; }

MDG_D void qr_givens(float a1, float a2, float& ch, float& sh) {
    const float epsilon = (float)1e-6;
    const float rho = __fsqrt_rn(a1 * a1 + a2 * a2);
    sh = rho > epsilon ? a2 : 0.0f;
    ch = fabsf(a1) + fmaxf(rho, epsilon);
    const bool b = a1 < 0.0f;
    cond_swap(b, sh, ch);
    const float w = inv_sqrtf_(ch * ch + sh * sh);
    ch *= w; sh *= w;
}

__device__ __noinline__ void svd3(const float A[3][3], float U[3][3], float S[3][3], float V[3][3]) {
    float ATA[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) ATA[i][j] = A[0][i] * A[0][j] + A[1][i] * A[1][j] + A[2][i] * A[2][j];
    float q[4] = { 0.f, 0.f, 0.f, 1.f };
    for (int it = 0; it < 4; ++it) { jacobi_conj(0, 1, 2, ATA, q); jacobi_conj(1, 2, 0, ATA, q); jacobi_conj(2, 0, 1, ATA, q); }
    {
        const float x = q[0], y = q[1], z = q[2], w = q[3];
        const float qxx = x * x, qyy = y * y, qzz = z * z, qxz = x * z, qxy = x * y, qyz = y * z, qwx = w * x, qwy = w * y, qwz = w * z;
        V[0][0] = 1.0f - 2.0f * (qyy + qzz); V[0][1] = 2.0f * (qxy - qwz);        V[0][2] = 2.0f * (qxz + qwy);
        V[1][0] = 2.0f * (qxy + qwz);        V[1][1] = 1.0f - 2.0f * (qxx + qzz); V[1][2] = 2.0f * (qyz - qwx);
        V[2][0] = 2.0f * (qxz - qwy);        V[2][1] = 2.0f * (qyz + qwx);        V[2][2] = 1.0f - 2.0f * (qxx + qyy);
    }
    float B[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) B[i][j] = A[i][0] * V[0][j] + A[i][1] * V[1][j] + A[i][2] * V[2][j];
    {
        float rho1 = dist2_(B[0][0], B[1][0], B[2][0]), rho2 = dist2_(B[0][1], B[1][1], B[2][1]), rho3 = dist2_(B[0][2], B[1][2], B[2][2]);
        bool c = rho1 < rho2;
#pragma unroll
        for (int r = 0; r < 3; ++r) { cond_neg_swap(c, B[r][0], B[r][1]); cond_neg_swap(c, V[r][0], V[r][1]); }
        cond_swap(c, rho1, rho2);
        c = rho1 < rho3;
#pragma unroll
        for (int r = 0; r < 3; ++r) { cond_neg_swap(c, B[r][0], B[r][2]); cond_neg_swap(c, V[r][0], V[r][2]); }
        cond_swap(c, rho1, rho3);
        c = rho2 < rho3;
#pragma unroll
        for (int r = 0; r < 3; ++r) { cond_neg_swap(c, B[r][1], B[r][2]); cond_neg_swap(c, V[r][1], V[r][2]); }
    }
    {
        float (*Q)[3] = U; float (*R)[3] = S;
        float ch1, sh1, ch2, sh2, ch3, sh3, a, b;
        qr_givens(B[0][0], B[1][0], ch1, sh1);
        a = 1.0f - 2.0f * sh1 * sh1; b = 2.0f * ch1 * sh1;
        R[0][0] = a * B[0][0] + b * B[1][0];  R[0][1] = a * B[0][1] + b * B[1][1];  R[0][2] = a * B[0][2] + b * B[1][2];
        R[1][0] = -b * B[0][0] + a * B[1][0]; R[1][1] = -b * B[0][1] + a * B[1][1]; R[1][2] = -b * B[0][2] + a * B[1][2];
        R[2][0] = B[2][0]; R[2][1] = B[2][1]; R[2][2] = B[2][2];
        qr_givens(R[0][0], R[2][0], ch2, sh2);
        a = 1.0f - 2.0f * sh2 * sh2; b = 2.0f * ch2 * sh2;
        B[0][0] = a * R[0][0] + b * R[2][0];  B[0][1] = a * R[0][1] + b * R[2][1];  B[0][2] = a * R[0][2] + b * R[2][2];
        B[1][0] = R[1][0]; B[1][1] = R[1][1]; B[1][2] = R[1][2];
        B[2][0] = -b * R[0][0] + a * R[2][0]; B[2][1] = -b * R[0][1] + a * R[2][1]; B[2][2] = -b * R[0][2] + a * R[2][2];
        qr_givens(B[1][1], B[2][1], ch3, sh3);
        a = 1.0f - 2.0f * sh3 * sh3; b = 2.0f * ch3 * sh3;
        R[0][0] = B[0][0]; R[0][1] = B[0][1]; R[0][2] = B[0][2];
        R[1][0] = a * B[1][0] + b * B[2][0];  R[1][1] = a * B[1][1] + b * B[2][1];  R[1][2] = a * B[1][2] + b * B[2][2];
        R[2][0] = -b * B[1][0] + a * B[2][0]; R[2][1] = -b * B[1][1] + a * B[2][1]; R[2][2] = -b * B[1][2] + a * B[2][2];
        const float sh12 = sh1 * sh1, sh22 = sh2 * sh2, sh32 = sh3 * sh3;
        Q[0][0] = (-1.0f + 2.0f * sh12) * (-1.0f + 2.0f * sh22);
        Q[0][1] = 4.0f * ch2 * ch3 * (-1.0f + 2.0f * sh12) * sh2 * sh3 + 2.0f * ch1 * sh1 * (-1.0f + 2.0f * sh32);
        Q[0][2] = 4.0f * ch1 * ch3 * sh1 * sh3 - 2.0f * ch2 * (-1.0f + 2.0f * sh12) * sh2 * (-1.0f + 2.0f * sh32);
        Q[1][0] = 2.0f * ch1 * sh1 * (1.0f - 2.0f * sh22);
        Q[1][1] = -8.0f * ch1 * ch2 * ch3 * sh1 * sh2 * sh3 + (-1.0f + 2.0f * sh12) * (-1.0f + 2.0f * sh32);
        Q[1][2] = -2.0f * ch3 * sh3 + 4.0f * sh1 * (ch3 * sh1 * sh3 + ch1 * ch2 * sh2 * (-1.0f + 2.0f * sh32));
        Q[2][0] = 2.0f * ch2 * sh2;
        Q[2][1] = 2.0f * ch3 * (1.0f - 2.0f * sh22) * sh3;
        Q[2][2] = (-1.0f + 2.0f * sh22) * (-1.0f + 2.0f * sh32);
    }
}

// ------------------------------------------------------------------------------------------------- small matrix helpers
MDG_D M3 m3_transpose(const M3& M) { M3 T; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) T.e[i][j] = M.e[j][i]; return T; }
MDG_D M3 m3_mul(const M3& A, const M3& B) {   // core/md_vec_math.h:1631
    M3 C;
    for (int col = 0; col < 3; ++col) for (int row = 0; row < 3; ++row)
        C.e[col][row] = A.e[0][row] * B.e[col][0] + A.e[1][row] * B.e[col][1] + A.e[2][row] * B.e[col][2];
    return C;
}
MDG_D float m3_det(const M3& M) {             // :1687
    return M.e[0][0] * (M.e[1][1] * M.e[2][2] - M.e[2][1] * M.e[1][2])
         - M.e[1][0] * (M.e[0][1] * M.e[2][2] - M.e[2][1] * M.e[0][2])
         + M.e[2][0] * (M.e[0][1] * M.e[1][2] - M.e[1][1] * M.e[0][2]);
}
MDG_D M4 m4_from_m3(const M3& M) { M4 R; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) R.e[i][j] = (i < 3 && j < 3) ? M.e[i][j] : 0.0f; R.e[3][3] = 1.0f; return R; }
MDG_D M4 m4_mul(const M4& A, const M4& B) {   // linear_combine_4 (:1512)
    M4 C;
    for (int j = 0; j < 4; ++j) for (int r = 0; r < 4; ++r) {
        float v = B.e[j][0] * A.e[0][r];
        v = v + B.e[j][1] * A.e[1][r];
        v = v + B.e[j][2] * A.e[2][r];
        v = v + B.e[j][3] * A.e[3][r];
        C.e[j][r] = v;
    }
    return C;
}
struct Svd { M3 U, V; float s[3]; };
MDG_D Svd m3_svd(const M3& M) {               // core/md_vec_math.c:7-20
    M3 Mt = m3_transpose(M), U, S, V;
    svd3(Mt.e, U.e, S.e, V.e);
    Svd r; r.U = m3_transpose(U); r.V = m3_transpose(V); r.s[0] = S.e[0][0]; r.s[1] = S.e[1][1]; r.s[2] = S.e[2][2];
    return r;
}

// mat3_covariance_matrix_vec4 (core/md_vec_math.c:101-156): double sums of the float products (w * x) * y about com, in index order
MDG_D M3 covariance(const float4* p, uint32_t n, const float com[3]) {
    double C[3][3] = { { 0 } }; double ws = 0.0;
    for (uint32_t k = 0; k < n; ++k) {
        const float4 v = p[k];
        const float x = v.x - com[0], y = v.y - com[1], z = v.z - com[2], w = v.w;
        C[0][0] += w * x * x; C[0][1] += w * x * y; C[0][2] += w * x * z;
        C[1][0] += w * y * x; C[1][1] += w * y * y; C[1][2] += w * y * z;
        C[2][0] += w * z * x; C[2][1] += w * z * y; C[2][2] += w * z * z;
        ws += w;
    }
    M3 cov; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) cov.e[i][j] = (float)(C[i][j] / ws);
    return cov;
}

// mat3_cross_covariance_matrix_vec4 (core/md_vec_math.c:256-289): a pair's weight is the mean of its two points' weights, each less the
// zero weight of its centre
MDG_D M3 cross_covariance(const float4* p0, const float com0[3], const float4* p1, const float com1[3], uint32_t n) {
    double C[3][3] = { { 0 } }; double ws = 0.0;
    for (uint32_t k = 0; k < n; ++k) {
        const float4 u = p0[k], v = p1[k];
        const float px = u.x - com0[0], py = u.y - com0[1], pz = u.z - com0[2], pw = u.w - 0.0f;
        const float qx = v.x - com1[0], qy = v.y - com1[1], qz = v.z - com1[2], qw = v.w - 0.0f;
        const float w = (pw + qw) * 0.5f;
        C[0][0] += w * px * qx; C[0][1] += w * px * qy; C[0][2] += w * px * qz;
        C[1][0] += w * py * qx; C[1][1] += w * py * qy; C[1][2] += w * py * qz;
        C[2][0] += w * pz * qx; C[2][1] += w * pz * qy; C[2][2] += w * pz * qz;
        ws += w;
    }
    M3 cc; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) cc.e[i][j] = (float)(C[i][j] / ws);
    return cc;
}

// mat3_eigen (core/md_vec_math.c:22-42): the svd's values normalised by the largest and sorted descending with three compares;
// vec.e[k] is the axis of val[k]
struct Eigen { M3 vec; float val[3]; };
MDG_D Eigen eigen_sorted(const M3& cov) {
    const Svd s = m3_svd(cov);
    const float mx = fmaxf(s.s[0], fmaxf(s.s[1], s.s[2]));
    const float ev[3] = { s.s[0] / mx, s.s[1] / mx, s.s[2] / mx };
    int l0 = 0, l1 = 1, l2 = 2, t;
    if (ev[l0] < ev[l1]) { t = l0; l0 = l1; l1 = t; }
    if (ev[l1] < ev[l2]) { t = l1; l1 = l2; l2 = t; }
    if (ev[l0] < ev[l1]) { t = l0; l0 = l1; l1 = t; }
    const int l[3] = { l0, l1, l2 };
    Eigen r; for (int k = 0; k < 3; ++k) { r.val[k] = ev[l[k]]; for (int i = 0; i < 3; ++i) r.vec.e[k][i] = s.U.e[l[k]][i]; }
    return r;
}

// mat3_extract_rotation (core/md_vec_math.c:292-300): V * diag(1, 1, sign det(V * Ut)) * Ut of the svd
MDG_D M3 extract_rotation(const M3& cc) {
    const Svd sv = m3_svd(cc);
    const M3 Ut = m3_transpose(sv.U);
    const float d = m3_det(m3_mul(sv.V, Ut));
    M3 D; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) D.e[i][j] = 0.0f; D.e[0][0] = 1.0f; D.e[1][1] = 1.0f; D.e[2][2] = (float)((d > 0.0f) - (d < 0.0f));
    return m3_mul(m3_mul(sv.V, D), Ut);
}

// The bond walk of md_util_unwrap_vec4 (md_util.c:8938) on atoms in scratch: each child of the (child, parent) pairs, in BFS order, moves
// to the image nearest its parent
MDG_D void unwrap_bonds(float4* p, const int2* pairs, uint32_t n_pairs, const mdgpu_unitcell_t& uc) {
    if (uc.flags & MDGPU_CELL_ORTHO) {
        const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
        for (uint32_t k = 0; k < n_pairs; ++k) {
            const int2 pr = pairs[k];
            const float4 ref = p[pr.y]; float4 v = p[pr.x];
            v.x = deperiodize1(v.x, ref.x, ext[0]); v.y = deperiodize1(v.y, ref.y, ext[1]); v.z = deperiodize1(v.z, ref.z, ext[2]);
            p[pr.x] = v;
        }
    } else if (uc.flags & MDGPU_CELL_TRICLINIC) {   // unwrap_atom_triclinic_vec4 -> deperiodize_triclinic md_util.c:1754-1766
        float box[3][3]; cell_box(uc, box);
        for (uint32_t k = 0; k < n_pairs; ++k) {
            const int2 pr = pairs[k];
            const float4 ref = p[pr.y]; float4 v = p[pr.x];
            float d[3] = { __fsub_rn(v.x, ref.x), __fsub_rn(v.y, ref.y), __fsub_rn(v.z, ref.z) };
            min_image_triclinic(d, box);
            v.x = __fadd_rn(ref.x, d[0]); v.y = __fadd_rn(ref.y, d[1]); v.z = __fadd_rn(ref.z, d[2]);
            p[pr.x] = v;
        }
    }
}

// bond walk + plain centre of mass of a structure in scratch
MDG_D void unwrap_com(float4* p, uint32_t n, const int2* pairs, uint32_t n_pairs, const mdgpu_unitcell_t& uc, float com[3]) {
    unwrap_bonds(p, pairs, n_pairs, uc);
    com_vec4(p, n, com);
}

// extract + unwrap + centre of mass of one structure into scratch (xyz, mass)
MDG_D void load_unwrap_com(float4* p, const float* x, const float* y, const float* z, const float* mass, const int32_t* sidx, uint32_t n,
                           const int2* pairs, uint32_t n_pairs, const mdgpu_unitcell_t& uc, float com[3]) {
    for (uint32_t k = 0; k < n; ++k) { const int a = sidx[k]; p[k] = make_float4(x[a], y[a], z[a], mass[a]); }
    unwrap_com(p, n, pairs, n_pairs, uc, com);
}

// cartesian -> fractional through the frame's float inverse basis, evaluated in double: ((I0 * x) + (I1 * y)) + (I2 * z) of r - origin
MDG_D void cart_to_fract_d(const FrameGeom& g, double x, double y, double z, double s[3]) {
    const double px = x - g.origin[0], py = y - g.origin[1], pz = z - g.origin[2];
    for (int k = 0; k < 3; ++k) s[k] = g.I[0][k] * px + g.I[1][k] * py + g.I[2][k] * pz;
}

// Reference structure (structure 0 of the INITIAL frame, unwrapped with the CURRENT frame's cell :5762-5782): PCA frame and V*A
__global__ void k_sdf_ref0(SdfArgs a, int B) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= B) return;
    const uint32_t n = a.struct_size;
    float4* p = a.scratch_xyzw + ((size_t)f * (a.n_struct + 1) + a.n_struct) * n;
    float com0[3];
    load_unwrap_com(p, a.init_xyz, a.init_xyz + a.init_axis_stride, a.init_xyz + 2 * a.init_axis_stride, a.mass, a.struct_idx, n,
                    a.unwrap_pairs, a.n_unwrap, a.cells[f], com0);
    const M4 A = m4_from_m3(m3_transpose(eigen_sorted(covariance(p, n, com0)).vec));
    // compute_volume_matrix (:5643-5655)
    const float voxel_ext = (2.0f * a.cutoff) / (float)MDGPU_VOL_DIM;
    const float sc = 1.0f / voxel_ext;
    M4 S; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) S.e[i][j] = 0.0f; S.e[0][0] = sc; S.e[1][1] = sc; S.e[2][2] = sc; S.e[3][3] = 1.0f;
    const float tt = (float)(MDGPU_VOL_DIM / 2);
    M4 T; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) T.e[i][j] = (i == j) ? 1.0f : 0.0f; T.e[3][0] = tt; T.e[3][1] = tt; T.e[3][2] = tt;
    const M4 VA = m4_mul(m4_mul(T, S), A);
    float* o = a.ref0 + (size_t)f * 20;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) o[i * 4 + j] = VA.e[i][j];
    o[16] = com0[0]; o[17] = com0[1]; o[18] = com0[2]; o[19] = 0.0f;
}

// K3: one thread per (structure, frame): M = V*A*R*T(-com) (:5788-5799)
__global__ void k_sdf_fit(SdfArgs a, int B) {
    const int f = blockIdx.y;
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_struct) return;
    const uint32_t n = a.struct_size;
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    float4* p1 = a.scratch_xyzw + ((size_t)f * (a.n_struct + 1) + s) * n;
    const float4* p0 = a.scratch_xyzw + ((size_t)f * (a.n_struct + 1) + a.n_struct) * n;
    const float* r0 = a.ref0 + (size_t)f * 20;
    const float com0[3] = { r0[16], r0[17], r0[18] };
    float com1[3];
    load_unwrap_com(p1, x, x + a.frames.axis_stride, x + 2 * a.frames.axis_stride, a.mass, a.struct_idx + (size_t)s * n, n,
                    a.unwrap_pairs, a.n_unwrap, a.cells[f], com1);
    const M3 R = extract_rotation(cross_covariance(p0, com0, p1, com1, n));
    M4 Tm; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) Tm.e[i][j] = (i == j) ? 1.0f : 0.0f; Tm.e[3][0] = -com1[0]; Tm.e[3][1] = -com1[1]; Tm.e[3][2] = -com1[2];
    const M4 RT = m4_mul(m4_from_m3(R), Tm);
    M4 VA; for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) VA.e[i][j] = r0[i * 4 + j];
    const M4 M = m4_mul(VA, RT);
    float* o = a.matrices + ((size_t)f * a.n_struct + s) * SDF_REC;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) o[i * 4 + j] = M.e[i][j];
    o[16] = com1[0]; o[17] = com1[1]; o[18] = com1[2]; o[19] = 0.0f;

    // cell_range_from_aabb_center_radius + the fractional bounds of for_each_point_in_aabb_ortho (core/md_spatial_acc.c:1805-1923),
    // double precision with the float matrix entries widened, evaluated once per structure
    const FrameGeom& g = a.geom[f];
    const double rad = (double)a.cutoff;
    const int pbc[3] = { (g.flags & MDGPU_CELL_PBC_X) != 0, (g.flags & MDGPU_CELL_PBC_Y) != 0, (g.flags & MDGPU_CELL_PBC_Z) != 0 };
    double sc[3], ccen[3];
    cart_to_fract_d(g, (double)com1[0], (double)com1[1], (double)com1[2], sc);
    for (int k = 0; k < 3; ++k) if (pbc[k]) sc[k] = sc[k] - floor(sc[k]);
    ccen[0] = g.A[0][0] * sc[0] + g.A[1][0] * sc[1] + g.A[2][0] * sc[2] + g.origin[0];
    ccen[1] = g.A[0][1] * sc[0] + g.A[1][1] * sc[1] + g.A[2][1] * sc[2] + g.origin[1];
    ccen[2] = g.A[0][2] * sc[0] + g.A[1][2] * sc[1] + g.A[2][2] * sc[2] + g.origin[2];
    double fmin_[3] = { DBL_MAX, DBL_MAX, DBL_MAX }, fmax_[3] = { -DBL_MAX, -DBL_MAX, -DBL_MAX };
    for (int corner = 0; corner < 8; ++corner) {
        const double pz = ccen[2] + ((corner & 4) ? rad : -rad), py = ccen[1] + ((corner & 2) ? rad : -rad), px = ccen[0] + ((corner & 1) ? rad : -rad);
        double sv[3]; cart_to_fract_d(g, px, py, pz, sv);
        for (int k = 0; k < 3; ++k) { fmin_[k] = fmin(fmin_[k], sv[k]); fmax_[k] = fmax(fmax_[k], sv[k]); }
    }
    int* oi = (int*)(o + 26);
    for (int k = 0; k < 3; ++k) {
        const int cdk = g.cdim[k];
        double frad = 0.5 * (fmax_[k] - fmin_[k]);
        int lo = (int)floor(fmin_[k] * (double)cdk), hi = (int)ceil(fmax_[k] * (double)cdk);
        if (hi <= lo) hi = lo + 1;
        if (!pbc[k]) { lo = max(0, min(lo, cdk)); hi = max(0, min(hi, cdk)); if (hi <= lo) hi = min(lo + 1, cdk); }
        frad = fmin(frad, 0.5);
        if (g.flags & MDGPU_CELL_TRICLINIC) { o[20 + k] = (float)(ccen[k] - rad); o[23 + k] = (float)(ccen[k] + rad); }   // cartesian bounds (:2041-2047)
        else { o[20 + k] = (float)(sc[k] - frad); o[23 + k] = (float)(sc[k] + frad); }                                   // fractional bounds (:1913-1923)
        oi[k] = lo; oi[3 + k] = hi;
    }
}

MDG_D int wrap_coord(int v, int N) { v += (v < 0) ? N : 0; v -= (v >= N) ? N : 0; return v; }
MDG_D int isign(int v) { return (v > 0) - (v < 0); }

// K4: one warp per (structure, frame): target points of the cells overlapping AABB(com, cutoff) -> voxel increments.
//  * lanes enumerate the cells of the range once (wrap, image code, offsets) into a small per-warp segment table;
//  * each HALF-warp then walks one cell at a time, 16 points per step (a cell of the bench workload holds ~45 targets: three steps at 94 %
//    lane use, where a full warp per cell would run two steps at 70 % and a flattened index space pays a boundary search per step);
//  * the box test passes ~60 % of the candidates (the box is 20 A wide, the 2-3 cells per axis it overlaps 22-33 A), so the transform
//    and the voxel increment run in place under the hit predicate — compacting hits first costs more than the idle lanes it would fill.
constexpr int SDF_WARPS = 8;
constexpr int SDF_MIN_CTAS = 4;   // resident CTAs / SM the register allocation of k_sdf_scatter aims for (MINB)
constexpr int SDF_MAXSEG = 128;
constexpr int SDF_EXCL_CACHE = 64;

struct SdfXform { float M[4][3]; float A00, A11, A22, O0, O1, O2, A10, A20, A21; };

// fractional (image-shifted) point -> cartesian -> structure frame -> voxel (:5664-5697)
template <bool TRI>
MDG_D void sdf_splat(float vx, float vy, float vz, const SdfXform& X, uint32_t* __restrict__ vol) {
    // ortho: batch_fract_to_cart_ort_256, one fused multiply-add per axis (md_spatial_acc.c:583-592).
    // triclinic: REFERENCE QUIRK — for_each_point_in_aabb_triclinic buffers the fractional image-shifted coordinates (:2122-2130) and its
    // *_CART_TRI callback macros (:715-737) skip the conversion, so sdf_cb transforms fractional numbers. Reproduced for parity.
    const float px = TRI ? vx : __fmaf_rn(vx, X.A00, X.O0), py = TRI ? vy : __fmaf_rn(vy, X.A11, X.O1), pz = TRI ? vz : __fmaf_rn(vz, X.A22, X.O2);
    float c[3];   // mat4_mul_vec4(M, (x,y,z,1)) = ((x*M0 + y*M1) + z*M2) + 1*M3; 1*M3 is M3 exactly
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        float v = __fmul_rn(px, X.M[0][r]);
        v = __fadd_rn(v, __fmul_rn(py, X.M[1][r]));
        v = __fadd_rn(v, __fmul_rn(pz, X.M[2][r]));
        v = __fadd_rn(v, X.M[3][r]);
        c[r] = v;
    }
    const uint32_t ix = (uint32_t)max(0, min(__float2int_rz(c[0]), MDGPU_VOL_DIM - 1));
    const uint32_t iy = (uint32_t)max(0, min(__float2int_rz(c[1]), MDGPU_VOL_DIM - 1));
    const uint32_t iz = (uint32_t)max(0, min(__float2int_rz(c[2]), MDGPU_VOL_DIM - 1));
    atomicAdd(&vol[(iz * MDGPU_VOL_DIM + iy) * MDGPU_VOL_DIM + ix], 1u);
}

template <bool TRI, int MINB>
__global__ void __launch_bounds__(SDF_WARPS * 32, MINB) k_sdf_scatter(SdfArgs a, int B) {
    const int f = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, hl = lane & 15, half = lane >> 4;
    const uint32_t s = blockIdx.x * SDF_WARPS + warp;
    __shared__ uint2 s_seg[SDF_WARPS][SDF_MAXSEG];        // x: first point of the cell, y: point count | image code << 26
    __shared__ int32_t s_excl[SDF_WARPS][SDF_EXCL_CACHE];
    if (s >= a.n_struct) return;
    const FrameGeom& g = a.geom[f];
    if (g.valid == -1) return;
    const float* rec = a.matrices + ((size_t)f * a.n_struct + s) * SDF_REC;
    SdfXform X;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) X.M[i][j] = rec[i * 4 + j];
    X.A00 = g.A[0][0]; X.A11 = g.A[1][1]; X.A22 = g.A[2][2]; X.O0 = g.origin[0]; X.O1 = g.origin[1]; X.O2 = g.origin[2];
    X.A10 = g.A[1][0]; X.A20 = g.A[2][0]; X.A21 = g.A[2][1];
    const float lo3[3] = { rec[20], rec[21], rec[22] }, hi3[3] = { rec[23], rec[24], rec[25] };
    const int* ri = (const int*)(rec + 26);
    const int cmin[3] = { ri[0], ri[1], ri[2] }, cmax[3] = { ri[3], ri[4], ri[5] };
    const int pbc[3] = { (g.flags & MDGPU_CELL_PBC_X) != 0, (g.flags & MDGPU_CELL_PBC_Y) != 0, (g.flags & MDGPU_CELL_PBC_Z) != 0 };
    const int cd[3] = { g.cdim[0], g.cdim[1], g.cdim[2] };
    const float4* __restrict__ pts = a.trg.sorted + (size_t)f * a.trg.max_points;
    const uint32_t* __restrict__ off = a.trg.cell_cnt + (size_t)f * (a.trg.cap + 1);
    const int32_t* sidx = a.struct_idx + (size_t)s * a.struct_size;
    // exclusion mask = the structure's own atoms (:5674). Ascending index lists: a contiguous run (the usual case: a residue)
    // is tested with one compare; otherwise the list (cached in shared memory when it fits) is scanned.
    const uint32_t ex_lo = (uint32_t)sidx[0], ex_n = a.struct_size;
    const bool ex_contig = ((uint32_t)sidx[a.struct_size - 1] - ex_lo + 1u) == ex_n;
    if (!ex_contig) { for (uint32_t k = lane; k < min(ex_n, (uint32_t)SDF_EXCL_CACHE); k += 32) s_excl[warp][k] = sidx[k]; }
    const int ex = cmax[0] - cmin[0], ey = cmax[1] - cmin[1], ez = cmax[2] - cmin[2];
    const int ncells = ex * ey * ez;
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t local = 0;                    // voxel increments of this lane
    for (int c0 = 0; c0 < ncells; c0 += SDF_MAXSEG) {   // (:1925-1943) cells of the range, SDF_MAXSEG at a time
        const int nc = min(SDF_MAXSEG, ncells - c0);
        int nseg = 0;
        __syncwarp();
        for (int n0 = 0; n0 < nc; n0 += 32) {
            const int n = n0 + lane;
            uint32_t len = 0, start = 0, code = 0x15;
            if (n < nc) {
                const int q = c0 + n;
                const int qx = q % ex, qyz = q / ex;
                const int icx = cmin[0] + qx, icy = cmin[1] + qyz % ey, icz = cmin[2] + qyz / ey;
                const int cx = pbc[0] ? wrap_coord(icx, cd[0]) : icx, cy = pbc[1] ? wrap_coord(icy, cd[1]) : icy, cz = pbc[2] ? wrap_coord(icz, cd[2]) : icz;
                if (!(cx < 0 || cx >= cd[0] || cy < 0 || cy >= cd[1] || cz < 0 || cz >= cd[2])) {
                    const uint32_t ci = ((uint32_t)cz * (uint32_t)cd[1] + (uint32_t)cy) * (uint32_t)cd[0] + (uint32_t)cx;
                    start = off[ci]; len = off[ci + 1] - start;
                    code = (uint32_t)(isign(icx - cx) + 1) | ((uint32_t)(isign(icy - cy) + 1) << 2) | ((uint32_t)(isign(icz - cz) + 1) << 4);
                }
            }
            const uint32_t have = __ballot_sync(0xffffffffu, len != 0u);   // keep non-empty cells only
            if (len) s_seg[warp][nseg + __popc(have & lt)] = make_uint2(start, len | (code << 26));
            nseg += __popc(have);
        }
        __syncwarp();
        for (int k0 = 0; k0 < nseg; k0 += 2) {   // one cell per half-warp
            const int k = k0 + half;
            const uint2 sg = (k < nseg) ? s_seg[warp][k] : make_uint2(0u, 0u);
            const uint32_t len = sg.y & 0x3ffffffu, code = sg.y >> 26;
            const uint32_t steps = max(__shfl_sync(0xffffffffu, len, 0), __shfl_sync(0xffffffffu, len, 16));
            const float shx = (float)((int)(code & 3u) - 1), shy = (float)((int)((code >> 2) & 3u) - 1), shz = (float)((int)((code >> 4) & 3u) - 1);
            auto visit = [&](const float4& t) {   // image shift, box test, exclusion, splat of one candidate
                float vx = t.x, vy = t.y, vz = t.z;
                if (code != 0x15u) {   // periodic image of the cell: + (-1|0|+1), rounded (:1962-1964); +0 is the identity
                    vx = __fadd_rn(vx, shx); vy = __fadd_rn(vy, shy); vz = __fadd_rn(vz, shz);
                }
                bool hit;
                if (TRI) {   // box test on the cartesian image (fract_to_cart_tri_256 md_spatial_acc.c:594-603), all axes periodic (:2009)
                    const float cx_ = __fmaf_rn(vx, X.A00, __fmaf_rn(vy, X.A10, __fmaf_rn(vz, X.A20, X.O0))), cy_ = __fmaf_rn(vy, X.A11, __fmaf_rn(vz, X.A21, X.O1)), cz_ = __fmaf_rn(vz, X.A22, X.O2);
                    hit = cx_ >= lo3[0] && cy_ >= lo3[1] && cz_ >= lo3[2] && cx_ <= hi3[0] && cy_ <= hi3[1] && cz_ <= hi3[2];
                } else hit = vx >= lo3[0] && vy >= lo3[1] && vz >= lo3[2] && vx <= hi3[0] && vy <= hi3[1] && vz <= hi3[2];
                if (hit) {
                    const uint32_t idx = __float_as_uint(t.w);
                    if (ex_contig) hit = (idx - ex_lo) >= ex_n;
                    else {
                        bool excluded = false;
                        const uint32_t nc_ = min(ex_n, (uint32_t)SDF_EXCL_CACHE);
                        for (uint32_t q = 0; q < nc_; ++q) excluded |= ((uint32_t)s_excl[warp][q] == idx);
                        for (uint32_t q = nc_; q < ex_n; ++q) excluded |= ((uint32_t)sidx[q] == idx);
                        hit = !excluded;
                    }
                    if (hit) { sdf_splat<TRI>(vx, vy, vz, X, a.vol); ++local; }
                }
            };
            for (uint32_t j0 = (uint32_t)hl; j0 < steps; j0 += 32u) {   // two candidates per lane and round: both loads in flight before the tests
                const uint32_t j1 = j0 + 16u;
                const bool k0_ = j0 < len, k1_ = j1 < len;
                float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f), t1 = t0;
                if (k0_) t0 = pts[sg.x + j0];
                if (k1_) t1 = pts[sg.x + j1];
                if (k0_) visit(t0);
                if (k1_) visit(t1);
            }
        }
    }
    __syncwarp();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if (lane == 0 && local) atomicAdd(&a.frame_total[a.frame0 + f], (unsigned long long)local);
}

// ------------------------------------------------------------------------------------------------- rmsd(selection)
// _rmsd (md_script_functions.inl:4287-4345): the selection's atoms of the INITIAL frame and of the current frame, both wrapped into the
// current cell (md_util_pbc_vec4 md_util.c:8603), made whole along the bonds (md_util_unwrap_vec4 :8938, same local-index-as-atom quirk as
// in _sdf), centred on their plain centres of mass, fitted with mat3_optimal_rotation_vec4 (core/md_vec_math.c:337) and compared:
// sqrt(sum w |u - R v|^2 / sum w) with double sums (md_util_rmsd_compute_vec4 md_util.c:9037-9068).
//
// One warp per frame. The lanes extract and wrap the atoms (independent per atom); lane 0 then runs the parts whose result depends on
// the order of operations — the bond walk, the float centre-of-mass sums, the double covariance and deviation sums — exactly in the
// reference's order. Selections of rmsd() are one molecule or its backbone (10^2..10^4 atoms), a serial pass over them costs microseconds.
MDG_D float4 pbc_wrap(float4 v, const mdgpu_unitcell_t& uc) {
    if (uc.flags & MDGPU_CELL_ORTHO) {            // pbc_ortho_vec4 :8506-8512: vec4_deperiodize_ortho about the box centre
        const float ex = (float)uc.x, ey = (float)uc.y, ez = (float)uc.z;
        v.x = deperiodize1(v.x, ex * 0.5f, ex); v.y = deperiodize1(v.y, ey * 0.5f, ey); v.z = deperiodize1(v.z, ez * 0.5f, ez);
    } else if (uc.flags & MDGPU_CELL_TRICLINIC) {  // pbc_triclinic_vec4 :8554-8574: A * fract(I * r) on the periodic axes, float matrices
        double Id[3][3]; cell_inverse(uc, Id);   // md_unitcell_I_extract_float: the double inverse, cast
        float A[3][3]; cell_box(uc, A);
        const float I00 = (float)Id[0][0], I10 = (float)Id[1][0], I11 = (float)Id[1][1], I20 = (float)Id[2][0], I21 = (float)Id[2][1], I22 = (float)Id[2][2];
        const float A00 = A[0][0], A10 = A[1][0], A11 = A[1][1], A20 = A[2][0], A21 = A[2][1], A22 = A[2][2];
        // linear_combine_3 (core/md_vec_math.h:1521): (x * col0 + y * col1) + z * col2, the zero entries of the matrices included
        float f0 = (v.x * I00 + v.y * I10) + v.z * I20;
        float f1 = (v.x * 0.0f + v.y * I11) + v.z * I21;
        float f2 = (v.x * 0.0f + v.y * 0.0f) + v.z * I22;
        f0 = f0 - floorf(f0); f1 = f1 - floorf(f1); f2 = f2 - floorf(f2);
        const float r0 = (f0 * A00 + f1 * A10) + f2 * A20;
        const float r1 = (f0 * 0.0f + f1 * A11) + f2 * A21;
        const float r2 = (f0 * 0.0f + f1 * 0.0f) + f2 * A22;
        if (uc.flags & MDGPU_CELL_PBC_X) v.x = r0;
        if (uc.flags & MDGPU_CELL_PBC_Y) v.y = r1;
        if (uc.flags & MDGPU_CELL_PBC_Z) v.z = r2;
    }
    return v;
}

// extract_xyzw_vec4 (:966) + md_util_pbc_vec4 of atom `at` in the initial frame (-> u) and in the current frame x (-> v)
MDG_D void rmsd_load(const RmsdArgs& a, const float* x, int at, const mdgpu_unitcell_t& uc, float4& u, float4& v) {
    const float w = a.mass[at];
    u = pbc_wrap(make_float4(a.init_xyz[at], a.init_xyz[a.init_axis_stride + at], a.init_xyz[2 * a.init_axis_stride + at], w), uc);
    v = pbc_wrap(make_float4(x[at], x[a.frames.axis_stride + at], x[2 * a.frames.axis_stride + at], w), uc);
}

// The ordered part of _rmsd on n wrapped atoms: bond walk and centre of both sets, rotation from their cross-covariance, weighted deviation
MDG_D float rmsd_fit(float4* p0, float4* p1, uint32_t n, const int2* pairs, uint32_t n_pairs, const mdgpu_unitcell_t& uc) {
    float com0[3], com1[3];
    unwrap_com(p0, n, pairs, n_pairs, uc, com0);
    unwrap_com(p1, n, pairs, n_pairs, uc, com1);
    const M3 R = extract_rotation(cross_covariance(p0, com0, p1, com1, n));
    double d_sum = 0.0, w_sum = 0.0;
    for (uint32_t k = 0; k < n; ++k) {
        const float4 u4 = p0[k], v4 = p1[k];
        const float u[3] = { u4.x - com0[0], u4.y - com0[1], u4.z - com0[2] };
        const float v[3] = { v4.x - com1[0], v4.y - com1[1], v4.z - com1[2] };
        float d[3];   // mat3_mul_vec3 (core/md_vec_math.h:1623): (x * col0 + y * col1) + z * col2
        for (int r = 0; r < 3; ++r) d[r] = u[r] - ((R.e[0][r] * v[0] + R.e[1][r] * v[1]) + R.e[2][r] * v[2]);
        const float w = (u4.w + v4.w) * 0.5f;
        const float dd = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
        d_sum += (double)(w * dd); w_sum += (double)w;
    }
    return (float)sqrt(d_sum / w_sum);
}

__global__ void __launch_bounds__(32) k_rmsd(RmsdArgs a, int B) {
    const int f = blockIdx.x, lane = threadIdx.x;
    if (f >= B) return;
    const uint32_t n = a.n;
    const mdgpu_unitcell_t uc = a.cells[f];
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    float4* p0 = a.scratch_xyzw + (size_t)f * 2 * n;   // initial frame
    float4* p1 = p0 + n;                               // current frame
    for (uint32_t k = lane; k < n; k += 32) rmsd_load(a, x, a.idx[k], uc, p0[k], p1[k]);
    __syncwarp();
    if (lane != 0) return;
    a.out[a.frame0 + f] = rmsd_fit(p0, p1, n, a.unwrap_pairs, a.n_unwrap, uc);
}

// rmsd(selection) in <contexts> (evaluate_context md_script.c:3418): group g of idx[0] (soff[g] .. soff[g+1]) is (selection AND context g).
// One thread per (group, frame), as k_sdf_fit maps structures: a context is a residue or a molecule (a few atoms), so the thread does the whole
// ordered computation of its group. An empty group keeps the value 0 (_rmsd :4311). The unwrap pairs depend on the group's size only (the
// local-index-as-atom quirk above): group g walks group_pairs[g] = (first pair in unwrap_pairs, pair count).
__global__ void k_rmsd_groups(RmsdArgs a, int B) {
    const int f = blockIdx.y;
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.n_groups) return;
    const uint32_t beg = a.soff[g], n = a.soff[g + 1] - beg;
    float* o = a.out + (size_t)(a.frame0 + f) * a.n_groups + g;
    if (n == 0) { *o = 0.0f; return; }
    const mdgpu_unitcell_t uc = a.cells[f];
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    float4* p0 = a.scratch_xyzw + (size_t)f * 2 * a.n + beg;   // [B][initial, current][all groups' atoms], as k_rmsd
    float4* p1 = p0 + a.n;
    for (uint32_t k = 0; k < n; ++k) rmsd_load(a, x, a.idx[beg + k], uc, p0[k], p1[k]);
    const uint2 gp = a.group_pairs[g];
    *o = rmsd_fit(p0, p1, n, a.unwrap_pairs + gp.x, gp.y, uc);
}

// plane(selection) (_plane md_script_functions.inl:4755-4822): positions with unit weights, bond walk, plain centre, covariance
// (mat3_covariance_matrix_vec4 core/md_vec_math.c:101-156), eigenvectors sorted by eigenvalue (mat3_eigen :22-42); the frame's row is
// (normalised third axis, normal . centre). One warp per frame, lane 0 does the ordered part, as in k_rmsd (init_xyz is not used).
__global__ void __launch_bounds__(32) k_plane(RmsdArgs a, int B) {
    const int f = blockIdx.x, lane = threadIdx.x;
    if (f >= B) return;
    const uint32_t n = a.n;
    const mdgpu_unitcell_t uc = a.cells[f];
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    float4* p = a.scratch_xyzw + (size_t)f * n;
    if (a.pos) for (uint32_t k = lane; k < n; k += 32) { const float* q = a.pos + ((size_t)f * n + k) * 3; p[k] = make_float4(q[0], q[1], q[2], 1.0f); }   // one centre of mass per selection (coordinate_extract :1503)
    else for (uint32_t k = lane; k < n; k += 32) { const int at = a.idx[k]; p[k] = make_float4(x[at], x[a.frames.axis_stride + at], x[2 * a.frames.axis_stride + at], 1.0f); }
    __syncwarp();
    if (lane != 0) return;
    float com[3];
    unwrap_com(p, n, a.unwrap_pairs, a.n_unwrap, uc, com);
    const Eigen eg = eigen_sorted(covariance(p, n, com));
    float nrm[3] = { eg.vec.e[2][0], eg.vec.e[2][1], eg.vec.e[2][2] };   // the axis of the smallest value
    normalize3(nrm);
    float* o = a.out + (size_t)(a.frame0 + f) * 4;
    o[0] = nrm[0]; o[1] = nrm[1]; o[2] = nrm[2]; o[3] = (nrm[0] * com[0] + nrm[1] * com[1]) + nrm[2] * com[2];
}

// ------------------------------------------------------------------------------------------------- shape weights of structures
// The loop body of VIAMD's shape-space component (src/components/shapespace/shapespace.cpp:418-431) and of _shape_weights
// (md_script_functions.inl:6033-6040): xyzw (mass or 1) -> md_util_com_compute_vec4 with the cell (com_pbc_vec4 md_util.c:8063-8162) ->
// md_util_deperiodize_vec4 about that centre (:8971-9005) -> mat3_covariance_matrix_vec4 -> md_util_shape_weights (:9070-9076).
// One warp per (structure, frame): the lanes extract, lane 0 does the ordered work (float sums over the atoms in index order, double
// covariance). Row (frame0 + f) of the property holds n_struct x (linear, planar, isotropic).
__global__ void __launch_bounds__(32) k_shape_weights(ShapeArgs a, int B) {
    const int f = blockIdx.y, lane = threadIdx.x;
    const uint32_t sidx = blockIdx.x;
    if (f >= B || sidx >= a.n_struct) return;
    const uint32_t beg = a.soff[sidx], n = a.soff[sidx + 1] - beg;
    float* o = a.out + ((size_t)(a.frame0 + f) * a.n_struct + sidx) * 3;
    if (n == 0) { if (lane == 0) { o[0] = 0.f; o[1] = 0.f; o[2] = 0.f; } return; }   // count == 0: the entry keeps its zero (:6029)
    const mdgpu_unitcell_t uc = a.cells[f];
    const float* x = a.frames.xyz + (size_t)f * a.frames.frame_stride;
    float4* p = a.scratch_xyzw + (size_t)f * a.n_atoms_total + beg;
    for (uint32_t k = lane; k < n; k += 32) { const int at = a.idx[beg + k]; p[k] = make_float4(x[at], x[a.frames.axis_stride + at], x[2 * a.frames.axis_stride + at], a.use_mass ? a.mass[at] : 1.0f); }
    __syncwarp();
    if (lane != 0) return;
    float com[3];
    com_compute_vec4(p, n, uc, com);
    if (uc.flags & MDGPU_CELL_ORTHO) {
        const float ext[3] = { (float)uc.x, (float)uc.y, (float)uc.z };
        for (uint32_t k = 0; k < n; ++k) { float4 v = p[k]; v.x = deperiodize1(v.x, com[0], ext[0]); v.y = deperiodize1(v.y, com[1], ext[1]); v.z = deperiodize1(v.z, com[2], ext[2]); p[k] = v; }
    } else if (uc.flags & MDGPU_CELL_TRICLINIC) {
        float box[3][3]; cell_box(uc, box);
        for (uint32_t k = 1; k < n; ++k) {   // deperiodize_triclinic from atom 1 on (:8993)
            float4 v = p[k];
            float d[3] = { __fsub_rn(v.x, com[0]), __fsub_rn(v.y, com[1]), __fsub_rn(v.z, com[2]) };
            min_image_triclinic(d, box);
            v.x = __fadd_rn(com[0], d[0]); v.y = __fadd_rn(com[1], d[1]); v.z = __fadd_rn(com[2], d[2]); p[k] = v;
        }
    }
    const Eigen eg = eigen_sorted(covariance(p, n, com));
    const float e0 = eg.val[0], e1 = eg.val[1], e2 = eg.val[2];
    const float sc = 1.0f / ((e0 + e1) + e2);   // md_util_shape_weights md_util.c:9070-9076
    o[0] = (e0 - e1) * sc; o[1] = 2.0f * (e1 - e2) * sc; o[2] = 3.0f * e2 * sc;
}

// An ARRAY of selections as one position argument of distance / angle / dihedral / com: the centres k_arg_com_parts left in `parts`
// (weight 1 each) -> md_util_com_compute_vec4 with the frame's cell (coordinate_extract_com md_script_functions.inl:1841). One thread per frame.
__global__ void k_arg_combine(const float4* __restrict__ parts, uint32_t n_parts, const mdgpu_unitcell_t* __restrict__ cells, float* __restrict__ out /* [B][4][3] */, int arg, int B) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= B) return;
    float com[3];
    com_compute_vec4(parts + (size_t)f * n_parts, n_parts, cells[f], com);
    float* o = out + ((size_t)f * 4 + arg) * 3;
    o[0] = com[0]; o[1] = com[1]; o[2] = com[2];
}

void launch_arg_combine(const float4* d_parts, uint32_t n_parts, const mdgpu_unitcell_t* d_cells, float* d_out, int arg, int B, cudaStream_t s) {
    if (B <= 0 || !n_parts) return;
    k_arg_combine<<<(B + 63) / 64, 64, 0, s>>>(d_parts, n_parts, d_cells, d_out, arg, B);
    note_launch("k_arg_combine", s);
}

void launch_shape_weights(const ShapeArgs& a, int B, cudaStream_t s) {
    if (!a.n_struct || B <= 0) return;
    k_shape_weights<<<dim3(a.n_struct, (unsigned)B), 32, 0, s>>>(a, B);
    note_launch("k_shape_weights", s);
}

void launch_plane(const RmsdArgs& a, int B, cudaStream_t s) {
    if (!a.n || B <= 0) return;
    k_plane<<<B, 32, 0, s>>>(a, B);
    note_launch("k_plane", s);
}

void launch_rmsd(const RmsdArgs& a, int B, cudaStream_t s) {
    if (!a.n || B <= 0) return;   // empty selection: the property stays 0 (:4311)
    k_rmsd<<<B, 32, 0, s>>>(a, B);
    note_launch("k_rmsd", s);
}

void launch_rmsd_groups(const RmsdArgs& a, int B, cudaStream_t s) {
    if (!a.n_groups || B <= 0) return;
    k_rmsd_groups<<<dim3((a.n_groups + 63) / 64, (unsigned)B), 64, 0, s>>>(a, B);
    note_launch("k_rmsd_groups", s);
}

void launch_sdf(const SdfArgs& a, int B, bool tri, cudaStream_t s) {
    k_sdf_ref0<<<(B + 31) / 32, 32, 0, s>>>(a, B);
    note_launch("k_sdf_ref0", s);
    dim3 g1((a.n_struct + 63) / 64, B);
    k_sdf_fit<<<g1, 64, 0, s>>>(a, B);
    note_launch("k_sdf_fit", s);
    dim3 g2((a.n_struct + SDF_WARPS - 1) / SDF_WARPS, B);
    if (tri) k_sdf_scatter<true, SDF_MIN_CTAS><<<g2, SDF_WARPS * 32, 0, s>>>(a, B); else k_sdf_scatter<false, SDF_MIN_CTAS><<<g2, SDF_WARPS * 32, 0, s>>>(a, B);
    note_launch("k_sdf_scatter", s);
}

}  // namespace mdg
