/* md_porosity.c — TEST INFRASTRUCTURE: plain-C restatement of porosity(selection) for one frame (_porosity, md_script_functions.inl:5858-6003).
 *
 * It includes md_oracle.c for the restatements it shares with the other procedures (com_compute_v4 = md_util_com_compute_vec4, deperiodize1 =
 * vec4_deperiodize_ortho) and is built on its own by tests/porosity_oracle.py (gcc, strict IEEE flags) into build/libporosity.so.
 *
 * One difference from the reference, on purpose: the reference takes the centre-of-mass weights and the box padding from rad[atom index] of an
 * array that holds the radii of atoms 0 .. n-1 only (:5906-5912), which is defined only for a selection that is a prefix of the atoms. Here each
 * selected atom's own radius is used, as the reference's voxel loop does (:5946); for prefix selections both agree.
 */
#include "md_oracle.c"

/* Returns 0 and fills the outputs, or 1 when the value is 0 without a grid (triclinic cell of the frame, empty selection).
 * out_tests: sphere-voxel tests the reference's loop executes (the voxels of every sphere's clamped index box). */
int mdo_porosity(const float* x, const float* y, const float* z, const float* radius, const int32_t* idx, size_t n, const mdo_unitcell_t* cell,
                 float* out_value, float out_com[3], float out_bmin[3], float out_bmax[3], int32_t out_dim[3], uint64_t* out_set, uint64_t* out_tests) {
    *out_value = 0.0f; *out_set = 0; *out_tests = 0;
    for (int c = 0; c < 3; ++c) { out_com[c] = out_bmin[c] = out_bmax[c] = 0.0f; out_dim[c] = 0; }
    if ((cell->flags & MDO_CELL_TRICLINIC) || n == 0) return 1;
    v4* p = malloc(sizeof(v4) * n);
    for (size_t k = 0; k < n; ++k) { const int32_t a = idx[k]; p[k][0] = x[a]; p[k][1] = y[a]; p[k][2] = z[a]; p[k][3] = radius[a]; }
    float com[3];
    com_compute_v4(com, p, n, cell);                    /* md_util_com_compute_vec4(xyzr, 0, count, cell) */
    if (cell->flags & MDO_CELL_ORTHO) {                 /* md_util_deperiodize_vec4 */
        const float ext[3] = { (float)cell->x, (float)cell->y, (float)cell->z };
        for (size_t k = 0; k < n; ++k) for (int a = 0; a < 3; ++a) p[k][a] = deperiodize1(p[k][a], com[a], ext[a]);
    }
    float bmin[3] = { FLT_MAX, FLT_MAX, FLT_MAX }, bmax[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };   /* md_util_aabb_compute_vec4 */
    for (size_t k = 0; k < n; ++k) for (int a = 0; a < 3; ++a) {
        const float lo = p[k][a] - p[k][3], hi = p[k][a] + p[k][3];
        bmin[a] = lo < bmin[a] ? lo : bmin[a]; bmax[a] = hi > bmax[a] ? hi : bmax[a];
    }
    float ext[3];
    for (int a = 0; a < 3; ++a) { const float e = bmax[a] - bmin[a]; ext[a] = e > 1.0f ? e : 1.0f; }
    const float max_ext = ext[0] > (ext[1] > ext[2] ? ext[1] : ext[2]) ? ext[0] : (ext[1] > ext[2] ? ext[1] : ext[2]);
    const float t = max_ext / 512;
    int dim[3]; float d[3];
    for (int a = 0; a < 3; ++a) { const int v = (int)(ext[a] / t); dim[a] = v > 1 ? v : 1; d[a] = ext[a] / (float)dim[a]; }
    const size_t num_bits = (size_t)dim[0] * (size_t)dim[1] * (size_t)dim[2];
    uint64_t* bits = calloc((num_bits + 63) / 64, sizeof(uint64_t));
    uint64_t tests = 0;
    for (size_t i = 0; i < n; ++i) {
        const float px = p[i][0], py = p[i][1], pz = p[i][2], r = p[i][3];
        int lo[3], hi[3]; const float pc[3] = { px, py, pz };
        for (int a = 0; a < 3; ++a) {
            lo[a] = (int)floorf((pc[a] - r - bmin[a]) / d[a]); hi[a] = (int)floorf((pc[a] + r - bmin[a]) / d[a]);
            lo[a] = lo[a] < 0 ? 0 : (lo[a] > dim[a] - 1 ? dim[a] - 1 : lo[a]); hi[a] = hi[a] < 0 ? 0 : (hi[a] > dim[a] - 1 ? dim[a] - 1 : hi[a]);
        }
        const float r2 = r * r;
        tests += (uint64_t)(hi[0] - lo[0] + 1) * (uint64_t)(hi[1] - lo[1] + 1) * (uint64_t)(hi[2] - lo[2] + 1);
        for (int iz = lo[2]; iz <= hi[2]; ++iz) {
            const float dzv = (bmin[2] + ((float)iz + 0.5f) * d[2]) - pz;
            for (int iy = lo[1]; iy <= hi[1]; ++iy) {
                const float dyv = (bmin[1] + ((float)iy + 0.5f) * d[1]) - py;
                for (int ix = lo[0]; ix <= hi[0]; ++ix) {
                    const float dxv = (bmin[0] + ((float)ix + 0.5f) * d[0]) - px;
                    if (fmaf(dxv, dxv, fmaf(dyv, dyv, dzv * dzv)) <= r2) {
                        const size_t b = (size_t)iz * dim[0] * dim[1] + (size_t)iy * dim[0] + (size_t)ix;
                        bits[b >> 6] |= 1ull << (b & 63);
                    }
                }
            }
        }
    }
    uint64_t set = 0;
    for (size_t w = 0; w < (num_bits + 63) / 64; ++w) set += (uint64_t)__builtin_popcountll(bits[w]);
    *out_value = set ? (float)(((double)num_bits - (double)set) / (double)num_bits) : 0.0f;
    *out_set = set; *out_tests = tests;
    for (int a = 0; a < 3; ++a) { out_com[a] = com[a]; out_bmin[a] = bmin[a]; out_bmax[a] = bmax[a]; out_dim[a] = dim[a]; }
    free(bits); free(p);
    return 0;
}
