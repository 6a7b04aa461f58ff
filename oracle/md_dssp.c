/* md_dssp.c — TEST INFRASTRUCTURE: plain-C restatement of the reference's secondary-structure inference for one frame
 * (md_util_backbone_secondary_structure_infer -> dssp(), md_util.c:2047-2550).
 *
 * It includes md_oracle.c for the spatial acceleration structure (acc_init = md_spatial_acc_init) and is built on its own by
 * tests/dssp_oracle.py (gcc, strict IEEE flags) into build/libdssp.so. The structure follows the reference step by step: the candidate pairs come
 * from the internal pair walk of the cell grid in the reference's order, each pair's two H-bond energies are evaluated in that order, bridges are
 * recorded in candidate order and ladders are grown by exact-key lookup. The device library reaches the same rows by another route (acceptors
 * scanned in ascending order per donor, bridges derived from the recorded bonds, ladders grown per bridge); equality of the two on the fixtures is
 * part of what the tests check.
 *
 * Two points differ from the reference, on purpose (include/mdgpu.h, MDGPU_OP_SECONDARY_STRUCTURE):
 *  - the turn masks and flags start at zero (the reference takes them from uncleared temporary memory, md_util.c:2071, 2085);
 *  - vec4_rsqrt (rsqrtps + one Newton step, host dependent) is 1.0f / sqrtf(d2).
 */
#include "md_oracle.c"

enum { SS_TURN = 1, SS_BEND = 2, SS_H310 = 4, SS_HALPHA = 8, SS_HPI = 16, SS_SHEET = 32, SS_BRIDGE = 64 };
enum { MDO_SS_COIL = 1, MDO_SS_TURN = 2, MDO_SS_BEND = 3, MDO_SS_H310 = 4, MDO_SS_HALPHA = 5, MDO_SS_HPI = 6, MDO_SS_SHEET = 7, MDO_SS_BRIDGE = 8 };

typedef struct { float N[3], CA[3], C[3], O[3], H[3]; } ss_res_t;
typedef struct { uint32_t idx; float e; } ss_hb_t;
typedef struct { ss_hb_t acc[2]; } ss_bonds_t;
typedef struct { uint32_t i, j; uint64_t key; } ss_bridge_t;

/* vec4 arithmetic with w = 0: vec4_dot = (x + y) + (z + w) (md_mm_reduce_add_ps), vec4_normalize multiplies by 1 / sqrtf(mag2) above 1e-5 */
static inline float ss_dot(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + (a[2] * b[2] + 0.0f); }
static inline float ss_dist2(const float a[3], const float b[3]) { const float d[3] = { a[0] - b[0], a[1] - b[1], a[2] - b[2] }; return ss_dot(d, d); }
static inline void ss_normalize(float v[3]) {
    const float m2 = ss_dot(v, v);
    if (m2 > 1.0e-5f) { const float s = 1.0f / sqrtf(m2); v[0] *= s; v[1] *= s; v[2] *= s; }
}
/* estimate_HN md_util.c:1974-1979 */
static void ss_estimate_hn(float H[3], const float N[3], const float CA[3], const float Cp[3]) {
    float U[3] = { N[0] - CA[0], N[1] - CA[1], N[2] - CA[2] }, V[3] = { N[0] - Cp[0], N[1] - Cp[1], N[2] - Cp[2] };
    ss_normalize(U); ss_normalize(V);
    float W[3] = { U[0] + V[0], U[1] + V[1], U[2] + V[2] }; ss_normalize(W);
    for (int k = 0; k < 3; ++k) H[k] = N[k] + W[k] * 1.01f;
}

/* calc_hbond_energy md_util.c:1910-1972 (the don[] half is never read): the energy of donor d and acceptor a, or 0 when above -0.5 */
static float ss_energy(const ss_res_t* don, const ss_res_t* acc) {
    const float d2[4] = { ss_dist2(don->N, acc->O), ss_dist2(don->H, acc->C), ss_dist2(don->N, acc->C), ss_dist2(don->H, acc->O) };
    float e;
    if (d2[0] < 0.25f || d2[1] < 0.25f || d2[2] < 0.25f || d2[3] < 0.25f) e = -9.9f;
    else {
        const float r0 = 1.0f / sqrtf(d2[0]), r1 = 1.0f / sqrtf(d2[1]), r2 = 1.0f / sqrtf(d2[2]), r3 = 1.0f / sqrtf(d2[3]);
        e = 27.888f * ((r0 + r1) + (-r2 + -r3));
    }
    if (e > -0.5f) return 0.0f;
    return e > -9.9f ? e : -9.9f;
}
static void ss_record(ss_bonds_t* b, uint32_t acc_idx, float e) {
    if (e < b->acc[0].e) { b->acc[1] = b->acc[0]; b->acc[0].idx = acc_idx; b->acc[0].e = e; }
    else if (e < b->acc[1].e) { b->acc[1].idx = acc_idx; b->acc[1].e = e; }
}
static void ss_pair_energies(ss_bonds_t* hb, const ss_res_t* rc, uint32_t don, uint32_t acc) {
    const float e = ss_energy(&rc[don], &rc[acc]);
    if (e != 0.0f) ss_record(&hb[don], acc, e);
}
/* dssp_test_bond md_util.c:1991-1995 */
static inline bool ss_bond(const ss_bonds_t* hb, uint32_t acceptor, uint32_t donor) {
    return (hb[donor].acc[0].idx == acceptor && hb[donor].acc[0].e < -0.5f) || (hb[donor].acc[1].idx == acceptor && hb[donor].acc[1].e < -0.5f);
}

/* distance_squared_ort_256 / _tri_256 (core/md_spatial_acc.c:503-529) in fractional coordinates */
static inline float ss_d2(const acc_t* acc, bool tri, float dx, float dy, float dz) {
    float d2 = fmaf(acc->G00, dx * dx, fmaf(acc->G11, dy * dy, acc->G22 * (dz * dz)));
    if (tri) d2 = d2 + fmaf(acc->H01, dx * dy, fmaf(acc->H02, dx * dz, acc->H12 * (dy * dz)));
    return d2;
}

/* md_spatial_acc_for_each_internal_pair_within_cutoff (core/md_spatial_acc.c:1089-1500): self cell j > i, then the forward neighbours
 * (generate_forward_neighbors4 :445-466) of every non-empty cell in z, y, x order; an orthorhombic grid skips wraps of non-periodic axes. */
typedef void (*ss_pair_fn)(uint32_t i, uint32_t j, void* user);
static void acc_internal_pairs(const acc_t* acc, double cutoff, ss_pair_fn cb, void* user) {
    if (acc->num_elems == 0) return;
    int ncell[3];
    for (int k = 0; k < 3; ++k) ncell[k] = (int)ceil(cutoff * (double)acc->inv_cell_ext[k] * acc->cell_dim[k]);
    for (int k = 0; k < 3; ++k) if (2 * ncell[k] + 1 > 5) return;
    const float r2 = calc_r2(cutoff);
    const bool tri = (acc->flags & MDO_CELL_TRICLINIC) != 0;
    const int cd[3] = { (int)acc->cell_dim[0], (int)acc->cell_dim[1], (int)acc->cell_dim[2] };
    int fwd[125][3]; int nf = 0;
    for (int dz = 0; dz <= ncell[2]; ++dz) for (int dy = -ncell[1]; dy <= ncell[1]; ++dy) for (int dx = -ncell[0]; dx <= ncell[0]; ++dx) {
        if (dx == 0 && dy == 0 && dz == 0) continue;
        if (dz > 0 || (dz == 0 && dy > 0) || (dz == 0 && dy == 0 && dx > 0)) { fwd[nf][0] = dx; fwd[nf][1] = dy; fwd[nf][2] = dz; ++nf; }
    }
    for (int cz = 0; cz < cd[2]; ++cz) for (int cy = 0; cy < cd[1]; ++cy) for (int cx = 0; cx < cd[0]; ++cx) {
        const size_t ci = ((size_t)cz * cd[1] + cy) * cd[0] + cx;
        const uint32_t oi = acc->cell_off[ci], li = acc->cell_off[ci + 1] - oi;
        if (!li) continue;
        for (uint32_t a = 0; a + 1 < li; ++a)
            for (uint32_t b = a + 1; b < li; ++b) {
                const float d2 = ss_d2(acc, tri, acc->ex[oi + a] - acc->ex[oi + b], acc->ey[oi + a] - acc->ey[oi + b], acc->ez[oi + a] - acc->ez[oi + b]);
                if (d2 <= r2) cb(acc->eidx[oi + a], acc->eidx[oi + b], user);
            }
        const int c[3] = { cx, cy, cz };
        for (int n = 0; n < nf; ++n) {
            int nv[3]; float sh[3]; bool skip = false;
            for (int k = 0; k < 3; ++k) {
                nv[k] = c[k] + fwd[n][k];
                const bool up = nv[k] > cd[k] - 1, lo = nv[k] < 0;
                if ((up || lo) && !tri && !(acc->flags & (MDO_CELL_PBC_X << k))) skip = true;
                if (lo) nv[k] += cd[k];
                if (up) nv[k] -= cd[k];
                sh[k] = (float)((lo ? 1 : 0) - (up ? 1 : 0));
            }
            if (skip) continue;
            const size_t cj = ((size_t)nv[2] * cd[1] + nv[1]) * cd[0] + nv[0];
            const uint32_t oj = acc->cell_off[cj], lj = acc->cell_off[cj + 1] - oj;
            for (uint32_t a = 0; a < li; ++a) {
                const float fx = acc->ex[oi + a] + sh[0], fy = acc->ey[oi + a] + sh[1], fz = acc->ez[oi + a] + sh[2];
                for (uint32_t b = 0; b < lj; ++b) {
                    const float d2 = ss_d2(acc, tri, fx - acc->ex[oj + b], fy - acc->ey[oj + b], fz - acc->ez[oj + b]);
                    if (d2 <= r2) cb(acc->eidx[oi + a], acc->eidx[oj + b], user);
                }
            }
        }
    }
}

typedef struct { const uint32_t* range_id; const ss_res_t* rc; ss_bonds_t* hb; ss_bridge_t* cand; size_t ncand, cap; } ss_walk_t;

/* dssp_hbond_energy_cb md_util.c:2021-2045 */
static void ss_walk_pair(uint32_t a, uint32_t b, void* user) {
    ss_walk_t* w = user;
    const uint32_t i = MINV(a, b), j = MAXV(a, b);
    const bool same = w->range_id[i] == w->range_id[j]; const int d = (int)j - (int)i;
    if (same && d <= 1) return;
    ss_pair_energies(w->hb, w->rc, i, j);
    ss_pair_energies(w->hb, w->rc, j, i);
    if (same && d <= 2) return;
    if (w->ncand == w->cap) { w->cap = w->cap ? 2 * w->cap : 1024; w->cand = realloc(w->cand, w->cap * sizeof(ss_bridge_t)); }
    w->cand[w->ncand].i = i; w->cand[w->ncand].j = j; w->cand[w->ncand].key = 0; ++w->ncand;
}

static int ss_find(const ss_bridge_t* br, size_t nb, uint32_t i, uint32_t j, uint64_t key) {
    for (size_t k = 0; k < nb; ++k) if (br[k].i == i && br[k].j == j && br[k].key == key) return (int)k;
    return -1;
}

/* One frame. atoms[S][5] = N, CA, C, O, HN (HN -1: estimated); range_off[R + 1] ascending from 0 to S. out[S] receives md_secondary_structure_t
 * codes. shuffle_seed != 0 permutes the recorded bridges before the ladders are grown (the rows must not change). Returns 0, -1 for malformed
 * input, -3 when a periodic axis of the frame's grid is too narrow for the candidate walk to visit each pair once, or the cell is triclinic
 * without periodicity on all axes or degenerate. */
int mdo_dssp(int32_t* out, const float* x, const float* y, const float* z, const mdo_unitcell_t* cell, const int32_t* atoms, size_t S,
             const uint32_t* range_off, size_t R, uint64_t shuffle_seed) {
    if (!S || !R || range_off[0] != 0 || range_off[R] != S) return -1;
    for (size_t r = 0; r < R; ++r) if (range_off[r] > range_off[r + 1]) return -1;
    const uint32_t flags = cell ? cell->flags : 0;
    if ((flags & MDO_CELL_TRICLINIC) && (flags & MDO_CELL_PBC_ALL) != MDO_CELL_PBC_ALL) return -3;

    ss_res_t* rc = calloc(S, sizeof(ss_res_t)); ss_bonds_t* hb = calloc(S, sizeof(ss_bonds_t)); uint32_t* rid = calloc(S, 4);
    uint8_t* turn = calloc(S, 1); uint32_t* fl = calloc(S, 4); float* ca = calloc(3 * S, 4);
    for (size_t r = 0; r < R; ++r) for (uint32_t i = range_off[r]; i < range_off[r + 1]; ++i) rid[i] = (uint32_t)r;
    for (size_t r = 0; r < R; ++r) for (uint32_t i = range_off[r]; i < range_off[r + 1]; ++i) {
        const int32_t* q = atoms + 5 * (size_t)i;
        float* dst[4] = { rc[i].N, rc[i].CA, rc[i].C, rc[i].O };
        for (int k = 0; k < 4; ++k) { dst[k][0] = x[q[k]]; dst[k][1] = y[q[k]]; dst[k][2] = z[q[k]]; }
        if (q[4] >= 0) { rc[i].H[0] = x[q[4]]; rc[i].H[1] = y[q[4]]; rc[i].H[2] = z[q[4]]; }
        else if (i > range_off[r]) ss_estimate_hn(rc[i].H, rc[i].N, rc[i].CA, rc[i - 1].C);
        else {   /* estimate_HN_term :1981-1989: C_prev = N + (CA - C) */
            const float cp[3] = { rc[i].N[0] + (rc[i].CA[0] - rc[i].C[0]), rc[i].N[1] + (rc[i].CA[1] - rc[i].C[1]), rc[i].N[2] + (rc[i].CA[2] - rc[i].C[2]) };
            ss_estimate_hn(rc[i].H, rc[i].N, rc[i].CA, cp);
        }
        ca[i] = rc[i].CA[0]; ca[S + i] = rc[i].CA[1]; ca[2 * S + i] = rc[i].CA[2];
    }
    /* candidate walk over the CA positions with the frame's cell (md_spatial_acc_init(&acc, ca, 9.0, cell) :2120-2122) */
    const stream_t st = { ca, ca + S, ca + 2 * S, NULL, NULL, S };
    acc_t acc; acc_init(&acc, &st, 9.0, cell, false);
    if ((flags & MDO_CELL_TRICLINIC) && acc.num_elems == 0) { acc_free(&acc); free(rc); free(hb); free(rid); free(turn); free(fl); free(ca); return -3; }
    for (int k = 0; k < 3; ++k) {
        const int nc = (int)ceil(9.0 * (double)acc.inv_cell_ext[k] * acc.cell_dim[k]);
        if ((flags & (MDO_CELL_PBC_X << k)) && (nc > 2 || (int)acc.cell_dim[k] < 2 * nc + 1)) { acc_free(&acc); free(rc); free(hb); free(rid); free(turn); free(fl); free(ca); return -3; }
    }
    ss_walk_t w = { rid, rc, hb, NULL, 0, 0 };
    acc_internal_pairs(&acc, 9.0, ss_walk_pair, &w);
    acc_free(&acc);

    /* helices, turns, bends per range :2155-2227 */
    for (size_t r = 0; r < R; ++r) {
        const uint32_t beg = range_off[r], end = range_off[r + 1];
        for (uint32_t i = beg; i < end; ++i) {
            if (i + 3 < end && ss_bond(hb, i, i + 3)) turn[i] |= 1;
            if (i + 4 < end && ss_bond(hb, i, i + 4)) turn[i] |= 2;
            if (i + 5 < end && ss_bond(hb, i, i + 5)) turn[i] |= 4;
        }
        for (uint32_t i = beg; i + 1 < end; ++i) {
            const uint8_t a = turn[i], b = turn[i + 1];
            if ((a & 1) && (b & 1)) for (uint32_t k = i + 1; k <= MINV(i + 3, end - 1); ++k) fl[k] |= SS_H310;
            if ((a & 2) && (b & 2)) for (uint32_t k = i + 1; k <= MINV(i + 4, end - 1); ++k) fl[k] |= SS_HALPHA;
            if ((a & 4) && (b & 4)) for (uint32_t k = i + 1; k <= MINV(i + 5, end - 1); ++k) fl[k] |= SS_HPI;
            if (a) { const uint32_t len = (a & 4) ? 5 : (a & 2) ? 4 : 3; for (uint32_t k = i + 1; k <= MINV(i + len, end - 1); ++k) fl[k] |= SS_TURN; }
        }
        for (uint32_t i = beg + 2; i + 2 < end; ++i) {
            const float v1[3] = { rc[i - 2].CA[0] - rc[i].CA[0], rc[i - 2].CA[1] - rc[i].CA[1], rc[i - 2].CA[2] - rc[i].CA[2] };
            const float v2[3] = { rc[i + 2].CA[0] - rc[i].CA[0], rc[i + 2].CA[1] - rc[i].CA[1], rc[i + 2].CA[2] - rc[i].CA[2] };
            const float c[3] = { v1[1] * v2[2] - v1[2] * v2[1], v1[2] * v2[0] - v1[0] * v2[2], v1[0] * v2[1] - v1[1] * v2[0] };
            const double angle = atan2f(sqrtf(ss_dot(c, c)), ss_dot(v1, v2));   /* vec4_angle */
            if (angle < 70.0 * (3.14159265358979323846 / 180.0)) for (int k = -2; k <= 2; ++k) fl[i + k] |= SS_BEND;
        }
    }

    /* bridges from the sheet candidates, in candidate order :2248-2316 */
    ss_bridge_t* br = malloc((w.ncand + 1) * sizeof(ss_bridge_t)); size_t nb = 0;
#define SAME(a, b) (rid[(a)] == rid[(b)])
    for (size_t c = 0; c < w.ncand; ++c) {
        const uint32_t i = w.cand[c].i, j = w.cand[c].j;
        const bool im = i > 0 && SAME(i - 1, i), ip = i + 1 < S && SAME(i + 1, i), jm = j > 0 && SAME(j - 1, j), jp = j + 1 < S && SAME(j + 1, j);
        bool anti = false, par = false;
        if (ss_bond(hb, i, j) && ss_bond(hb, j, i)) anti = true;
        else if (im && ip && jm && jp && ss_bond(hb, i - 1, j + 1) && ss_bond(hb, j - 1, i + 1)) anti = true;
        if (!anti) {
            if (im && ip && ss_bond(hb, i - 1, j) && ss_bond(hb, j, i + 1)) par = true;
            if (!par && jm && jp && ss_bond(hb, j - 1, i) && ss_bond(hb, i, j + 1)) par = true;
        }
        if (!anti && !par) continue;
        const uint64_t packed = (uint64_t)MINV(rid[i], rid[j]) << 32 | MAXV(rid[i], rid[j]);
        br[nb].i = i; br[nb].j = j; br[nb].key = (uint64_t)(par ? 1 : 0) << 63 | packed; ++nb;
        fl[i] |= SS_BRIDGE; fl[j] |= SS_BRIDGE;
    }
#undef SAME
    if (shuffle_seed) {   /* Fisher-Yates with xorshift64 */
        uint64_t s = shuffle_seed;
        for (size_t k = nb; k > 1; --k) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; const size_t m = (size_t)(s % k); const ss_bridge_t t = br[k - 1]; br[k - 1] = br[m]; br[m] = t; }
    }
    /* ladders by exact-key lookup, whatever `used` says :2390-2453 */
    bool* used = calloc(nb + 1, 1);
    for (size_t b = 0; b < nb; ++b) {
        if (used[b]) continue;
        used[b] = true;
        uint32_t i_min = br[b].i, i_max = br[b].i, j_min = br[b].j, j_max = br[b].j;
        const uint64_t key = br[b].key; const bool par = (key >> 63) != 0;
        for (bool grew = true; grew; ) {
            grew = false;
            const uint32_t n1i = i_max + 1, n1j = par ? j_max + 1 : j_min - 1, n2i = i_min - 1, n2j = par ? j_min - 1 : j_max + 1;
            const int f1 = ss_find(br, nb, n1i, n1j, key), f2 = ss_find(br, nb, n2i, n2j, key);
            const int f = f1 >= 0 ? f1 : f2;
            if (f >= 0) {
                used[f] = true;
                i_min = MINV(i_min, br[f].i); i_max = MAXV(i_max, br[f].i); j_min = MINV(j_min, br[f].j); j_max = MAXV(j_max, br[f].j);
                grew = true;
            }
        }
        if (i_max - i_min + 1 >= 3 || j_max - j_min + 1 >= 3) {
            for (uint32_t k = i_min; k <= i_max; ++k) fl[k] |= SS_SHEET;
            for (uint32_t k = j_min; k <= j_max; ++k) fl[k] |= SS_SHEET;
        }
    }
    /* priority :2523-2547 */
    for (size_t i = 0; i < S; ++i) {
        const uint32_t f = fl[i];
        out[i] = (f & SS_HPI) ? MDO_SS_HPI : (f & SS_HALPHA) ? MDO_SS_HALPHA : (f & SS_H310) ? MDO_SS_H310 : (f & SS_SHEET) ? MDO_SS_SHEET
               : (f & SS_BRIDGE) ? MDO_SS_BRIDGE : (f & SS_TURN) ? MDO_SS_TURN : (f & SS_BEND) ? MDO_SS_BEND : MDO_SS_COIL;
    }
    free(used); free(br); free(w.cand); free(rc); free(hb); free(rid); free(turn); free(fl); free(ca);
    return 0;
}
