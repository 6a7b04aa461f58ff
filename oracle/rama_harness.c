/* rama_harness.c — TEST INFRASTRUCTURE: VIAMD's Ramachandran density task driven through the UNMODIFIED reference.
 *
 * Nothing under viamd_b200/ may link, import or execute this. It is linked (oracle/rama.mk) against the objects oracle/Makefile compiles from the
 * sources under /root/reference/ext/mdlib and against rama_blur.cpp, which compiles the application's own blur cut out of ramachandran.cpp;
 * outputs go to oracle/_ref/. It generates tests/golden/rama.npz (tests/golden/make_golden_rama.py) and times the task on one CPU thread.
 *
 * usage:
 *   rama_harness rama --sys F --traj SPEC [--frames B:E] [--range B:E] [--sigma S] --out O
 *   rama_harness rama --time F:S [--repeat R]
 * traj SPEC as for ref_harness (raw:<file> | synthwater:<n>:<seed>:<nframes> | sys).
 */
#include <md_system.h>
#include <md_trajectory.h>
#include <md_gro.h>
#include <md_pdb.h>
#include <md_util.h>
#include <md_xtc.h>
#include <core/md_allocator.h>
#include <core/md_arena_allocator.h>
#include <core/md_str.h>
#include <core/md_os.h>
#include <core/md_log.h>

#include "harness_common.h"

static void wr(FILE* f, const void* p, size_t n) { if (fwrite(p, 1, n, f) != n) { perror("fwrite"); exit(3); } }
static void wr_i64(FILE* f, int64_t v) { wr(f, &v, 8); }
static void wr_u64(FILE* f, uint64_t v) { wr(f, &v, 8); }

/* VIAMD's Ramachandran density task (src/components/ramachandran/ramachandran.cpp:1277-1370). The backbone angles of every frame come from
 * md_util_backbone_angles_compute as in mode_backbone, the four class lists from segment.rama_type (general, glycine, proline, pre-proline, as the
 * component collects them, :636-643); the accumulation loop of the task is restated below and the map is blurred by the reference's own
 * blur_density_gaussian (rama_blur.cpp). Frames [B,E) of the trajectory are read; --range B:E (relative to them) and --sigma choose the task's inputs.
 * MDRAMADN | u64 F | u64 nseg | i32 atoms[nseg][5] | f32 angles[F][nseg][2] | u32 class_count[4] | u32 class_idx[...] | i64 beg, end | f32 sigma
 *          | f32 tex[512][512][4] | f32 sums[4]
 * --time F:S instead times the task on one thread for F frames x S segments of seeded angles (no system needed). */
enum { RAMA_DIM = 512 };
extern void ref_rama_blur_density_gaussian(float* rgba, int dim, float sigma);

static void rama_accumulate(float* tex, double sum[4], const md_backbone_angles_t* ang, size_t frame_stride, uint32_t* const cls[4], const uint32_t ncls[4],
                            size_t beg, size_t end) {
    const float scale = 1.0f / (2.0f * PI), offset = 0.5f;   /* PI is a double literal (md_common.h:157): the scale is (float)(1 / 2pi) */
    for (size_t f = beg; f < end; ++f) {
        for (int c = 0; c < 4; ++c) {
            for (uint32_t i = 0; i < ncls[c]; ++i) {
                const md_backbone_angles_t a = ang[f * frame_stride + cls[c][i]];
                if (a.phi == 0 && a.psi == 0) continue;   /* segments without angles */
                const float u = a.phi * scale + offset, v = a.psi * scale + offset;
                const uint32_t x = (uint32_t)(u * (float)RAMA_DIM) & (RAMA_DIM - 1), y = (uint32_t)(v * (float)RAMA_DIM) & (RAMA_DIM - 1);
                tex[((size_t)y * RAMA_DIM + x) * 4 + c] += 1.0f;
                sum[c] += 1.0;
            }
        }
    }
}

static uint64_t rama_rng(uint64_t* s) { *s ^= *s << 13; *s ^= *s >> 7; *s ^= *s << 17; return *s; }
static float rama_unit(uint64_t* s) { return (float)((rama_rng(s) >> 40) + 1) * (1.0f / 16777217.0f); }   /* (0, 1) */

/* timing: F x S angles drawn around the helix (-63, -43 deg) and sheet (-120, 130 deg) basins (45 % each, sd 12 deg) and uniform (10 %), classes
 * S - 3 * S / 16 general, S / 16 glycine, S / 16 proline, S / 16 pre-proline; the full range and the first 10 % of it at sigma = 5, and the blur alone */
static int mode_rama_time(int argc, char** argv) {
    long F = 0, S = 0; if (!parse_range(arg_val(argc, argv, "--time", NULL), &F, &S) || F <= 0 || S < 16) { fprintf(stderr, "--time F:S\n"); return 2; }
    const int R = atoi(arg_val(argc, argv, "--repeat", "3"));
    md_backbone_angles_t* ang = malloc((size_t)F * S * sizeof(md_backbone_angles_t)); float* tex = malloc(sizeof(float) * RAMA_DIM * RAMA_DIM * 4);
    if (!ang || !tex) { fprintf(stderr, "out of memory for %ld x %ld angles\n", F, S); return 2; }
    uint64_t st = 0x9E3779B97F4A7C15ull; const float deg = (float)(PI / 180.0);
    for (size_t i = 0; i < (size_t)F * S; ++i) {
        const float r = rama_unit(&st), g1 = sqrtf(-2.0f * logf(rama_unit(&st))) * cosf(6.2831853f * rama_unit(&st)), g2 = sqrtf(-2.0f * logf(rama_unit(&st))) * cosf(6.2831853f * rama_unit(&st));
        float phi, psi;
        if (r < 0.45f) { phi = (-63.0f + 12.0f * g1) * deg; psi = (-43.0f + 12.0f * g2) * deg; }
        else if (r < 0.9f) { phi = (-120.0f + 12.0f * g1) * deg; psi = (130.0f + 12.0f * g2) * deg; }
        else { phi = (rama_unit(&st) * 2.0f - 1.0f) * (float)PI; psi = (rama_unit(&st) * 2.0f - 1.0f) * (float)PI; }
        ang[i].phi = phi; ang[i].psi = psi;
    }
    uint32_t ncls[4] = { (uint32_t)(S - 3 * (S / 16)), (uint32_t)(S / 16), (uint32_t)(S / 16), (uint32_t)(S / 16) }; uint32_t* cls[4];
    for (int c = 0, k = 0; c < 4; ++c) { cls[c] = malloc(sizeof(uint32_t) * ncls[c]); for (uint32_t i = 0; i < ncls[c]; ++i) cls[c][i] = (uint32_t)k++; }
    double best[3] = { 1e300, 1e300, 1e300 }; double chk = 0;
    for (int r = 0; r < R; ++r) {
        for (int w = 0; w < 2; ++w) {
            const size_t end = w == 0 ? (size_t)F : (size_t)F / 10;
            memset(tex, 0, sizeof(float) * RAMA_DIM * RAMA_DIM * 4); double sum[4] = { 0, 0, 0, 0 };
            const double t0 = now_s(); rama_accumulate(tex, sum, ang, (size_t)S, cls, ncls, 0, end); ref_rama_blur_density_gaussian(tex, RAMA_DIM, 5.0f);
            const double dt = now_s() - t0; if (dt < best[w]) best[w] = dt; chk = sum[0] + tex[(256 * RAMA_DIM + 256) * 4];
        }
        const double t0 = now_s(); ref_rama_blur_density_gaussian(tex, RAMA_DIM, 5.0f); const double dt = now_s() - t0; if (dt < best[2]) best[2] = dt;
    }
    printf("{\"frames\": %ld, \"segments\": %ld, \"threads\": 1, \"repeat\": %d, \"sigma\": 5.0, \"full_s\": %.6f, \"range10_s\": %.6f, \"blur_s\": %.6f, \"samples_per_s_full\": %.1f, \"checksum\": %.3f}\n",
           F, S, R, best[0], best[1], best[2], (double)F * S / best[0], chk);
    return 0;
}

static int mode_rama(int argc, char** argv) {
    if (arg_val(argc, argv, "--time", NULL)) return mode_rama_time(argc, argv);
    md_allocator_i* alloc = md_vm_arena_create(GIGABYTES(8));
    md_system_t sys; if (!load_system(&sys, arg_val(argc, argv, "--sys", ""), alloc)) return 2;
    md_trajectory_i traj = {0}; mem_traj_t mt;
    if (!make_traj(&traj, &mt, arg_val(argc, argv, "--traj", "sys"), &sys)) return 2;
    long b = 0, e = (long)md_trajectory_num_frames(&traj); parse_range(arg_val(argc, argv, "--frames", NULL), &b, &e);
    const size_t F = (size_t)(e - b);
    long rb = 0, re = (long)F; parse_range(arg_val(argc, argv, "--range", NULL), &rb, &re);
    if (rb < 0 || rb > re || re > (long)F) { fprintf(stderr, "bad --range\n"); return 2; }
    const float sigma = (float)atof(arg_val(argc, argv, "--sigma", "5"));
    const md_protein_backbone_data_t* bb = &sys.protein_backbone;
    const size_t nseg = bb->segment.count; if (!nseg || !bb->segment.rama_type) { fprintf(stderr, "system has no classified protein backbone\n"); return 2; }
    int32_t* five = calloc(nseg * 5, sizeof(int32_t));
    for (size_t i = 0; i < nseg * 5; ++i) five[i] = -1;
    for (size_t r = 0; r < bb->range.count; ++r) {   /* as mode_backbone */
        const size_t rb0 = bb->range.offset[r], re0 = bb->range.offset[r + 1];
        if (re0 - rb0 < 4) continue;
        for (size_t i = rb0 + 1; i + 1 < re0; ++i) {
            five[5 * i + 0] = bb->segment.atoms[i - 1].c; five[5 * i + 1] = bb->segment.atoms[i].n; five[5 * i + 2] = bb->segment.atoms[i].ca;
            five[5 * i + 3] = bb->segment.atoms[i].c; five[5 * i + 4] = bb->segment.atoms[i + 1].n;
        }
    }
    const size_t n = sys.atom.count; float* x = malloc(n * 4); float* y = malloc(n * 4); float* z = malloc(n * 4);
    md_backbone_angles_t* ang = calloc(F * nseg, sizeof(md_backbone_angles_t));
    for (size_t f = 0; f < F; ++f) {
        md_trajectory_frame_header_t hdr = {0};
        if (!md_trajectory_load_frame(&traj, b + (long)f, &hdr, x, y, z)) return 2;
        md_util_backbone_angles_compute(ang + f * nseg, nseg, x, y, z, &hdr.unitcell, bb);
    }
    uint32_t ncls[4] = { 0, 0, 0, 0 }; uint32_t* cls[4];
    for (int c = 0; c < 4; ++c) cls[c] = malloc(sizeof(uint32_t) * nseg);
    for (size_t i = 0; i < nseg; ++i) {
        const int t = (int)bb->segment.rama_type[i];
        const int c = t == MD_RAMACHANDRAN_TYPE_GENERAL ? 0 : t == MD_RAMACHANDRAN_TYPE_GLYCINE ? 1 : t == MD_RAMACHANDRAN_TYPE_PROLINE ? 2 : t == MD_RAMACHANDRAN_TYPE_PREPROL ? 3 : -1;
        if (c >= 0) cls[c][ncls[c]++] = (uint32_t)i;
    }
    float* tex = calloc((size_t)RAMA_DIM * RAMA_DIM * 4, sizeof(float)); double sum[4] = { 0, 0, 0, 0 };
    rama_accumulate(tex, sum, ang, nseg, cls, ncls, (size_t)rb, (size_t)re);
    ref_rama_blur_density_gaussian(tex, RAMA_DIM, sigma);
    const float sums[4] = { (float)sum[0], (float)sum[1], (float)sum[2], (float)sum[3] };
    FILE* f = fopen(arg_val(argc, argv, "--out", "rama.bin"), "wb"); if (!f) return 2;
    wr(f, "MDRAMADN", 8); wr_u64(f, (uint64_t)F); wr_u64(f, (uint64_t)nseg);
    wr(f, five, nseg * 5 * sizeof(int32_t)); wr(f, ang, F * nseg * sizeof(md_backbone_angles_t));
    wr(f, ncls, sizeof(ncls)); for (int c = 0; c < 4; ++c) wr(f, cls[c], ncls[c] * sizeof(uint32_t));
    wr_i64(f, rb); wr_i64(f, re); wr(f, &sigma, 4);
    wr(f, tex, sizeof(float) * RAMA_DIM * RAMA_DIM * 4); wr(f, sums, sizeof(sums));
    fclose(f);
    printf("{\"frames\": %zu, \"segments\": %zu, \"classes\": [%u, %u, %u, %u]}\n", F, nseg, ncls[0], ncls[1], ncls[2], ncls[3]);
    return 0;
}


int main(int argc, char** argv) {
    /* arg_val (harness_common.h) scans argv from index 2 on, as ref_harness's modes do: argv[1] names the mode here too */
    if (argc < 2 || strcmp(argv[1], "rama") != 0) { fprintf(stderr, "usage: rama_harness rama --sys F --traj SPEC ... | rama_harness rama --time F:S\n"); return 1; }
    return mode_rama(argc, argv);
}
