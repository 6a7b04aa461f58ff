/* dssp_harness.c — TEST INFRASTRUCTURE: the reference's secondary-structure inference (md_util_backbone_secondary_structure_infer,
 * md_util.c:2552) driven through the UNMODIFIED reference, frame by frame.
 *
 * Nothing under viamd_b200/ may link, import or execute this. It is linked (oracle/dssp.mk) against the objects oracle/Makefile compiles from the
 * sources under /root/reference/ext/mdlib; outputs go to oracle/_ref/. It generates tests/golden/dssp.npz (tests/golden/make_golden_dssp.py) and
 * times the reference on one thread and on all cores (profiles/secondary_structure.py).
 *
 * The reference takes its turn masks and flags from md_temp_alloc_array without clearing them (md_util.c:2071, 2085), so its rows depend on what
 * the thread's temporary arena held before. Before every call this harness allocates a block over that region, fills it with --prefill (default 0)
 * and releases it again: the call then finds cleared memory where its arrays land, which is the contract of the library. The timing mode clears
 * the region once per thread, outside the timed loop.
 *
 * usage:
 *   dssp_harness dssp --sys F --traj SPEC [--frames B:E] [--reverse] [--prefill BYTE] [--hn-cb-every K] --out O
 *   dssp_harness dssp --sys F --traj SPEC --time R [--threads T]   (secondary structure, backbone angles, both: VIAMD's backbone pass)
 * --hn-cb-every K: segments i with i % K == 0 that have a CB take it as their HN atom (an explicit H position for the test of that path).
 * out: MDSSPRED | u64 F | u64 S | u64 R | i32 atoms[S][5] (N, CA, C, O, HN) | u32 range_off[R + 1] | i32 ss[F][S]
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
#include <pthread.h>

#include "harness_common.h"

static void wr(FILE* f, const void* p, size_t n) { if (fwrite(p, 1, n, f) != n) { perror("fwrite"); exit(3); } }
static void wr_u64(FILE* f, uint64_t v) { wr(f, &v, 8); }

/* a block over the temporary arena that the next md_temp_begin scope will reuse, filled with `byte`, then released */
static void fill_temp_arena(size_t nseg, int byte) {
    const size_t bytes = nseg * 512 + (4u << 20);
    md_temp_scope_t t = md_temp_begin();
    void* p = md_temp_alloc(t, bytes);
    memset(p, byte, bytes);
    md_temp_end(t);
}

/* timing: `kind` 0 = md_util_backbone_secondary_structure_infer, 1 = md_util_backbone_angles_compute, 2 = both per frame, as VIAMD's backbone
 * pass calls them (src/viamd.cpp:488-525, frames already in memory: the pass's frame loads are not timed). The arena region is cleared once per
 * thread before the barrier that starts the clock; the timed loop calls the reference functions only. */
typedef struct {
    const md_system_t* sys; const float* xyz; size_t n, S; int reps, kind; md_secondary_structure_t* ss; md_backbone_angles_t* ang; size_t beg, end;
    pthread_barrier_t* start;
} dssp_job_t;

static void* dssp_worker(void* arg) {
    dssp_job_t* j = arg;
    fill_temp_arena(j->S, 0);
    pthread_barrier_wait(j->start);
    for (int r = 0; r < j->reps; ++r)
        for (size_t f = j->beg; f < j->end; ++f) {
            const float* x = j->xyz + f * 3 * j->n; md_unitcell_t cell = j->sys->unitcell;
            if (j->kind != 0) md_util_backbone_angles_compute(j->ang + f * j->S, j->S, x, x + j->n, x + 2 * j->n, &cell, &j->sys->protein_backbone);
            if (j->kind != 1) md_util_backbone_secondary_structure_infer(j->ss + f * j->S, j->S, x, x + j->n, x + 2 * j->n, &cell, &j->sys->protein_backbone);
        }
    return NULL;
}

static double time_kind(const md_system_t* sys, const float* xyz, size_t n, size_t F, size_t S, int reps, int T, int kind,
                        md_secondary_structure_t* ss, md_backbone_angles_t* ang) {
    double best = 1e300;
    for (int trial = 0; trial < 3; ++trial) {
        pthread_t th[256]; dssp_job_t jobs[256]; pthread_barrier_t start;
        pthread_barrier_init(&start, NULL, (unsigned)T + 1);
        for (int t = 0; t < T; ++t) {
            jobs[t] = (dssp_job_t){ sys, xyz, n, S, reps, kind, ss, ang, F * t / T, F * (t + 1) / T, &start };
            pthread_create(&th[t], NULL, dssp_worker, &jobs[t]);
        }
        pthread_barrier_wait(&start);
        const double t0 = now_s();
        for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
        const double dt = now_s() - t0; if (dt < best) best = dt;
        pthread_barrier_destroy(&start);
    }
    return best;
}

static int mode_dssp(int argc, char** argv) {
    md_allocator_i* alloc = md_vm_arena_create(GIGABYTES(8));
    md_system_t sys; if (!load_system(&sys, arg_val(argc, argv, "--sys", ""), alloc)) return 2;
    md_trajectory_i traj = {0}; mem_traj_t mt;
    if (!make_traj(&traj, &mt, arg_val(argc, argv, "--traj", "sys"), &sys)) return 2;
    long b = 0, e = (long)md_trajectory_num_frames(&traj); parse_range(arg_val(argc, argv, "--frames", NULL), &b, &e);
    const size_t F = (size_t)(e - b);
    md_protein_backbone_data_t* bb = &sys.protein_backbone;
    const size_t S = bb->segment.count, R = bb->range.count;
    if (!S || !R) { fprintf(stderr, "system has no protein backbone\n"); return 2; }
    const long every = atol(arg_val(argc, argv, "--hn-cb-every", "0"));
    if (every > 0) for (size_t i = 0; i < S; i += (size_t)every) if (bb->segment.atoms[i].cb >= 0) bb->segment.atoms[i].hn = bb->segment.atoms[i].cb;
    const size_t n = sys.atom.count;
    float* xyz = malloc(F * 3 * n * sizeof(float)); md_unitcell_t* cells = malloc(F * sizeof(md_unitcell_t));
    for (size_t f = 0; f < F; ++f) {
        md_trajectory_frame_header_t hdr = {0};
        if (!md_trajectory_load_frame(&traj, b + (long)f, &hdr, xyz + f * 3 * n, xyz + f * 3 * n + n, xyz + f * 3 * n + 2 * n)) return 2;
        cells[f] = hdr.unitcell;
    }
    const char* time_s = arg_val(argc, argv, "--time", NULL);
    md_secondary_structure_t* ss = calloc(F * S, sizeof(md_secondary_structure_t));
    if (time_s) {   /* R repetitions over all frames on T threads (contiguous frame blocks), best wall time of 3, for each kind */
        const int reps = atoi(time_s), T = atoi(arg_val(argc, argv, "--threads", "1"));
        if (T < 1 || T > 256) { fprintf(stderr, "--threads 1..256\n"); return 2; }
        sys.unitcell = cells[0];
        md_backbone_angles_t* ang = calloc(F * S, sizeof(md_backbone_angles_t));
        const char* name[3] = { "secondary_structure", "backbone_angles", "backbone_pass" };
        printf("{\"frames\": %zu, \"segments\": %zu, \"threads\": %d, \"repeat\": %d", F, S, T, reps);
        for (int k = 0; k < 3; ++k) {
            const double sec = time_kind(&sys, xyz, n, F, S, reps, T, k, ss, ang);
            printf(", \"%s\": {\"seconds\": %.6f, \"frames_per_s\": %.1f}", name[k], sec, (double)F * reps / sec);
        }
        printf("}\n");
        return 0;
    }
    const bool reverse = arg_val(argc, argv, "--reverse", NULL) != NULL || (argc > 2 && strcmp(argv[argc - 1], "--reverse") == 0);
    const int prefill = atoi(arg_val(argc, argv, "--prefill", "0"));
    for (size_t k = 0; k < F; ++k) {
        const size_t f = reverse ? F - 1 - k : k;
        const float* x = xyz + f * 3 * n;
        fill_temp_arena(S, prefill);
        if (!md_util_backbone_secondary_structure_infer(ss + f * S, S, x, x + n, x + 2 * n, &cells[f], bb)) return 2;
    }
    FILE* fo = fopen(arg_val(argc, argv, "--out", "dssp.bin"), "wb"); if (!fo) return 2;
    wr(fo, "MDSSPRED", 8); wr_u64(fo, F); wr_u64(fo, S); wr_u64(fo, R);
    for (size_t i = 0; i < S; ++i) {
        const md_amino_acid_atoms_t* a = &bb->segment.atoms[i];
        const int32_t q[5] = { a->n, a->ca, a->c, a->o, a->hn };
        wr(fo, q, sizeof(q));
    }
    wr(fo, bb->range.offset, (R + 1) * sizeof(uint32_t));
    for (size_t i = 0; i < F * S; ++i) { const int32_t v = (int32_t)ss[i]; wr(fo, &v, 4); }
    fclose(fo);
    printf("{\"frames\": %zu, \"segments\": %zu, \"ranges\": %zu}\n", F, S, R);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2 || strcmp(argv[1], "dssp") != 0) { fprintf(stderr, "usage: dssp_harness dssp --sys F --traj SPEC ...\n"); return 1; }
    return mode_dssp(argc, argv);
}
