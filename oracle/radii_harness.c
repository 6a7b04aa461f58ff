/* radii_harness.c — TEST INFRASTRUCTURE: dumps the van der Waals radii the UNMODIFIED reference gives a system,
 * md_atom_extract_radii(r, 0, n, &sys.atom) (mdlib/src/md_system.h:782), the array porosity() reads them from.
 * Built by oracle/porosity.mk against oracle/Makefile's strict reference objects; outputs only into _ref/.
 *
 * usage: radii_harness radii --sys F --out O      O = "MDRADII\0", u64 n, float32 radius[n]
 */
#include <md_system.h>
#include <md_trajectory.h>
#include <md_gro.h>
#include <md_pdb.h>
#include <md_util.h>
#include <core/md_allocator.h>
#include <core/md_arena_allocator.h>
#include <core/md_str.h>
#include <core/md_os.h>

#include "harness_common.h"

int main(int argc, char** argv) {
    if (argc < 2 || strcmp(argv[1], "radii") != 0) { fprintf(stderr, "usage: radii_harness radii --sys F --out O\n"); return 1; }
    md_allocator_i* alloc = md_vm_arena_create(GIGABYTES(8));
    md_system_t sys; if (!load_system(&sys, arg_val(argc, argv, "--sys", ""), alloc)) return 2;
    FILE* f = fopen(arg_val(argc, argv, "--out", "radii.bin"), "wb"); if (!f) return 2;
    const uint64_t n = sys.atom.count;
    float* rad = malloc(n * sizeof(float) + 1);
    md_atom_extract_radii(rad, 0, n, &sys.atom);
    if (fwrite("MDRADII", 1, 8, f) != 8 || fwrite(&n, 8, 1, f) != 1 || fwrite(rad, sizeof(float), n, f) != n) { perror("fwrite"); return 3; }
    fclose(f); free(rad);
    printf("{\"atoms\": %llu}\n", (unsigned long long)n);
    return 0;
}
