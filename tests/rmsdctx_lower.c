/* rmsdctx_lower.c — helper of tests/test_rmsd_contexts.py: the reference's md_script.c followed by integration/md_script_mdgpu.inl in one
 * translation unit, as tests/range_lower.c builds it. Compiles a script with the unmodified md_script front end, lowers it with the shim and
 * prints one JSON object per property: op, the index lists, and the groups of idx[0] (num_structures, structure_offsets) and of each argument
 * (arg_parts, arg_offsets).
 *   rmsdctx_lower lower --sys F --script S
 * Exit code 3 when the shim reports a statement it does not lower (its MD_LOG_ERROR goes to the log), 2 when the script does not compile. */
#include "../integration/md_script_mdgpu_pre.h"
#include <md_script.c>
#include <md_gro.h>
#include <md_pdb.h>
#include "../oracle/harness_common.h"
#include "../integration/md_script_mdgpu.inl"

static void print_ints(const int32_t* v, size_t n) {
    printf("[");
    for (size_t i = 0; i < n; ++i) printf(i ? ",%d" : "%d", v[i]);
    printf("]");
}

static void print_offsets(const uint32_t* v, size_t n) {   /* n groups: n + 1 offsets, or null */
    if (!v) { printf("null"); return; }
    printf("[");
    for (size_t i = 0; i <= n; ++i) printf(i ? ",%u" : "%u", v[i]);
    printf("]");
}

int main(int argc, char** argv) {
    md_allocator_i* alloc = md_vm_arena_create(GIGABYTES(8));
    md_system_t sys; if (!load_system(&sys, arg_val(argc, argv, "--sys", ""), alloc)) return 2;
    const char* src = arg_val(argc, argv, "--script", "");
    md_script_ir_t* ir = md_script_ir_create(alloc);
    if (!md_script_ir_compile_from_source(ir, (str_t){ src, strlen(src) }, &sys, NULL, NULL) || !md_script_ir_valid(ir)) { fprintf(stderr, "script failed to compile\n"); return 2; }
    md_script_gpu_lowered_t low = {0};
    if (!md_script_gpu_lower_sys(&low, ir, &sys, alloc)) return 3;
    for (size_t i = 0; i < low.num_props; ++i) {
        const mdgpu_property_desc_t* p = &low.props[i];
        printf("{\"name\": \"%s\", \"op\": %u, \"com_args\": %u, \"num_structures\": %zu, \"structure_size\": %zu, \"structure_offsets\": ",
               low.names[i], p->op, p->com_args, p->num_structures, p->structure_size);
        print_offsets(p->structure_offsets, p->num_structures);
        printf(", \"idx\": [");
        for (int k = 0; k < 4; ++k) { if (k) printf(", "); print_ints(p->idx[k], p->idx_count[k]); }
        printf("], \"arg_offsets\": [");
        for (int k = 0; k < 4; ++k) { if (k) printf(", "); print_offsets(p->arg_parts[k] ? p->arg_offsets[k] : NULL, p->arg_parts[k]); }
        printf("]}\n");
    }
    return 0;
}
