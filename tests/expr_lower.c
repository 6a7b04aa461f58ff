/* expr_lower.c — helper of tests/test_temporal_expressions.py: the reference's md_script.c followed by integration/md_script_mdgpu.inl in one
 * translation unit, as oracle/shim_harness.c builds it. Compiles a script with the unmodified md_script front end, lowers it with the shim and
 * prints one JSON object per property (the script's own, then the hidden ones of calls inside expressions): name, op, index lists, and the
 * postfix program of an expression as [kind, value, prop] triples.
 *   expr_lower lower --sys F --script S   (the mode word keeps the argument layout of oracle/harness_common.h)
 * Exit code 3 when the shim reports a statement it does not lower (its MD_LOG_ERROR goes to the log), 2 when the script does not compile. */
#include "../integration/md_script_mdgpu_pre.h"
#include <md_script.c>
#include <md_gro.h>
#include <md_pdb.h>
#include "../oracle/harness_common.h"
#include "../integration/md_script_mdgpu.inl"

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
        printf("{\"name\": \"%s\", \"op\": %u, \"own\": %d, \"num_structures\": %zu, \"idx\": [", low.names[i], p->op, i < md_array_size(ir->property_names), p->num_structures);
        for (int k = 0; k < 4; ++k) {
            printf(k ? ", [" : "[");
            for (size_t j = 0; j < p->idx_count[k]; ++j) printf(j ? ",%d" : "%d", p->idx[k][j]);
            printf("]");
        }
        printf("], \"program\": [");
        for (size_t x = 0; x < low.num_exprs; ++x) if (low.exprs[x].prop == i)
            for (size_t j = 0; j < low.exprs[x].num_nodes; ++j) { const mdgpu_expr_node_t* n = &low.exprs[x].nodes[j]; printf("%s[%u, %.9g, %u]", j ? ", " : "", n->kind, n->value, n->prop); }
        printf("]}\n");
    }
    return 0;
}
