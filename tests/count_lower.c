/* count_lower.c — helper of tests/test_group_counts.py and tests/golden/make_golden_count.py: the reference's md_script.c followed by
 * integration/md_script_mdgpu.inl in one translation unit, as tests/range_lower.c builds it.
 *   count_lower lower --sys F --script S   compiles a script with the unmodified md_script front end, lowers it with the shim and prints one JSON
 *                                          object per property: op, cutoffs, com_args, the index lists, the groups of idx[1] (num_structures,
 *                                          structure_offsets) and argument 0's dynamic part (radius, coordinate range, static `and` side).
 *                                          Exit code 3 when the shim reports a statement it does not lower, 2 when the script does not compile.
 *   count_lower groups --sys F             prints the system's groups as the reference holds them after loading (md_util_system_postprocess):
 *                                          component atom offsets, instance atom ranges (md_system_instance_atom_range) and the structures
 *                                          (md_util_system_infer_structures) as CSR offsets + atoms. */
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

static int mode_groups(const md_system_t* sys) {
    printf("{\"components\": ");
    print_offsets(sys->component.atom_offset, sys->component.count);
    printf(", \"instances\": [");
    for (size_t i = 0; i < sys->instance.count; ++i) { const md_urange_t r = md_system_instance_atom_range(sys, i); printf(i ? ",[%u,%u]" : "[%u,%u]", r.beg, r.end); }
    const size_t ns = md_structure_count(&sys->structure);
    printf("], \"structure_offsets\": ");
    if (ns) print_offsets(sys->structure.offset, ns); else printf("[0]");
    printf(", \"structure_atoms\": ");
    print_ints(ns ? (const int32_t*)sys->structure.atom_idx : NULL, ns ? sys->structure.offset[ns] : 0);
    printf("}\n");
    return 0;
}

int main(int argc, char** argv) {
    md_allocator_i* alloc = md_vm_arena_create(GIGABYTES(8));
    md_system_t sys; if (!load_system(&sys, arg_val(argc, argv, "--sys", ""), alloc)) return 2;
    if (argc >= 2 && strcmp(argv[1], "groups") == 0) return mode_groups(&sys);
    const char* src = arg_val(argc, argv, "--script", "");
    md_script_ir_t* ir = md_script_ir_create(alloc);
    if (!md_script_ir_compile_from_source(ir, (str_t){ src, strlen(src) }, &sys, NULL, NULL) || !md_script_ir_valid(ir)) { fprintf(stderr, "script failed to compile\n"); return 2; }
    md_script_gpu_lowered_t low = {0};
    if (!md_script_gpu_lower_sys(&low, ir, &sys, alloc)) return 3;
    for (size_t i = 0; i < low.num_props; ++i) {
        const mdgpu_property_desc_t* p = &low.props[i];
        printf("{\"name\": \"%s\", \"op\": %u, \"cutoff\": [%.9g, %.9g], \"com_args\": %u, \"num_structures\": %zu, \"structure_size\": %zu, \"structure_offsets\": ",
               low.names[i], p->op, p->cutoff_min, p->cutoff_max, p->com_args, p->num_structures, p->structure_size);
        print_offsets(p->structure_offsets, p->num_structures);
        printf(", \"idx\": [");
        for (int k = 0; k < 4; ++k) { if (k) printf(", "); print_ints(p->idx[k], p->idx_count[k]); }
        const mdgpu_dynamic_arg_t* d = &p->dyn[0];
        const mdgpu_range_arg_t* r = NULL;
        for (size_t j = 0; j < low.num_ranges; ++j) if (low.ranges[j].prop == i && low.ranges[j].arg == 0) r = &low.ranges[j];
        const float none[3] = { 0, 0, 0 }; const float* lo = r ? r->lo : none; const float* hi = r ? r->hi : none;
        printf("], \"dyn0\": {\"radius\": [%.9g, %.9g], \"range\": %u, \"lo\": [%.9g, %.9g, %.9g], \"hi\": [%.9g, %.9g, %.9g], \"has_and\": %u, \"and_idx\": ",
               d->radius_min, d->radius_max, r ? 1u : 0u, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], d->has_and);
        print_ints(d->and_idx, d->has_and ? d->and_count : 0);
        printf("}}\n");
    }
    return 0;
}
