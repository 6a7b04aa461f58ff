/* range_lower.c — helper of tests/test_range_selections.py: the reference's md_script.c followed by integration/md_script_mdgpu.inl in one
 * translation unit, as oracle/shim_harness.c builds it. Compiles a script with the unmodified md_script front end, lowers it with the shim and
 * prints one JSON object per property: op, the index lists, and per argument its dynamic part (radius, coordinate range from
 * md_script_gpu_lowered_t::ranges, static `and` side).
 *   range_lower lower --sys F --script S   (the mode word keeps the argument layout of oracle/harness_common.h)
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
        printf("{\"name\": \"%s\", \"op\": %u, \"cutoff\": [%.9g, %.9g], \"com_args\": %u, \"idx\": [", low.names[i], p->op, p->cutoff_min, p->cutoff_max, p->com_args);
        for (int k = 0; k < 4; ++k) { if (k) printf(", "); print_ints(p->idx[k], p->idx_count[k]); }
        printf("], \"dyn\": [");
        for (int k = 0; k < 4; ++k) {
            const mdgpu_dynamic_arg_t* d = &p->dyn[k];
            const mdgpu_range_arg_t* r = NULL;
            for (size_t j = 0; j < low.num_ranges; ++j) if (low.ranges[j].prop == i && low.ranges[j].arg == (uint32_t)k) r = &low.ranges[j];
            const float none[3] = { 0, 0, 0 }; const float* lo = r ? r->lo : none; const float* hi = r ? r->hi : none;
            printf("%s{\"radius\": [%.9g, %.9g], \"range\": %u, \"lo\": [%.9g, %.9g, %.9g], \"hi\": [%.9g, %.9g, %.9g], \"has_and\": %u, \"and_idx\": ", k ? ", " : "",
                   d->radius_min, d->radius_max, r ? 1u : 0u, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], d->has_and);
            print_ints(d->and_idx, d->has_and ? d->and_count : 0);
            printf("}");
        }
        printf("]}\n");
    }
    return 0;
}
