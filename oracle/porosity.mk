# oracle/porosity.mk — TEST INFRASTRUCTURE: the reference's van der Waals radii of a system (oracle/radii_harness.c), which porosity() needs
# as an input of the library and which tests/golden/make_golden_porosity.py stores with the reference's porosity values.
#
#  make -C oracle -f porosity.mk   -> _ref/radii_harness   (only where the reference sources exist; outputs only into _ref/)
#
# The mdlib objects and flags are oracle/Makefile's (included).
include Makefile
.DEFAULT_GOAL := porosity

.PHONY: porosity
porosity: $(OUT)/radii_harness

$(OUT)/radii_harness: radii_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(STRICT_OBJ)
	$(CC) $(COMMON) $(STRICT) radii_harness.c $(STRICT_OBJ) -o $@ -lm -lpthread

# The reference's _porosity takes its bit grid from md_temp_alloc_array, which does not clear memory (md_allocator.c:262), and never clears it:
# the voxels of whatever the thread's temporary arena held before count as occupied, e.g. the previous frame's grid. Its values are only defined
# with cleared temporaries. ref_harness_zt is ref_harness_strict with md_script.c compiled so that every temporary allocation is cleared
# (md_temp_alloc -> md_temp_alloc_zero); nothing else changes, and code that initialises what it allocates computes exactly as before.
porosity: $(OUT)/ref_harness_zt

$(OUT)/obj_strict_zt/md_script.o: md_script.c
	@mkdir -p $(dir $@)
	$(CC) $(COMMON) $(STRICT) -Dmd_temp_alloc=md_temp_alloc_zero -c $< -o $@

$(OUT)/ref_harness_zt: ref_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(SHIM_OBJ) $(OUT)/obj_strict_zt/md_script.o
	$(CC) $(COMMON) $(STRICT) ref_harness.c $(SHIM_OBJ) $(OUT)/obj_strict_zt/md_script.o -o $@ -lm -lpthread
