# oracle/dssp.mk — TEST INFRASTRUCTURE: the reference's secondary-structure inference on the unmodified reference (oracle/dssp_harness.c).
#
#  make -C oracle -f dssp.mk   -> _ref/dssp_harness_{strict,fast}   (only where the reference sources exist; outputs only into _ref/)
#
# The mdlib objects and flags are oracle/Makefile's (included).
include Makefile
.DEFAULT_GOAL := dssp

.PHONY: dssp
dssp: $(OUT)/dssp_harness_strict $(OUT)/dssp_harness_fast

$(OUT)/dssp_harness_strict: dssp_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(STRICT_OBJ)
	$(CC) $(COMMON) $(STRICT) dssp_harness.c $(STRICT_OBJ) -o $@ -lm -lpthread

$(OUT)/dssp_harness_fast: dssp_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(FAST_OBJ)
	$(CC) $(COMMON) $(FAST) dssp_harness.c $(FAST_OBJ) -o $@ -lm -lpthread
