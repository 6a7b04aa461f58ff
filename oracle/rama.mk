# oracle/rama.mk — TEST INFRASTRUCTURE: VIAMD's Ramachandran density task on the unmodified reference (oracle/rama_harness.c).
#
#  make -C oracle -f rama.mk   -> _ref/rama_harness_{strict,fast}   (only where /root/reference exists; outputs only into _ref/)
#
# The mdlib objects and flags are oracle/Makefile's (included). VIAMD's blur (blur_rows_acc, boxes_for_gauss, blur_density_gaussian) lives in a
# C++ source of the application, not in mdlib: the block from `static inline void blur_rows_acc` up to `static void rama_rep_init` is cut out of
# it at build time (each marker must occur exactly once) into _ref/rama_blur.inc and compiled as C++ by rama_blur.cpp against mdlib's headers.
include Makefile
.DEFAULT_GOAL := rama

VIAMD     ?= $(REF)/../..
RAMA_CPP  := $(VIAMD)/src/components/ramachandran/ramachandran.cpp
CXXCOMMON := -std=gnu++20 -w -mavx2 -mfma -fms-extensions -fno-exceptions -fno-rtti $(REF_DEF) -I$(REF)/src -I$(REF)/ext/simde -I$(REF)/ext -I$(OUT)

.PHONY: rama
rama: $(OUT)/rama_harness_strict $(OUT)/rama_harness_fast

$(OUT)/rama_blur.inc: $(RAMA_CPP)
	@mkdir -p $(OUT)
	awk -v b='static inline void blur_rows_acc' -v e='static void rama_rep_init' \
	    'index($$0, b) == 1 { nb++; on = 1 } index($$0, e) == 1 { ne++; on = 0 } on { print } \
	     END { if (nb != 1 || ne != 1) { print "rama_blur.inc: markers found " nb + 0 " / " ne + 0 " times" > "/dev/stderr"; exit 1 } }' $< > $@.tmp && mv $@.tmp $@

$(OUT)/obj_strict/rama_blur.o: rama_blur.cpp $(OUT)/rama_blur.inc
	@mkdir -p $(dir $@)
	$(CXX) $(CXXCOMMON) $(STRICT) -c rama_blur.cpp -o $@

$(OUT)/obj_fast/rama_blur.o: rama_blur.cpp $(OUT)/rama_blur.inc
	@mkdir -p $(dir $@)
	$(CXX) $(CXXCOMMON) $(FAST) -c rama_blur.cpp -o $@

$(OUT)/rama_harness_strict: rama_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(STRICT_OBJ) $(OUT)/obj_strict/rama_blur.o
	$(CC) $(COMMON) $(STRICT) rama_harness.c $(STRICT_OBJ) $(OUT)/obj_strict/rama_blur.o -o $@ -lm -lpthread

$(OUT)/rama_harness_fast: rama_harness.c harness_common.h ../viamd_b200/csrc/synth.h $(FAST_OBJ) $(OUT)/obj_fast/rama_blur.o
	$(CC) $(COMMON) $(FAST) rama_harness.c $(FAST_OBJ) $(OUT)/obj_fast/rama_blur.o -o $@ -lm -lpthread
