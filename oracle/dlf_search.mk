# oracle/dlf_search.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libsvtav1_dlf_search.so: the checker of the deblocking filter-level search (ref_dlf_search.c: the reference's own
# try_filter_frame steps and svt_av1_pick_filter_level on ref_dlf.c's picture) plus the reference-side glue of the T2 calls.
# Variables and the glue object come from dlf.mk; every reference symbol comes from _ref/libsvtav1_ref.so (build that first:
# `make -C oracle ref`), found next to this library at run time.
include dlf.mk

.PHONY: dlf_search
dlf_search: $(OUT)/libsvtav1_dlf_search.so

$(OBJ)/dlf_search.o: ref_dlf_search.c ref_dlf.c ../include/svt_b200.h ../integration/svt_b200_dlf_glue.h ../svt-av1-psy_b200/csrc/dlf_tables.h
	@mkdir -p $(OBJ)
	$(CC) -O2 -fPIC -Wall -DEN_AVX512_SUPPORT=0 $(INC) -I../include -c $< -o $@

$(OUT)/libsvtav1_dlf_search.so: $(OBJ)/dlf_search.o $(OBJ)/dlf_glue.o $(OUT)/libsvtav1_ref.so
	$(CC) -shared -Wl,-z,defs -o $@ $(OBJ)/dlf_search.o $(OBJ)/dlf_glue.o -L$(OUT) -lsvtav1_ref '-Wl,-rpath,$$ORIGIN' -lm
	@echo built $@
