# oracle/dlf.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libsvtav1_dlf.so: the deblocking checker (ref_dlf.c: the reference's own svt_av1_loop_filter_frame on a picture
# built from flat mode-info records, and its two-pass replay) plus the reference-side glue of the T2 call
# (../integration/svt_b200_dlf_glue.c, type-checked against the reference headers, warnings are errors).  Every reference
# symbol comes from _ref/libsvtav1_ref.so (build that first: `make -C oracle ref`), found next to this library at run time.
REF      ?= /root/reference
SRC      := $(REF)/Source
OUT      := _ref
OBJ      := $(OUT)/obj
CC       ?= gcc
INC      := -I$(SRC)/API -I$(SRC)/Lib/Codec -I$(SRC)/Lib/C_DEFAULT -I$(SRC)/Lib/Globals \
            -I$(REF)/third_party/aom/inc -I$(REF)/third_party -I$(REF)/third_party/safestringlib

.PHONY: dlf
dlf: $(OUT)/libsvtav1_dlf.so

$(OBJ)/dlf_ref_dlf.o: ref_dlf.c ../include/svt_b200.h ../integration/svt_b200_dlf_glue.h ../svt-av1-psy_b200/csrc/dlf_tables.h
	@mkdir -p $(OBJ)
	$(CC) -O2 -fPIC -Wall -DEN_AVX512_SUPPORT=0 $(INC) -I../include -c $< -o $@
$(OBJ)/dlf_glue.o: ../integration/svt_b200_dlf_glue.c ../integration/svt_b200_dlf_glue.h ../include/svt_b200.h
	@mkdir -p $(OBJ)
	$(CC) -O2 -fPIC -Wall -Werror -DEN_AVX512_SUPPORT=0 $(INC) -I../include -I../integration -c $< -o $@

$(OUT)/libsvtav1_dlf.so: $(OBJ)/dlf_ref_dlf.o $(OBJ)/dlf_glue.o $(OUT)/libsvtav1_ref.so
	$(CC) -shared -Wl,-z,defs -o $@ $(OBJ)/dlf_ref_dlf.o $(OBJ)/dlf_glue.o -L$(OUT) -lsvtav1_ref '-Wl,-rpath,$$ORIGIN' -lm
	@echo built $@
