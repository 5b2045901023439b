# oracle/pa_stats.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libsvtav1_pa_stats.so: the picture-analysis statistics checker (ref_pa_stats.c: the reference's own
# svt_aom_gathering_picture_statistics on a caller's picture) plus the reference-side glue of the T2 call
# (../integration/svt_b200_pa_glue.c, type-checked against the reference headers, warnings are errors).  Every reference
# symbol comes from _ref/libsvtav1_ref.so (build that first: `make -C oracle ref`), found next to this library at run time.
REF      ?= /root/reference
SRC      := $(REF)/Source
OUT      := _ref
OBJ      := $(OUT)/obj
CC       ?= gcc
INC      := -I$(SRC)/API -I$(SRC)/Lib/Codec -I$(SRC)/Lib/C_DEFAULT -I$(SRC)/Lib/Globals \
            -I$(REF)/third_party/aom/inc -I$(REF)/third_party -I$(REF)/third_party/safestringlib

.PHONY: pa_stats
pa_stats: $(OUT)/libsvtav1_pa_stats.so

$(OBJ)/pa_ref_pa_stats.o: ref_pa_stats.c ../include/svt_b200.h ../integration/svt_b200_pa_glue.h
	@mkdir -p $(OBJ)
	$(CC) -O2 -fPIC -Wall -DEN_AVX512_SUPPORT=0 $(INC) -I../include -I../integration -c $< -o $@
$(OBJ)/pa_glue.o: ../integration/svt_b200_pa_glue.c ../integration/svt_b200_pa_glue.h ../include/svt_b200.h
	@mkdir -p $(OBJ)
	$(CC) -O2 -fPIC -Wall -Werror -DEN_AVX512_SUPPORT=0 $(INC) -I../include -I../integration -c $< -o $@

$(OUT)/libsvtav1_pa_stats.so: $(OBJ)/pa_ref_pa_stats.o $(OBJ)/pa_glue.o $(OUT)/libsvtav1_ref.so
	$(CC) -shared -Wl,-z,defs -o $@ $(OBJ)/pa_ref_pa_stats.o $(OBJ)/pa_glue.o -L$(OUT) -lsvtav1_ref '-Wl,-rpath,$$ORIGIN' -lm
	@echo built $@
