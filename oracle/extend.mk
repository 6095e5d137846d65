# oracle/extend.mk -- builds the dataset-tooling checkers (make -f oracle/extend.mk <target>):
#
#   oracle  -> oracle/libpvnet_extend_oracle.so  (extend_oracle.c: farthest point sampling and binary mesh
#                                                rasterisation restated in C, OpenMP over the batch)
#   ref     -> oracle/_ref/libpvnet_refextend.so (given REF_EXT_SRC, the reference project's
#                                                lib/utils/extend_utils/src: its farthest_point_sampling.cpp and
#                                                mesh_rasterization.cpp compiled verbatim from where they lie, with
#                                                the flags of its build_extend_utils_cffi.py, plus ref_rand_shim.c,
#                                                which makes the random start an input)
#
# Both outputs are git-ignored (*.so, oracle/_ref/).  The oracle's flags are oracle/eval.mk's: -march=x86-64-v3
# because the .so may run on another host, -ffp-contract=off so that no product is fused into a sum.

CC          := gcc
CXX         := g++
REF_EXT_SRC ?= $(PVNET_REFERENCE)/lib/utils/extend_utils/src
HERE        := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

CFLAGS := -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared \
          -fvisibility=hidden -Wall -Wextra -std=c11
# build_extend_utils_cffi.py:10-11
REF_FLAGS := -fopenmp -fPIC -O2 -std=c++11

oracle: $(HERE)libpvnet_extend_oracle.so

$(HERE)libpvnet_extend_oracle.so: $(HERE)extend_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

ref:
	@if [ -f $(REF_EXT_SRC)/farthest_point_sampling.cpp ] && [ -f $(REF_EXT_SRC)/mesh_rasterization.cpp ]; then \
	  mkdir -p $(HERE)_ref/extend_obj && \
	  $(CXX) $(REF_FLAGS) -c $(REF_EXT_SRC)/farthest_point_sampling.cpp -o $(HERE)_ref/extend_obj/fps.o && \
	  $(CXX) $(REF_FLAGS) -c $(REF_EXT_SRC)/mesh_rasterization.cpp -o $(HERE)_ref/extend_obj/raster.o && \
	  $(CC) -O2 -fPIC -c $(HERE)ref_rand_shim.c -o $(HERE)_ref/extend_obj/rand_shim.o && \
	  $(CXX) -shared -fopenmp -Wl,-Bsymbolic -o $(HERE)_ref/libpvnet_refextend.so \
	    $(HERE)_ref/extend_obj/fps.o $(HERE)_ref/extend_obj/raster.o $(HERE)_ref/extend_obj/rand_shim.o && \
	  echo "built oracle/_ref/libpvnet_refextend.so"; \
	else \
	  echo "reference sources not present at $(REF_EXT_SRC); keeping prebuilt oracle/_ref if any"; \
	fi

.PHONY: oracle ref
