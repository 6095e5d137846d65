# oracle/eval.mk -- builds the pose-evaluation checkers (make -f oracle/eval.mk <target>):
#
#   oracle  -> oracle/libpvnet_eval_oracle.so  (eval_oracle.c: the nearest-point search restated in C, OpenMP)
#   ref     -> oracle/_ref/libpvnet_refnn.so   (given REF_NN_SRC, the reference project's
#                                              lib/utils/extend_utils/src: its nearest_neighborhood.cu compiled
#                                              verbatim from where it lies; the launcher is plain extern "C" on
#                                              host pointers, so no shim is needed)
#
# Both outputs are git-ignored (*.so, oracle/_ref/).  Flags as oracle/Makefile: -march=x86-64-v3 because the .so
# may run on another host, -ffp-contract=off because the FMA placement is explicit in the source (fmaf).

CC         := gcc
NVCC       ?= nvcc
REF_NN_SRC ?= $(PVNET_REFERENCE)/lib/utils/extend_utils/src
HERE       := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

CFLAGS := -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared \
          -fvisibility=hidden -Wall -Wextra -std=c11

oracle: $(HERE)libpvnet_eval_oracle.so

$(HERE)libpvnet_eval_oracle.so: $(HERE)eval_oracle.c
	$(CC) $(CFLAGS) -o $@ $< -lm

ref:
	@if [ -f $(REF_NN_SRC)/nearest_neighborhood.cu ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(NVCC) -O3 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -shared \
	    -o $(HERE)_ref/libpvnet_refnn.so $(REF_NN_SRC)/nearest_neighborhood.cu && \
	  echo "built oracle/_ref/libpvnet_refnn.so"; \
	else \
	  echo "reference sources not present at $(REF_NN_SRC); keeping prebuilt oracle/_ref if any"; \
	fi

.PHONY: oracle ref
