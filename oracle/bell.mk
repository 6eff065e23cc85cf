# oracle/bell.mk -- the reference sample that exercises cusparseSpMM on a Blocked-ELL matrix, built with the sample's own nvcc line.
#
#   make -f oracle/bell.mk ref   -> oracle/_ref/spmm_blockedell_example.{cusparse,b200}
#
# .cusparse: the unmodified sample against the closed library; .b200: the same source linked `-lb200spmv -lcusparse`, so
# cusparseSpMM* resolves to libb200spmv.so (cusparseCreateBlockedEll stays the closed library's).  Same rpaths as oracle/Makefile.
# Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64
SRC        := $(REF)/cuSPARSE/spmm_blockedell/spmm_blockedell_example.cpp

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the Blocked-ELL sample in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	nvcc -I$(CUDA)/include $(SRC) -o $(REFOUT)/spmm_blockedell_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64
	nvcc -I$(CUDA)/include $(SRC) -o $(REFOUT)/spmm_blockedell_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM)

.PHONY: ref
