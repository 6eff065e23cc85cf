# oracle/sddmm_bsr.mk -- the reference sample that exercises cusparseSDDMM on a BSR C, built like oracle/sddmm.mk.
#
#   make -f oracle/sddmm_bsr.mk ref   -> oracle/_ref/sddmm_bsr_example.{cusparse,b200}
#
# .cusparse: the unmodified sample against the closed library; .b200: the same source linked `-lb200spmv -lcusparse`, so
# cusparseSDDMM* and cusparseCreateBsr resolve to libb200spmv.so.  Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

SAMPLES := sddmm_bsr

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the BSR SDDMM sample in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	for s in $(SAMPLES); do \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64 || exit 1; \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM) || exit 1; \
	done

.PHONY: ref
