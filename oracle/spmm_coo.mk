# oracle/spmm_coo.mk -- the reference samples that exercise cusparseSpMM on a COO matrix, built with the samples' own nvcc line.
#
#   make -f oracle/spmm_coo.mk ref   -> oracle/_ref/spmm_coo_example.{cusparse,b200}, oracle/_ref/spmm_coo_batched_example.{cusparse,b200}
#
# .cusparse: the unmodified sample against the closed library; .b200: the same source linked `-lb200spmv -lcusparse`, so cusparseSpMM*,
# cusparseCreateCoo and cusparseCooSetStridedBatch resolve to libb200spmv.so.  Same rpaths as oracle/Makefile.  Skipped when REF does
# not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64
SAMPLES    := spmm_coo spmm_coo_batched

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the COO SpMM samples in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	for s in $(SAMPLES); do \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64 || exit 1; \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM) || exit 1; \
	done

.PHONY: ref
