# oracle/sddmm.mk -- the reference samples that exercise cusparseSDDMM_*, built like the SpMV samples of oracle/Makefile.
#
#   make -f oracle/sddmm.mk ref   -> oracle/_ref/sddmm_csr_example.{cusparse,b200},
#                                    oracle/_ref/sddmm_csr_batched_example.{cusparse,b200}
#
# .cusparse: the unmodified sample against the closed library; .b200: the same source linked `-lb200spmv -lcusparse`, so
# cusparseSDDMM* and cusparseCreateCsr / cusparseCsrSetStridedBatch resolve to libb200spmv.so.  Same compile lines and rpaths
# as oracle/Makefile.  Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

SAMPLES := sddmm_csr sddmm_csr_batched

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the SDDMM samples in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	for s in $(SAMPLES); do \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64 || exit 1; \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM) || exit 1; \
	done

.PHONY: ref
