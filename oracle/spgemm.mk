# oracle/spgemm.mk -- the reference samples that exercise cusparseSpGEMM*, against the closed library and against the shim.
#
#   make -f oracle/spgemm.mk ref   -> oracle/_ref/spgemm_reuse_example.{cusparse,b200}, spgemm_example.*, spgemm_mem_example.*
#
# The .b200 binaries are the unmodified samples linked `-lb200spmv -lcusparse`: cusparseSpGEMM_createDescr / destroyDescr,
# cusparseSpGEMMreuse_copy / _compute and the descriptors resolve to libb200spmv.so, everything else (reuse_workEstimation /
# reuse_nnz, the non-reuse SpGEMM calls) to the closed library.  Same compile line and rpaths as oracle/spsm.mk.  Skipped when REF
# does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

SAMPLES := spgemm_reuse spgemm spgemm_mem

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the SpGEMM samples in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	for s in $(SAMPLES); do \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64 || exit 1; \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM) || exit 1; \
	done

.PHONY: ref
