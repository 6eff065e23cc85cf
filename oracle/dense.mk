# oracle/dense.mk -- the reference samples that exercise sparse <-> dense conversion, against the closed library and against the shim.
#
#   make -f oracle/dense.mk ref   -> oracle/_ref/{sparse2dense_csr,dense2sparse_csr,dense2sparse_blockedell}_example.{cusparse,b200}
#
# The .b200 binaries are the unmodified samples linked `-lb200spmv -lcusparse`: cusparseSparseToDense, cusparseDenseToSparse_convert
# and cusparseCsrSetPointers resolve to libb200spmv.so, the bufferSize calls and cusparseDenseToSparse_analysis to the closed
# library.  The samples' own nvcc line; same rpaths as oracle/convert.mk.  Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref
SAMPLES   := sparse2dense_csr dense2sparse_csr dense2sparse_blockedell

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the sparse <-> dense samples in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	for s in $(SAMPLES); do \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64 && \
	  nvcc -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM) || exit 1; \
	done

.PHONY: ref
