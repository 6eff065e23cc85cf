# oracle/convert.mk -- the reference sample that exercises the COO sort, against the closed library and against the shim.
#
#   make -f oracle/convert.mk ref   -> oracle/_ref/coosort_example.{cusparse,b200}
#
# The .b200 binary is the unmodified sample linked `-lb200spmv -lcusparse`: cusparseXcoosort_bufferSizeExt, cusparseXcoosortByRow and
# cusparseCreateIdentityPermutation resolve to libb200spmv.so, everything else (cusparseGather among them) to the closed library.
# The sample's own nvcc line; CUDA 12.9 warns that cusparseCreateIdentityPermutation is deprecated.  Same rpaths as oracle/spsm.mk.
# Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the COO sort sample in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/coosort/coosort_example.c -o $(REFOUT)/coosort_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/coosort/coosort_example.c -o $(REFOUT)/coosort_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM)

.PHONY: ref
