# oracle/spsm.mk -- the reference sample that exercises cusparseSpSM_*, against the closed library and against the shim.
#
#   make -f oracle/spsm.mk ref   -> oracle/_ref/spsm_csr_example.{cusparse,b200}
#
# The .b200 binary is the unmodified sample linked `-lb200spmv -lcusparse`: cusparseSpSM_* and the descriptors resolve to
# libb200spmv.so, everything else to the closed library.  Same compile line and rpaths as oracle/spsv.mk.  Skipped when REF
# does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the SpSM sample in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/spsm_csr/spsm_csr_example.c -o $(REFOUT)/spsm_csr_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/spsm_csr/spsm_csr_example.c -o $(REFOUT)/spsm_csr_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse $(RPATH_SHIM)

.PHONY: ref
