# oracle/spsv.mk -- the reference samples that exercise cusparseSpSV_*, linked with libb200spsv.so first.
#
#   make -f oracle/spsv.mk ref   -> oracle/_ref/spsv_csr_example.{cusparse,b200spsv}, cg_example.b200spsv,
#                                   bicgstab_example.b200spsv
#
# The .b200spsv binaries are the unmodified samples linked `-lb200spsv -lb200spmv -lcusparse`: SpSV and SpMV resolve to
# this project's libraries, everything else to the closed library.  Same compile lines and rpaths as oracle/Makefile,
# whose .cusparse / .b200 binaries this recipe leaves alone.  Skipped when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64
RPATH_GCC  := -Wl,-rpath,'$$ORIGIN/../../cudalibrarysamples_b200' -Wl,-rpath,$(CUDA)/lib64

GCC_SAMPLES := cg bicgstab

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the SpSV samples in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/spsv_csr/spsv_csr_example.c -o $(REFOUT)/spsv_csr_example.cusparse -lcusparse -Xlinker -rpath -Xlinker $(CUDA)/lib64
	nvcc -I$(CUDA)/include $(REF)/cuSPARSE/spsv_csr/spsv_csr_example.c -o $(REFOUT)/spsv_csr_example.b200spsv -L$(SHIM_DIR) -lb200spsv -lb200spmv -lcusparse $(RPATH_SHIM)
	for s in $(GCC_SAMPLES); do \
	  gcc -DNDEBUG -O3 -Wno-unused-result -Wno-deprecated-declarations -I$(CUDA)/include $(REF)/cuSPARSE/$$s/$${s}_example.c -o $(REFOUT)/$${s}_example.b200spsv -L$(SHIM_DIR) -L$(CUDA)/lib64 -lb200spsv -lb200spmv -lcudart -lcusparse -lcublas -lm $(RPATH_GCC) || exit 1; \
	done

.PHONY: ref
