# oracle/banded.mk -- the reference sample that exercises the batched pentadiagonal solve, against the closed library and the shim.
#
#   make -f oracle/banded.mk ref   -> oracle/_ref/gpsvInterleavedBatch_example.{cusparse,b200}
#
# The .b200 binary is the unmodified sample linked `-lb200spmv -lcusparse -lcublas`: cusparseSgpsvInterleavedBatch_bufferSizeExt and
# cusparseSgpsvInterleavedBatch resolve to libb200spmv.so, everything else to the closed libraries (the sample transposes its
# arrays into the interleaved layout with cublasSgeam).  The sample's own nvcc line; same rpaths as oracle/convert.mk.  Skipped
# when REF does not exist.

HERE      := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF       ?= /root/reference
CUDA      ?= /usr/local/cuda
SHIM_DIR  := $(HERE)../cudalibrarysamples_b200
REFOUT    := $(HERE)_ref
SAMPLE    := $(REF)/cuSPARSE/gpsvInterleavedBatch/gpsvInterleavedBatch_example.c

RPATH_SHIM := -Xlinker -rpath -Xlinker '$$ORIGIN/../../cudalibrarysamples_b200' -Xlinker -rpath -Xlinker $(CUDA)/lib64

ref:
	@test -d $(REF)/cuSPARSE || { echo "no $(REF): skipping the gpsvInterleavedBatch sample in oracle/_ref"; exit 0; }
	mkdir -p $(REFOUT)
	nvcc -I$(CUDA)/include $(SAMPLE) -o $(REFOUT)/gpsvInterleavedBatch_example.cusparse -lcusparse -lcublas -Xlinker -rpath -Xlinker $(CUDA)/lib64
	nvcc -I$(CUDA)/include $(SAMPLE) -o $(REFOUT)/gpsvInterleavedBatch_example.b200 -L$(SHIM_DIR) -lb200spmv -lcusparse -lcublas $(RPATH_SHIM)

.PHONY: ref
