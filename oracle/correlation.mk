# Builds the reference's lmbspecialops/src/{correlation,correlation_1d}.cc and {correlation,correlation_1d}_cuda.cu (test
# infrastructure), compiled unmodified for sm_90a from where they lie against the stub headers of ref_stub_gpu/ (GPU kernel
# context) and ref_stub/ (the rest), with ref_stub_gpu/cuda_helper_shim.h force-included in place of the reference's
# cuda_helper.h, into _ref/libref_correlation.so.  Nothing is copied into this repository.
#   make -C oracle -f correlation.mk REF_SRC=<reference>/lmbspecialops/src
NVCC ?= /usr/local/cuda/bin/nvcc
REF_SRC ?= $(DEMON_REF_SRC)
CORR_SRCS = correlation.cc correlation_1d.cc correlation_cuda.cu correlation_1d_cuda.cu
# nvcc's defaults otherwise (FMA contraction on, IEEE division), as the reference's CMake build compiles them
CORR_NVCCFLAGS = -gencode arch=compute_90a,code=sm_90a -O3 -std=c++14 -Xcompiler -fPIC -w \
                 -include ref_stub_gpu/cuda_helper_shim.h -I ref_stub_gpu -I ref_stub -I $(REF_SRC)

correlation: _ref/libref_correlation.so

_ref/libref_correlation.so: correlation_harness.cu correlation.mk ref_stub_gpu/tf_gpu_stub.h ref_stub_gpu/cuda_helper_shim.h \
                            ref_stub/tf_stub.h $(addprefix $(REF_SRC)/,$(CORR_SRCS))
	mkdir -p _ref
	$(NVCC) $(CORR_NVCCFLAGS) -shared -o $@ correlation_harness.cu $(addprefix $(REF_SRC)/,$(CORR_SRCS))

.PHONY: correlation
