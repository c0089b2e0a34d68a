# Builds the reference's lmbspecialops/src/{flowwarp,flow_out_of_frame,resample}.cc and {flowwarp,resample}_cuda.cu (test
# infrastructure), compiled unmodified for sm_90a from where they lie, with flow_ops_stub.h force-included ahead of the stub
# headers of ref_stub/ and ref_stub_gpu/cuda_helper_shim.h in place of the reference's cuda_helper.h, into
# _ref/libref_flow_ops.so.  It holds the CPU kernels (FlowWarp, FlowWarpGrad, FlowOutOfFrame), which run without a device,
# and the GPU kernels (FlowWarp, FlowWarpGrad, Resample).  Nothing is copied into this repository.
#   make -C oracle -f flow_ops.mk REF_SRC=<reference>/lmbspecialops/src
NVCC ?= /usr/local/cuda/bin/nvcc
REF_SRC ?= $(DEMON_REF_SRC)
FLOW_SRCS = flowwarp.cc flow_out_of_frame.cc resample.cc flowwarp_cuda.cu resample_cuda.cu
# nvcc's defaults otherwise (FMA contraction on, IEEE division), as the reference's CMake build compiles them; the host
# compiler targets baseline x86-64, which has no FMA instruction to contract into
FLOW_NVCCFLAGS = -gencode arch=compute_90a,code=sm_90a -O3 -std=c++14 -Xcompiler -fPIC -w \
                 -include flow_ops_stub.h -include ref_stub_gpu/cuda_helper_shim.h -I ref_stub -I $(REF_SRC)

flow_ops: _ref/libref_flow_ops.so

_ref/libref_flow_ops.so: flow_ops_harness.cu flow_ops.mk flow_ops_stub.h ref_stub_gpu/cuda_helper_shim.h ref_stub/tf_stub.h \
                         ref_stub/tensorflow/core/framework/common_shape_fns.h $(addprefix $(REF_SRC)/,$(FLOW_SRCS))
	mkdir -p _ref
	$(NVCC) $(FLOW_NVCCFLAGS) -shared -o $@ flow_ops_harness.cu $(addprefix $(REF_SRC)/,$(FLOW_SRCS))

.PHONY: flow_ops
