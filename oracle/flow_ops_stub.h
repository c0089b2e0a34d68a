/*
 * ORACLE support (test infrastructure, NOT product code): the kernel context of the stub TensorFlow API for the
 * reference's FlowNet ops (flowwarp.cc, flowwarp_cuda.cu, flow_out_of_frame.cc, resample.cc, resample_cuda.cu), force-
 * included by oracle/flow_ops.mk ahead of everything else so that those sources compile unmodified into
 * oracle/_ref/libref_flow_ops.so, CPU and GPU kernels side by side.
 *
 * Everything but the context and the registry comes from the CPU stub (ref_stub/tf_stub.h).  It differs from the
 * correlation stub (ref_stub_gpu/tf_gpu_stub.h) in three ways the FlowNet ops need:
 *   - buffers are sized by the element size of the call (Resample is registered for double too);
 *   - a call runs either on the host (the CPU kernels) or on the device (the GPU kernels), and its buffers live there;
 *   - every buffer holds at least `min_elems` elements, zero-filled: FlowWarpGrad_CPU (flowwarp.cc:263-266) zeroes
 *     n*c*h*w elements of its [n,2,h,w] flow gradient, which for c > 2 runs past the end of a buffer of the output's size.
 * Defining the include guards of tf_gpu_stub.h keeps the correlation stub out.
 */
#ifndef ORACLE_FLOW_OPS_STUB_H
#define ORACLE_FLOW_OPS_STUB_H
#define ORACLE_TF_GPU_STUB_H

#include <cuda_runtime.h>
#include <cstring>
#include <deque>

#define OpKernelContext OracleCpuOpKernelContext
#define OpKernel OracleCpuOpKernel
#include "tf_stub.h"
#undef OpKernel
#undef OpKernelContext
#undef REGISTER_KERNEL_BUILDER

namespace tensorflow {

enum DataType { DT_FLOAT = 1 };

struct GpuDeviceStub {
  cudaStream_t s;
  cudaStream_t stream() const { return s; }
};

class OpKernelContext {
 public:
  std::vector<Tensor> inputs;
  std::deque<Tensor> outputs;   // an op keeps output 0's Tensor* while it allocates output 1
  cudaStream_t stream = 0;
  bool on_device = false;
  size_t elem_bytes = 4;
  int64 min_elems = 0;
  Status status;
  ~OpKernelContext() {
    for (void* p : buffers_) on_device ? (void)cudaFree(p) : free(p);
  }
  const Tensor& input(int i) { return inputs[i]; }
  int num_inputs() const { return (int)inputs.size(); }
  Status allocate_output(int i, const TensorShape& s, Tensor** out) {
    if ((int)outputs.size() <= i) outputs.resize(i + 1);
    void* p = alloc(s);
    if (!p) return Status("allocation failed for an output");
    outputs[i] = Tensor(s, p);
    *out = &outputs[i];
    return Status::OK();
  }
  Status allocate_temp(DataType, const TensorShape& s, Tensor* out) {
    void* p = alloc(s);
    if (!p) return Status("allocation failed for a temporary");
    *out = Tensor(s, p);
    return Status::OK();
  }
  GpuDeviceStub eigen_gpu_device() const { return GpuDeviceStub{stream}; }
  void SetStatus(const Status& s) { if (status.ok()) status = s; }
  void CtxFailureWithWarning(const Status& s) { SetStatus(s); }

 private:
  std::vector<void*> buffers_;
  void* alloc(const TensorShape& s) {
    const size_t bytes = (size_t)std::max<int64>(std::max<int64>(1, s.num_elements()), min_elems) * elem_bytes;
    void* p = nullptr;
    if (on_device) {
      if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
      if (cudaMemset(p, 0, bytes) != cudaSuccess) { cudaFree(p); return nullptr; }
    } else {
      p = calloc(1, bytes);
      if (!p) return nullptr;
    }
    buffers_.push_back(p);
    return p;
  }
};

class OpKernel {
 public:
  explicit OpKernel(OpKernelConstruction*) {}
  virtual ~OpKernel() {}
  virtual void Compute(OpKernelContext* context) = 0;
};

typedef OpKernel* (*FlowKernelFactory)(OpKernelConstruction*);
struct FlowKernelRegistry {
  static std::map<std::string, FlowKernelFactory>& table() {
    static std::map<std::string, FlowKernelFactory> t;
    return t;
  }
};
struct FlowKernelRegistrar {
  FlowKernelRegistrar(const Name& n, FlowKernelFactory f) { FlowKernelRegistry::table()[n.def().op + "/" + n.def().device + "/" + n.def().dtype] = f; }
};
#define REGISTER_KERNEL_BUILDER(kernel_builder, ...)                                                         \
  static ::tensorflow::FlowKernelRegistrar ORACLE_TF_CAT(oracle_flow_kernel_, __COUNTER__)(                  \
      ::tensorflow::kernel_builder,                                                                            \
      [](::tensorflow::OpKernelConstruction* c) -> ::tensorflow::OpKernel* { return new __VA_ARGS__(c); })

}  // namespace tensorflow
#endif
