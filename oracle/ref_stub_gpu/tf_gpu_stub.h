/*
 * ORACLE support (test infrastructure, NOT product code): the GPU side of the stub TensorFlow API, for the reference's
 * Correlation / Correlation1D ops (correlation_cuda.cu, correlation_1d_cuda.cu), compiled unmodified by
 * oracle/correlation.mk into oracle/_ref/libref_correlation.so.  Only that recipe puts this directory on the include path;
 * libref_ops.so keeps the CPU stub alone.
 *
 * Everything but the kernel context comes from the CPU stub (ref_stub/tf_stub.h).  A GPU op needs more of OpKernelContext
 * than a CPU op: eigen_gpu_device() (whose stream() it launches on), allocate_temp(DT_FLOAT, ...) and device memory behind
 * allocate_output.  So this header takes the CPU stub's OpKernelContext and OpKernel under other names and states GPU ones,
 * with a kernel registry of their own that REGISTER_KERNEL_BUILDER fills and oracle/correlation_harness.cu reads.
 */
#ifndef ORACLE_TF_GPU_STUB_H
#define ORACLE_TF_GPU_STUB_H

#include <cuda_runtime.h>
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

// Outputs and temporaries are device buffers owned by the context and freed with it.  The outputs live in a deque: an op
// keeps the Tensor* of output 0 while it allocates output 1, and a deque's elements do not move when it grows.
class OpKernelContext {
 public:
  std::vector<Tensor> inputs;
  std::deque<Tensor> outputs;
  cudaStream_t stream = 0;
  Status status;
  ~OpKernelContext() {
    for (void* p : buffers_) cudaFree(p);
  }
  const Tensor& input(int i) { return inputs[i]; }
  int num_inputs() const { return (int)inputs.size(); }
  Status allocate_output(int i, const TensorShape& s, Tensor** out) {
    if ((int)outputs.size() <= i) outputs.resize(i + 1);
    void* p = device_alloc(s);
    if (!p) return Status("cudaMalloc failed for an output");
    outputs[i] = Tensor(s, p);
    *out = &outputs[i];
    return Status::OK();
  }
  Status allocate_temp(DataType, const TensorShape& s, Tensor* out) {
    void* p = device_alloc(s);
    if (!p) return Status("cudaMalloc failed for a temporary");
    *out = Tensor(s, p);
    return Status::OK();
  }
  GpuDeviceStub eigen_gpu_device() const { return GpuDeviceStub{stream}; }
  void SetStatus(const Status& s) { if (status.ok()) status = s; }
  void CtxFailureWithWarning(const Status& s) { SetStatus(s); }

 private:
  std::vector<void*> buffers_;
  void* device_alloc(const TensorShape& s) {
    void* p = nullptr;
    const size_t bytes = (size_t)std::max<int64>(1, s.num_elements()) * sizeof(float);
    if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
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

typedef OpKernel* (*GpuKernelFactory)(OpKernelConstruction*);
struct GpuKernelRegistry {
  static std::map<std::string, GpuKernelFactory>& table() {
    static std::map<std::string, GpuKernelFactory> t;
    return t;
  }
};
struct GpuKernelRegistrar {
  GpuKernelRegistrar(const Name& n, GpuKernelFactory f) { GpuKernelRegistry::table()[n.def().op + "/" + n.def().device + "/" + n.def().dtype] = f; }
};
#define REGISTER_KERNEL_BUILDER(kernel_builder, ...)                                                         \
  static ::tensorflow::GpuKernelRegistrar ORACLE_TF_CAT(oracle_gpu_kernel_, __COUNTER__)(                    \
      ::tensorflow::kernel_builder,                                                                            \
      [](::tensorflow::OpKernelConstruction* c) -> ::tensorflow::OpKernel* { return new __VA_ARGS__(c); })

}  // namespace tensorflow
#endif
