/*
 * ORACLE harness (test infrastructure): runs the reference's own Correlation, CorrelationGrad, Correlation1D and
 * Correlation1DGrad kernels (OpKernel::Compute of correlation_cuda.cu / correlation_1d_cuda.cu, compiled unmodified) on
 * device buffers the caller owns, through the stub API of ref_stub_gpu/tf_gpu_stub.h.  Built by oracle/correlation.mk into
 * oracle/_ref/libref_correlation.so and driven by oracle/correlation_ref.py.
 *
 * The device is synchronised before and after every call: the op's cudaMemsets run on the legacy default stream, and its
 * kernels run on the context's stream, which is that stream too.
 */
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>

#include "tensorflow/core/framework/op_kernel.h"

using namespace tensorflow;

static int fail(char* err, int errlen, const std::string& m) {
  if (err && errlen > 0) snprintf(err, errlen, "%s", m.c_str());
  return 1;
}

/* op: "Correlation", "CorrelationGrad", "Correlation1D" or "Correlation1DGrad".  in1, in2 [n,c,h,w], grad [gn,gc,gh,gw]
 * (the Grad ops) device float32.  out0 / out1: device buffers of out0_cap / out1_cap floats for output 0 / 1 (out1 for the
 * Grad ops); out0_shape[4] gets output 0's shape.  Returns 0, or 1 with a message in err. */
extern "C" int ref_correlation_run(const char* op, const char* corr_type, int kernel_size, int max_displacement, int stride1, int stride2,
                                   int pad_size, int do_abs, int single_dir, int n, int c, int h, int w, const float* in1, const float* in2,
                                   const float* grad, const int64_t* grad_shape, float* out0, int64_t out0_cap, float* out1,
                                   int64_t out1_cap, int64_t* out0_shape, char* err, int errlen) {
  const std::string name(op);
  const bool is_grad = name == "CorrelationGrad" || name == "Correlation1DGrad";
  const bool one_d = name == "Correlation1D" || name == "Correlation1DGrad";
  auto it = GpuKernelRegistry::table().find(name + "/GPU/float");
  if (it == GpuKernelRegistry::table().end()) return fail(err, errlen, "no GPU kernel registered for " + name);
  if (cudaDeviceSynchronize() != cudaSuccess) return fail(err, errlen, "cudaDeviceSynchronize failed before the call");

  OpKernelConstruction con;
  auto set_i = [&](const char* k, int v) { con.attrs[k].has_i = true; con.attrs[k].i = v; };
  con.attrs["corr_type"].has_s = true;
  con.attrs["corr_type"].s = corr_type;
  set_i("kernel_size", kernel_size);
  set_i("max_displacement", max_displacement);
  set_i("stride1", stride1);
  set_i("stride2", stride2);
  set_i("pad_size", pad_size);
  con.attrs["do_abs"].has_b = true;
  con.attrs["do_abs"].b = do_abs != 0;
  if (one_d) set_i("single_dir", single_dir);

  OpKernelContext ctx;   // declared first: its device buffers outlive the kernel object
  std::unique_ptr<OpKernel> kernel(it->second(&con));
  if (!con.status.ok()) return fail(err, errlen, con.status.error_message());
  const TensorShape in_shape(std::vector<int64>{n, c, h, w});
  ctx.inputs.push_back(Tensor(in_shape, (void*)in1));
  ctx.inputs.push_back(Tensor(in_shape, (void*)in2));
  if (is_grad)
    ctx.inputs.push_back(Tensor(TensorShape(std::vector<int64>(grad_shape, grad_shape + 4)), (void*)grad));
  try {
    kernel->Compute(&ctx);
  } catch (const std::exception& e) {
    cudaDeviceSynchronize();
    return fail(err, errlen, e.what());
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(err, errlen, std::string("after Compute: ") + cudaGetErrorString(e));
  if (!ctx.status.ok()) return fail(err, errlen, ctx.status.error_message());
  const int nout = is_grad ? 2 : 1;
  if ((int)ctx.outputs.size() != nout) return fail(err, errlen, "the op produced an unexpected number of outputs");
  float* dst[2] = {out0, out1};
  const int64_t cap[2] = {out0_cap, out1_cap};
  for (int i = 0; i < nout; ++i) {
    const int64_t count = ctx.outputs[i].NumElements();
    if (count > cap[i]) return fail(err, errlen, "output buffer too small");
    if (count > 0 && cudaMemcpy(dst[i], ctx.outputs[i].raw(), count * sizeof(float), cudaMemcpyDeviceToDevice) != cudaSuccess)
      return fail(err, errlen, "cudaMemcpy of an output failed");
  }
  for (int d = 0; d < 4; ++d) out0_shape[d] = ctx.outputs[0].dims() == 4 ? ctx.outputs[0].dim_size(d) : -1;
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : fail(err, errlen, "cudaDeviceSynchronize failed after the copies");
}
