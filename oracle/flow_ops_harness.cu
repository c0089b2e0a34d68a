/*
 * ORACLE harness (test infrastructure): runs the reference's own FlowWarp, FlowWarpGrad, FlowOutOfFrame and Resample
 * kernels (OpKernel::Compute of flowwarp.cc, flowwarp_cuda.cu, flow_out_of_frame.cc, resample.cc and resample_cuda.cu,
 * compiled unmodified) through the stub API of oracle/flow_ops_stub.h.  Built by oracle/flow_ops.mk into
 * oracle/_ref/libref_flow_ops.so and driven by oracle/flow_ops_ref.py.
 *
 * A CPU kernel ("<op>/CPU/<type>") runs on host buffers and touches no device.  A GPU kernel runs on device buffers the
 * caller owns; the device is synchronised before and after it, because resample_cuda.cu launches InterpolationKernel on
 * the legacy default stream and flowwarp_cuda.cu's cudaMemsets run there too.
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

/* key: "<op>/<CPU|GPU>/<float|double>" ("FlowOutOfFrame/CPU/": registered without a type).  Attributes: fill_parameter
 * (FlowWarp), width, height, antialias, type (Resample).  inputs[i] has shape shapes[4 i .. 4 i + 3]; outs[j] holds
 * out_caps[j] elements and gets output j; out0_shape[4] gets output 0's shape.  min_elems: the least number of elements
 * of every buffer the op allocates.  Returns 0, or 1 with a message in err. */
extern "C" int ref_flow_run(const char* key, const char* fill_parameter, int width, int height, int antialias, const char* type,
                            int ninputs, const void* const* inputs, const int64_t* shapes, int64_t min_elems, int nout,
                            void* const* outs, const int64_t* out_caps, int64_t* out0_shape, char* err, int errlen) {
  const std::string k(key);
  auto it = FlowKernelRegistry::table().find(k);
  if (it == FlowKernelRegistry::table().end()) return fail(err, errlen, "no kernel registered for " + k);
  const bool gpu = k.find("/GPU/") != std::string::npos;
  const size_t esz = k.size() >= 7 && k.compare(k.size() - 7, 7, "/double") == 0 ? 8 : 4;
  if (gpu && cudaDeviceSynchronize() != cudaSuccess) return fail(err, errlen, "cudaDeviceSynchronize failed before the call");

  OpKernelConstruction con;
  con.attrs["fill_parameter"].has_s = true;
  con.attrs["fill_parameter"].s = fill_parameter ? fill_parameter : "zero";
  con.attrs["width"].has_i = true;
  con.attrs["width"].i = width;
  con.attrs["height"].has_i = true;
  con.attrs["height"].i = height;
  con.attrs["antialias"].has_b = true;
  con.attrs["antialias"].b = antialias != 0;
  con.attrs["type"].has_s = true;
  con.attrs["type"].s = type ? type : "LINEAR";

  OpKernelContext ctx;   // declared first: its buffers outlive the kernel object
  ctx.on_device = gpu;
  ctx.elem_bytes = esz;
  ctx.min_elems = min_elems;
  std::unique_ptr<OpKernel> kernel(it->second(&con));
  if (!con.status.ok()) return fail(err, errlen, con.status.error_message());
  for (int i = 0; i < ninputs; ++i)
    ctx.inputs.push_back(Tensor(TensorShape(std::vector<int64>(shapes + 4 * i, shapes + 4 * i + 4)), const_cast<void*>(inputs[i])));
  try {
    kernel->Compute(&ctx);
  } catch (const std::exception& e) {
    if (gpu) cudaDeviceSynchronize();
    return fail(err, errlen, e.what());
  }
  if (gpu) {
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail(err, errlen, std::string("after Compute: ") + cudaGetErrorString(e));
  }
  if (!ctx.status.ok()) return fail(err, errlen, ctx.status.error_message());
  if ((int)ctx.outputs.size() != nout) return fail(err, errlen, "the op produced an unexpected number of outputs");
  for (int i = 0; i < nout; ++i) {
    const int64_t count = ctx.outputs[i].NumElements();
    if (count > out_caps[i]) return fail(err, errlen, "output buffer too small");
    if (count == 0) continue;
    if (gpu) {
      if (cudaMemcpy(outs[i], ctx.outputs[i].raw(), count * esz, cudaMemcpyDeviceToDevice) != cudaSuccess)
        return fail(err, errlen, "cudaMemcpy of an output failed");
    } else {
      memcpy(outs[i], ctx.outputs[i].raw(), count * esz);
    }
  }
  for (int d = 0; d < 4; ++d) out0_shape[d] = ctx.outputs[0].dims() == 4 ? ctx.outputs[0].dim_size(d) : -1;
  if (gpu && cudaDeviceSynchronize() != cudaSuccess) return fail(err, errlen, "cudaDeviceSynchronize failed after the copies");
  return 0;
}
