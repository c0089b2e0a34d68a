// Tensor-core convolution path (sm_90a): the shape rules and the per-device launch state.  The kernel is
// conv_tc_halo_kernel (conv_tc_halo.cu); layers whose problems the halo planner does not take run on it in per-tap mode.
#include <cuda.h>

#include <cstring>
#include <mutex>

#include "conv_tc.cuh"

namespace demon {

bool tc_layer_supported(const ConvProblem& p) {
  if (p.Cin < 32 || (p.Cin % 32) != 0) return false;
  if (p.Cout < 16 || (p.Cout % 4) != 0) return false;
  if ((p.in_pitch % 4) != 0 || (p.out_pitch % 4) != 0) return false;
  if ((reinterpret_cast<uintptr_t>(p.in) & 15) != 0 || (reinterpret_cast<uintptr_t>(p.out) & 15) != 0) return false;
  if (p.sy < 1 || p.sx < 1 || (p.Hi % p.sy) != 0 || (p.Wi % p.sx) != 0) return false;
  if (p.ntaps < 1 || p.ntaps > kMaxTaps) return false;
  if (p.scale != nullptr) return false;
  if (p.Ho != p.Hi / p.sy || p.Wo != p.Wi / p.sx) return false;
  return true;
}

void tc_layer_free(TcLayer& t) {
  tc_halo_free(t);
  if (t.w_packed) cudaFree(t.w_packed);
  t.w_packed = nullptr;
}

TcDeviceState& tc_device_state() {
  constexpr int kMaxDevices = 64;
  static TcDeviceState states[kMaxDevices];
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) dev = 0;
  std::lock_guard<std::mutex> lock(mu);
  TcDeviceState& s = states[dev];
  if (s.device != dev) {
    s = TcDeviceState();
    s.device = dev;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    s.sms = sms > 0 ? sms : 132;
    if (cudaMalloc(&s.err_dev, sizeof(int)) == cudaSuccess) cudaMemset(s.err_dev, 0, sizeof(int));
    else s.err_dev = nullptr;
  }
  return s;
}

int conv_tc_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream) { return conv_tc_halo_launch(t, probs, stream); }

int tc_read_error_flag(bool clear) {
  TcDeviceState& ds = tc_device_state();
  if (!ds.err_dev) return 0;
  int v = 0;
  cudaMemcpy(&v, ds.err_dev, sizeof(int), cudaMemcpyDeviceToHost);
  if (v && clear) cudaMemset(ds.err_dev, 0, sizeof(int));
  return v;
}

}  // namespace demon
