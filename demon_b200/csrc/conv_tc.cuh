// Tensor-core (wgmma) implicit-GEMM convolution for sm_90a -- interface.
#pragma once
#include "conv.cuh"

namespace demon {

// Per-layer state of the tensor-core path: packed (pre-swizzled, hi/lo split) weights on the device and
// the TMA tensor map of the input activation slice.
struct TcLayer {
  void* w_packed = nullptr;   // device, owned
  int nclass = 1;             // 4 for the sub-pixel classes of a transposed convolution (one launch)
  int n_tile = 0;             // wgmma N of this layer (16, 32, 64 or 128)
  int n_tiles = 0;            // grid.y
  int k_chunks = 0;           // Cin / 32
  int th = 0, tw = 0, tb = 0; // output tile: tb images x th rows x tw columns = 128 (or fewer) GEMM rows
  int nsplit = 3;             // 3 = error-compensated 3xTF32, 1 = plain TF32
  int stages = 0;
  int smem_bytes = 0;
  int per_tap = 0;            // halo kernel in per-tap mode (low-resolution layers)
  void* halo_plan = nullptr;  // non-null: the layer runs on the halo kernel (conv_tc_halo.cu); owned
  int ksplit = 1;             // halo kernel: K loop split over `ksplit` work items per tile; then the launch needs
  size_t splitk_bytes = 0;    //   `splitk_bytes` of scratch in probs[0].partial (partial sums, reduced by a second kernel)
};

bool tc_layer_supported(const ConvProblem& p);
// `nclass` problems that share input, tiling and Cout (1 for a convolution, 4 for the sub-pixel classes of a transposed
// convolution) are packed into one layer and run in ONE launch.  w_hosts[c]: [ntaps][Cin][Cout_pad] fp32, the same
// packing the SIMT path uses.  tc_layer_prepare plans the per-tap mode of the halo kernel (one TMA box per filter tap).
int tc_layer_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision);
void tc_layer_free(TcLayer& t);
int conv_tc_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream);
// Halo variant (conv_tc_halo.cu): one fetch of every input pixel per output tile; for layers made of whole 16x8 tiles.
bool tc_halo_supported(const ConvProblem* probs, int nclass);
int tc_halo_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision);
void tc_halo_free(TcLayer& t);
int conv_tc_halo_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream);
int tc_halo_describe(const ConvProblem* probs, int nclass, int nsplit, char* buf, int buflen);
// debug: per-CTA wait-cycle counters of the halo kernel (slots documented in tools/bench_conv.py)
void tc_halo_enable_timing(bool on);
int tc_halo_read_timing(long long* host, int nblocks);
// Per-DEVICE launch state of the tensor-core kernels (one process may drive several GPUs): the dynamic shared-memory
// attribute has to be set on every device a kernel is launched on, the SM count and the pipeline-timeout flag live on
// the device.  tc_device_state() returns the state of the CURRENT device (cudaGetDevice), creating it on first use.
struct TcDeviceState {
  int device = -1;
  int sms = 132;
  int* err_dev = nullptr;        // device int: set to 1 by a bounded mbarrier wait that timed out
};
TcDeviceState& tc_device_state();
// 1 if an mbarrier wait of the tensor-core kernel has timed out on the current device since the flag was last cleared
// (synchronises the device); `clear` resets it.  A timed-out wait lets the kernel run to completion with garbage, so the
// forward entry points and demon_check_errors() turn this flag into DEMON_E_STATE.
int tc_read_error_flag(bool clear);

}  // namespace demon
