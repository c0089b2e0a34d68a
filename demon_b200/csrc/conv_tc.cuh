// Tensor-core (wgmma) implicit-GEMM convolution for sm_90a (conv_tc_halo.cu) -- interface.
#pragma once
#include "conv.cuh"

namespace demon {

struct HaloPlan;   // tiling, TMA descriptors and packed weights of one layer (conv_tc_halo.cu)

// Per-layer state of the tensor-core path.
struct TcLayer {
  HaloPlan* plan = nullptr;   // owned, with the packed weights on the device; null: the layer has no tensor-core plan
  size_t splitk_bytes = 0;    // split-K layers: scratch the launch needs in probs[0].partial (partial sums); else 0
  bool per_tap = false;       // the plan runs the kernel in per-tap mode
};

// tc_prepare's result for a layer the tensor-core path does not take (not an error: the layer stays on the SIMT path)
constexpr int kTcNoPlan = 1;
// tc_prepare's result at DEMON_PREC_FP16 for a layer that has a plan but a weight FP16 cannot hold (|w| > 65504 or not
// finite); nothing is allocated, the caller names the variable
constexpr int kTcWeightRange = 2;

// Decides whether a layer runs on the tensor cores and in which mode, and if so uploads its weights packed for the
// kernel.  `nclass` problems that share input, tiling and Cout (1 for a convolution, 4 for the sub-pixel classes of a
// transposed convolution) run in ONE launch.  w_hosts[c]: [ntaps][Cin][Cout_pad] fp32, the same packing the SIMT path
// uses.  Returns DEMON_OK, kTcNoPlan, kTcWeightRange or an error code.
int tc_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision);
int conv_tc_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream);
// The plan tc_prepare would choose, as text (no device needed); 0 if the layer has no plan.
int tc_describe(const ConvProblem* probs, int nclass, int precision, char* buf, int buflen);
void tc_layer_free(TcLayer& t);
// 1 if an mbarrier wait of the tensor-core kernel has timed out on the current device since the flag was last cleared
// (synchronises the device); `clear` resets it.  A timed-out wait lets the kernel run to completion with garbage, so the
// forward entry points and demon_check_errors() turn this flag into DEMON_E_STATE.
int tc_read_error_flag(bool clear);
// debug: per-CTA wait-cycle counters of the kernel (slots documented in tools/bench_conv.py)
void tc_halo_enable_timing(bool on);
int tc_halo_read_timing(long long* host, int nblocks);

}  // namespace demon
