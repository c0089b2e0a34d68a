// Convolution problem descriptor shared by the fp32 SIMT path (conv_simt.cu), the tensor-core path
// (conv_tc_halo.cu) and the network plan (net.cu).
//
// Every convolution-like layer of the DeMoN graphs -- the caffe-padded conv2d (helpers.py:70-94), the
// separable k x 1 / 1 x k pairs (helpers.py:105-153), the k4 s2 transposed conv (blocks_original.py:54-117,
// as four sub-pixel 2x2 convolutions) and the dense layers (blocks_original.py:390-410, a 1x1 conv on a
// 1x1 image) -- is one implicit GEMM
//
//     out[n, oy*osy+ooy, ox*osx+oox, co] = act( bias[co] + sum_{t, ci} in[n, oy*sy+dy[t], ox*sx+dx[t], ci] * w[t][ci][co] )
//
// over NHWC activations; taps that fall outside the input read zero (the explicit tf.pad of the
// reference).  Inputs and outputs are channel SLICES of wider NHWC buffers (pitch/offset), which is how
// the skip-concats of the graphs (blocks_original.py:111,186,366,482) cost nothing: producers write
// straight into their slice of the concat buffer.
#pragma once
#include "common.cuh"

namespace demon {

constexpr int kMaxTaps = 16;

struct ConvProblem {
  // input slice
  const float* in;
  int in_pitch;   // channels per pixel of the underlying buffer
  int B, Hi, Wi;  // input image size
  int Cin;        // channels read (multiple of 4; padded channels must hold finite values, their weights are 0)
  // output slice
  float* out;
  int out_pitch;
  int Ho, Wo;          // size of the output index space of THIS launch
  int Hfull, Wfull;    // size of the output image the slice lives in
  int osy, osx, ooy, oox;  // output pixel = (oy*osy+ooy, ox*osx+oox)
  int Cout;            // logical output channels written
  int Cout_pad;        // row pitch of w (multiple of 4)
  // geometry
  int sy, sx;
  int ntaps;
  int dy[kMaxTaps], dx[kMaxTaps];
  // parameters
  const float* w;     // [ntaps][Cin][Cout_pad] fp32 (SIMT path)
  const float* bias;  // [Cout_pad]
  int leaky;          // apply max(0.1f*x, x)
  const float* scale; // optional [B]: channel 0 is multiplied by scale[n*scale_stride] after bias (depth = scale * ch0,
  int scale_stride;   //   blocks_original.py:281-283)
  // split-K (dense layers, SIMT path only): `ksplit` CTAs along K write partial sums to `partial`
  // ([ksplit][M][Cout_pad] floats) and a second kernel reduces them in a fixed order (deterministic)
  float* partial;
  int ksplit;
};

// fp32 CUDA-core implicit GEMM (conv_simt.cu)
int conv_simt_launch(const ConvProblem& p, cudaStream_t stream);

}  // namespace demon
