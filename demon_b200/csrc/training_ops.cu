// Training-side companions of the hot-path ops (SURVEY.md section 8 f4): the gradient kernels the reference registers for
// its custom ops and the small element-wise ops its v2 losses use.  Same layout conventions and the same IEEE operation
// order as the reference CPU kernels (checked bit for bit against oracle/_ref, the reference's own sources compiled here).
//   ScaleInvariantGradientGrad   scaleinvariantgradient.cc:294-404 (GATHER form like the CPU kernel: deterministic, no atomics)
//   LeakyReluLmbGrad             leakyrelu.cc:127-155
//   ReplaceNonfinite / Grad      replacenonfinite.cc:49-80,115-150
//   DepthToNormals               depthtonormals.cc:147-238 (normal map of a depth map; used by the v2 losses and blocks)
#include "geometry.cuh"

namespace demon {
namespace {

template <class T>
struct SigGradParams {
  int deltas[16];
  T weights[16];
  int num;
  T eps;
};

// input [z][h][w], grad [z][2][h][w] -> out [z][h][w]; thread = one input pixel
template <class T>
__global__ void __launch_bounds__(128) sig_grad_kernel(const T* __restrict__ in, const T* __restrict__ grad, T* __restrict__ out, int H, int W,
                                                      int zbase, SigGradParams<T> prm) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int64_t z = (int64_t)zbase + blockIdx.z;
  if (x >= W) return;
  const size_t hw = (size_t)H * W;
  const T* p = in + z * hw;
  const T* gx = grad + z * 2 * hw;
  const T* gy = gx + hw;
  const size_t i0 = (size_t)y * W + x;
  const T v0 = __ldg(p + i0);
  T diff = 0;
  if (isfinite(v0)) {
    for (int c = 0; c < prm.num; ++c) {
      const int d = prm.deltas[c];
      T tmp = 0;
      if (x + d >= 0 && x + d < W) {
        const T vx = __ldg(p + i0 + d);
        if (isfinite(vx)) tmp = fadd(tmp, fmul(sig_dcenter(v0, vx, prm.eps), __ldg(gx + i0)));
      }
      if (x - d >= 0 && x - d < W) {
        const T vx = __ldg(p + i0 - d);
        if (isfinite(vx)) tmp = fadd(tmp, fmul(sig_dneighbour(vx, v0, prm.eps), __ldg(gx + i0 - d)));
      }
      if (y + d >= 0 && y + d < H) {
        const T vy = __ldg(p + i0 + (ptrdiff_t)d * W);
        if (isfinite(vy)) tmp = fadd(tmp, fmul(sig_dcenter(v0, vy, prm.eps), __ldg(gy + i0)));
      }
      if (y - d >= 0 && y - d < H) {
        const T vy = __ldg(p + i0 - (ptrdiff_t)d * W);
        if (isfinite(vy)) tmp = fadd(tmp, fmul(sig_dneighbour(vy, v0, prm.eps), __ldg(gy + i0 - (ptrdiff_t)d * W)));
      }
      diff = fadd(diff, fmul(prm.weights[c], tmp));
    }
  }
  if (!isfinite(diff)) diff = 0;
  out[z * hw + i0] = diff;
}

template <class T>
int sig_grad_launch(const T* grad, const T* in, T* out, int64_t z, int h, int w, const int* deltas, const T* weights, int num, T eps, void* stream) {
  DEMON_REQUIRE(z >= 0 && h >= 0 && w >= 0, "scale_invariant_gradient_grad: negative size");
  DEMON_REQUIRE(num >= 0 && num <= 16, "scale_invariant_gradient_grad: at most 16 deltas (got %d)", num);
  DEMON_REQUIRE(num == 0 || (deltas && weights), "scale_invariant_gradient_grad: null deltas/weights");
  if (z * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(in && grad && out, "scale_invariant_gradient_grad: null pointer");
  DEMON_REQUIRE(h <= 65535, "scale_invariant_gradient_grad: h must be <= 65535 (got %d)", h);
  SigGradParams<T> prm;
  prm.num = num;
  prm.eps = eps;
  for (int i = 0; i < 16; ++i) { prm.deltas[i] = i < num ? deltas[i] : 0; prm.weights[i] = i < num ? weights[i] : (T)0; }
  for (int64_t z0 = 0; z0 < z; z0 += 32768) {
    const int zn = (int)((z - z0 < 32768) ? (z - z0) : 32768);
    sig_grad_kernel<T><<<dim3(ceil_div(w, 128), h, zn), 128, 0, (cudaStream_t)stream>>>(in, grad, out, h, w, (int)z0, prm);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

// element-wise ops: 0 leaky_relu_grad (a = gradients, b = input), 1 replace_nonfinite (a = input), 2 replace_nonfinite_grad
template <class T, int OP>
__global__ void __launch_bounds__(256) elementwise_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int64_t size, T param) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < size; i += stride) {
    if (OP == 0) {          // leakyrelu.cc:147-153
      const T tmp = b[i];
      const T leak_tmp = fmul(param, tmp);
      out[i] = (tmp >= leak_tmp) ? a[i] : fmul(param, a[i]);
    } else if (OP == 1) {   // replacenonfinite.cc:72-76
      const T tmp = a[i];
      out[i] = isfinite(tmp) ? tmp : param;
    } else {                // replacenonfinite.cc:141-146
      out[i] = isfinite(b[i]) ? a[i] : (T)0;
    }
  }
}

template <class T, int OP>
int elementwise_launch(const T* a, const T* b, T* out, int64_t size, T param, void* stream, const char* what) {
  DEMON_REQUIRE(size >= 0, "%s: negative size", what);
  if (size == 0) return DEMON_OK;
  DEMON_REQUIRE(a && out && (OP == 1 || b), "%s: null pointer", what);
  int64_t blocks = ceil_div64(size, 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  elementwise_kernel<T, OP><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a, b, out, size, param);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

namespace demon {
namespace {

// ---- depth_to_normals (depthtonormals.cc:147-238; the per-pixel arithmetic is d2n_pixel, geometry.cuh) -------------------
// depth [z][h][w], intrinsics [z][4] -> out [z][3][h][w]; thread = one pixel, W on threadIdx.x
template <class T>
__global__ void __launch_bounds__(128) depth_to_normals_kernel(const T* __restrict__ depth, const T* __restrict__ intrinsics, T* __restrict__ out,
                                                              int H, int W, int zbase, bool inverse_depth) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int64_t z = (int64_t)zbase + blockIdx.z;
  if (x >= W) return;
  const size_t hw = (size_t)H * W;
  const T* dm = depth + z * hw;
  T* o = out + z * 3 * hw + (size_t)y * W + x;
  T nrm[3];
  d2n_pixel(nrm, dm, intrinsics + 4 * z, x, y, H, W, inverse_depth);
  o[0] = nrm[0]; o[hw] = nrm[1]; o[2 * hw] = nrm[2];
}

template <class T>
static int depth_to_normals_launch(const T* depth, const T* intrinsics, T* out, int64_t z, int h, int w, int inverse_depth, void* stream) {
  DEMON_REQUIRE(z >= 0 && h >= 0 && w >= 0, "depth_to_normals: negative size");
  if (z * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && intrinsics && out, "depth_to_normals: null pointer");
  DEMON_REQUIRE(h <= 65535, "depth_to_normals: h must be <= 65535 (got %d)", h);
  for (int64_t z0 = 0; z0 < z; z0 += 32768) {
    const int zn = (int)((z - z0 < 32768) ? (z - z0) : 32768);
    depth_to_normals_kernel<T><<<dim3(ceil_div(w, 128), h, zn), 128, 0, (cudaStream_t)stream>>>(depth, intrinsics, out, h, w, (int)z0, inverse_depth != 0);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

extern "C" {

int demon_depth_to_normals_f32(const float* depth, const float* intrinsics, float* output, int64_t z, int h, int w, int inverse_depth, void* stream) {
  return depth_to_normals_launch<float>(depth, intrinsics, output, z, h, w, inverse_depth, stream);
}
int demon_depth_to_normals_f64(const double* depth, const double* intrinsics, double* output, int64_t z, int h, int w, int inverse_depth, void* stream) {
  return depth_to_normals_launch<double>(depth, intrinsics, output, z, h, w, inverse_depth, stream);
}

int demon_scale_invariant_gradient_grad_f32(const float* gradients, const float* input, float* output, int64_t z, int h, int w,
                                            const int* deltas, const float* weights, int num, float epsilon, void* stream) {
  return sig_grad_launch<float>(gradients, input, output, z, h, w, deltas, weights, num, epsilon, stream);
}
int demon_scale_invariant_gradient_grad_f64(const double* gradients, const double* input, double* output, int64_t z, int h, int w,
                                            const int* deltas, const double* weights, int num, double epsilon, void* stream) {
  return sig_grad_launch<double>(gradients, input, output, z, h, w, deltas, weights, num, epsilon, stream);
}
int demon_leaky_relu_grad_f32(const float* gradients, const float* input, float* output, int64_t size, float leak, void* stream) {
  return elementwise_launch<float, 0>(gradients, input, output, size, leak, stream, "leaky_relu_grad");
}
int demon_leaky_relu_grad_f64(const double* gradients, const double* input, double* output, int64_t size, double leak, void* stream) {
  return elementwise_launch<double, 0>(gradients, input, output, size, leak, stream, "leaky_relu_grad");
}
int demon_replace_nonfinite_f32(const float* input, float* output, int64_t size, float value, void* stream) {
  return elementwise_launch<float, 1>(input, nullptr, output, size, value, stream, "replace_nonfinite");
}
int demon_replace_nonfinite_f64(const double* input, double* output, int64_t size, double value, void* stream) {
  return elementwise_launch<double, 1>(input, nullptr, output, size, value, stream, "replace_nonfinite");
}
int demon_replace_nonfinite_grad_f32(const float* gradients, const float* input, float* output, int64_t size, void* stream) {
  return elementwise_launch<float, 2>(gradients, input, output, size, 0.f, stream, "replace_nonfinite_grad");
}
int demon_replace_nonfinite_grad_f64(const double* gradients, const double* input, double* output, int64_t size, void* stream) {
  return elementwise_launch<double, 2>(gradients, input, output, size, 0.0, stream, "replace_nonfinite_grad");
}

}  // extern "C"
