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

// scaleinvariantgradient.cc:247-268
template <class T>
__device__ __forceinline__ T sig_dcenter(T c, T n, T eps) {
  const T sum_abs = fadd(fadd(tabs(c), tabs(n)), eps);
  const T sign = (c < 0) ? (T)1 : (T)-1;
  return fadd(fdiv((T)-1, sum_abs), fdiv(fmul(sign, fsub(n, c)), fmul(sum_abs, sum_abs)));
}
template <class T>
__device__ __forceinline__ T sig_dneighbour(T c, T n, T eps) {
  const T sum_abs = fadd(fadd(tabs(c), tabs(n)), eps);
  const T sign = (n < 0) ? (T)1 : (T)-1;
  return fadd(fdiv((T)1, sum_abs), fdiv(fmul(sign, fsub(n, c)), fmul(sum_abs, sum_abs)));
}

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
  DEMON_REQUIRE(h <= 65535, "scale_invariant_gradient_grad: height too large");
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

// ---- depth_to_normals (depthtonormals.cc:147-238) --------------------------------------------------------------------------
// inv_K of K = [[fx*W, 0, cx*W], [0, fy*H, cy*H], [0, 0, 1]] the way Eigen 3.3 inverts a fixed 3x3 matrix
// (Eigen/src/LU/InverseImpl.h, compute_inverse<.,.,3>: cofactors times 1/det), restricted to the four entries the op reads.
template <class T>
struct D2NCamera { T i00, i02, i11, i12; };

template <class T>
__device__ __forceinline__ void d2n_point(T p[3], int x, int y, T depth, const D2NCamera<T>& c) {   // compute3dPoint, depthtonormals.cc:95-101
  p[0] = fmul(fadd(fmul(fadd((T)x, (T)0.5), c.i00), c.i02), depth);
  p[1] = fmul(fadd(fmul(fadd((T)y, (T)0.5), c.i11), c.i12), depth);
  p[2] = depth;
}
template <class T>
__device__ __forceinline__ void d2n_cross(T r[3], const T a[3], const T b[3]) {
  r[0] = fsub(fmul(a[1], b[2]), fmul(a[2], b[1]));
  r[1] = fsub(fmul(a[2], b[0]), fmul(a[0], b[2]));
  r[2] = fsub(fmul(a[0], b[1]), fmul(a[1], b[0]));
}
template <class T>
__device__ __forceinline__ void d2n_normalize(T v[3]) {   // MatrixBase::normalize(): z = squaredNorm(); if (z > 0) v /= sqrt(z)
  const T z = fadd(fadd(fmul(v[0], v[0]), fmul(v[1], v[1])), fmul(v[2], v[2]));
  if (z > (T)0) {
    const T n = sqrt(z);   // IEEE sqrt (sqrt.rn for float: no -use_fast_math in this build)
    v[0] = fdiv(v[0], n); v[1] = fdiv(v[1], n); v[2] = fdiv(v[2], n);
  }
}

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
  const T nan = (T)NAN;
  T n0 = nan, n1 = nan, n2 = nan;
  if (!(x == 0 || y == 0 || x == W - 1 || y == H - 1)) {
    const size_t i = (size_t)y * W + x;
    T d = __ldg(dm + i), d_y0 = __ldg(dm + i - W), d_x0 = __ldg(dm + i - 1), d_y1 = __ldg(dm + i + W), d_x1 = __ldg(dm + i + 1);
    if (inverse_depth) { d = fdiv((T)1, d); d_y0 = fdiv((T)1, d_y0); d_x0 = fdiv((T)1, d_x0); d_y1 = fdiv((T)1, d_y1); d_x1 = fdiv((T)1, d_x1); }
    const bool bad = d <= 0 || !isfinite(d) || d_y0 <= 0 || !isfinite(d_y0) || d_x0 <= 0 || !isfinite(d_x0) || d_y1 <= 0 || !isfinite(d_y1) ||
                     d_x1 <= 0 || !isfinite(d_x1);
    if (!bad) {
      D2NCamera<T> c;
      {
        const T* k = intrinsics + 4 * z;
        const T a = fmul(__ldg(k + 0), (T)W), b = fmul(__ldg(k + 1), (T)H), cx = fmul(__ldg(k + 2), (T)W), cy = fmul(__ldg(k + 3), (T)H);
        // cofactors of column 0: (b*1 - cy*0, 0*cx - 1*0, 0*cy - cx*b); det = (c0*a + c1*0) + c2*0; invdet = 1 / det
        const T c0 = fsub(fmul(b, (T)1), fmul(cy, (T)0));
        const T c1 = fsub(fmul((T)0, cx), fmul((T)1, (T)0));
        const T c2 = fsub(fmul((T)0, cy), fmul(cx, b));
        const T det = fadd(fadd(fmul(c0, a), fmul(c1, (T)0)), fmul(c2, (T)0));
        const T invdet = fdiv((T)1, det);
        c.i00 = fmul(c0, invdet);                                                     // result.row(0) = cofactors_col0 * invdet
        c.i02 = fmul(c2, invdet);
        c.i11 = fmul(fsub(fmul((T)1, a), fmul((T)0, cx)), invdet);                    // cofactor<1,1> = m22*m00 - m20*m02
        c.i12 = fmul(fsub(fmul(cx, (T)0), fmul(a, cy)), invdet);                      // cofactor<2,1> = m02*m10 - m00*m12
      }
      T p[3], p_y0[3], p_x0[3], p_y1[3], p_x1[3];
      d2n_point(p, x, y, d, c);
      d2n_point(p_y0, x, y - 1, d_y0, c);
      d2n_point(p_x0, x - 1, y, d_x0, c);
      d2n_point(p_y1, x, y + 1, d_y1, c);
      d2n_point(p_x1, x + 1, y, d_x1, c);
      T a1[3], b1[3], a0[3], b0[3], v1[3], v0[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) { a1[k] = fsub(p[k], p_x1[k]); b1[k] = fsub(p_y1[k], p[k]); a0[k] = fsub(p[k], p_x0[k]); b0[k] = fsub(p_y0[k], p[k]); }
      d2n_cross(v1, a1, b1);
      d2n_cross(v0, a0, b0);
      d2n_normalize(v1);
      d2n_normalize(v0);
      T v[3] = {fadd(v1[0], v0[0]), fadd(v1[1], v0[1]), fadd(v1[2], v0[2])};
      d2n_normalize(v);
      n0 = v[0]; n1 = v[1]; n2 = v[2];
    }
  }
  o[0] = n0; o[hw] = n1; o[2 * hw] = n2;
}

template <class T>
static int depth_to_normals_launch(const T* depth, const T* intrinsics, T* out, int64_t z, int h, int w, int inverse_depth, void* stream) {
  DEMON_REQUIRE(z >= 0 && h >= 0 && w >= 0, "depth_to_normals: negative size");
  if (z * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && intrinsics && out, "depth_to_normals: null pointer");
  DEMON_REQUIRE(h <= 65535, "depth_to_normals: height too large");
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
