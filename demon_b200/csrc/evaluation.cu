// Ground-truth preparation of the DeMoN evaluation (python/depthmotionnet/evaluation/evaluate_to_xarray.py:93-124) on the
// device: the mask of the pixels of view 1 that are visible in view 2, compute_visible_points_mask
// (dataset_tools/view_tools_cython.pyx:9-58).  The .pyx computes in float32 C arithmetic in a fixed order; the kernel does
// the same operations in the same order with round-to-nearest intrinsics (no contraction into FMAs; the projection is
// view_projection.cuh's, shared with the depth ratios), so the mask equals the compiled Cython bit for bit.  One thread
// per pixel, K1, R1^T and t1 of the sample in shared memory.
#include "common.cuh"
#include "view_projection.cuh"
#include <cstdint>

namespace demon {
namespace {

template <bool kInverse>
__global__ void __launch_bounds__(256) visible_points_mask_kernel(const float* __restrict__ depth, const float* __restrict__ K1,
                                                                 const float* __restrict__ R1, const float* __restrict__ t1,
                                                                 const float* __restrict__ P2, int h, int w, int width2, int height2,
                                                                 int borderx, int bordery, uint8_t* __restrict__ mask) {
  __shared__ float cam[21];   // K1 (9), RT = R1^T (9), t1 (3) of this sample
  const int n = blockIdx.y;
  if (threadIdx.x < 9) {
    const int r = threadIdx.x / 3, c = threadIdx.x % 3;
    cam[threadIdx.x] = K1[9 * n + threadIdx.x];
    cam[9 + threadIdx.x] = R1[9 * n + c * 3 + r];   // RT[r][c] = R1[c][r] (.pyx:27)
  } else if (threadIdx.x < 12) {
    cam[18 + threadIdx.x - 9] = t1[3 * n + threadIdx.x - 9];
  }
  __syncthreads();
  const long hw = (long)h * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const float* K = cam;
  const float* RT = cam + 9;
  const float* t = cam + 18;
  const float* P = P2 + 12 * n;   // [3][4], read through the cache: 12 floats shared by every thread of the sample
  const int y = (int)(i / w), x = (int)(i - (long)y * w);
  float d = __ldg(depth + n * hw + i);
  if (kInverse) d = fdiv(1.0f, d);   // abs_depth = 1/depth (evaluate_to_xarray.py:110)
  uint8_t m = 0;
  float u, v, z;
  if (isfinite(d) && d > 0.0f && project_into_view2(d, x, y, K, RT, t, P, u, v, z)) {
    if (u > (float)borderx && v > (float)bordery && u < (float)(width2 - borderx) && v < (float)(height2 - bordery)) m = 1;
  }
  mask[n * hw + i] = m;
}

template <bool kInverse>
int visible_points_mask(const float* depth, const float* K1, const float* R1, const float* t1, const float* P2, int n, int h, int w,
                        int width2, int height2, int borderx, int bordery, uint8_t* mask, void* stream) {
  DEMON_REQUIRE(n >= 0 && n <= 65535 && h >= 0 && w >= 0, "visible_points_mask: bad size");
  if (n == 0 || h == 0 || w == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && K1 && R1 && t1 && P2 && mask, "visible_points_mask: null pointer");
  const long hw = (long)h * w;
  DEMON_REQUIRE(hw <= (long)65535 * 256, "visible_points_mask: %dx%d pixels per view is too many", h, w);
  visible_points_mask_kernel<kInverse><<<dim3((unsigned)((hw + 255) / 256), n), 256, 0, (cudaStream_t)stream>>>(
      depth, K1, R1, t1, P2, h, w, width2, height2, borderx, bordery, mask);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int demon_visible_points_mask_f32(const float* depth, const float* K1, const float* R1, const float* t1, const float* P2, int n, int h,
                                  int w, int width2, int height2, int borderx, int bordery, uint8_t* mask, void* stream) {
  return visible_points_mask<false>(depth, K1, R1, t1, P2, n, h, w, width2, height2, borderx, bordery, mask, stream);
}

int demon_visible_points_mask_inverse_f32(const float* inverse_depth, const float* K1, const float* R1, const float* t1, const float* P2,
                                          int n, int h, int w, int width2, int height2, int borderx, int bordery, uint8_t* mask,
                                          void* stream) {
  return visible_points_mask<true>(inverse_depth, K1, R1, t1, P2, n, h, w, width2, height2, borderx, bordery, mask, stream);
}

}  // extern "C"
