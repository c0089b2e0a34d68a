// The projection of a view-1 pixel into view 2 that dataset_tools/view_tools_cython.pyx writes out three times
// (_compute_visible_points_mask :34-54, _compute_depth_ratios :129-149), as float32 C operations in the .pyx's order with
// round-to-nearest intrinsics (no contraction into FMAs).  The visibility mask (evaluation.cu) and the depth ratios
// (dataset_tools.cu) both call it, so the two cannot drift apart.
#pragma once
#include "common.cuh"

namespace demon {

// Camera z d (finite, > 0) of pixel (x, y) of view 1 with K1 [3][3], RT = R1^T [3][3], t1 [3] projected by P2 [3][4].
// Returns false where the .pyx's `point_proj[2] > 0.0` fails; otherwise u = pr0/pr2, v = pr1/pr2 and z = pr2.
__device__ __forceinline__ bool project_into_view2(float d, int x, int y, const float* K, const float* RT, const float* t,
                                                  const float* P, float& u, float& v, float& z) {
  const float px = fadd((float)x, 0.5f), py = fadd((float)y, 0.5f);
  float p0 = fdiv(fmul(d, fsub(px, K[2])), K[0]);
  float p1 = fdiv(fmul(d, fsub(py, K[5])), K[4]);
  float p2 = d;
  p0 = fsub(p0, t[0]);
  p1 = fsub(p1, t[1]);
  p2 = fsub(p2, t[2]);
  float q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) q[r] = fadd(fadd(fmul(RT[3 * r], p0), fmul(RT[3 * r + 1], p1)), fmul(RT[3 * r + 2], p2));
  float pr[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    pr[r] = fadd(fadd(fadd(fmul(P[4 * r], q[0]), fmul(P[4 * r + 1], q[1])), fmul(P[4 * r + 2], q[2])), fmul(P[4 * r + 3], 1.0f));
  if (!(pr[2] > 0.0f)) return false;
  u = fdiv(pr[0], pr[2]);
  v = fdiv(pr[1], pr[2]);
  z = pr[2];
  return true;
}

}  // namespace demon
