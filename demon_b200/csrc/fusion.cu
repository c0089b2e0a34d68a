// Fusion of depth maps into one surface on the device: a truncated signed distance volume (TSDF) integrated frame by frame,
// and marching cubes on it.
//
// * tsdf_integrate_kernel: one thread per voxel.  The thread keeps its voxel's state (tsdf, weight and colour) in registers
//   while it loops over the call's frames, so HBM sees one read and one write of the state per launch; the depth maps and
//   images are gathered through L2 (a 192x256 float32 depth map is 196 KB, so a few hundred frames stay resident).  The
//   cameras of up to kFuseChunk frames at a time are staged in shared memory.
// * marching cubes: launch 1 counts the triangles of every 2048-cube tile into the caller's scratch, launch 2 (one CTA)
//   turns the counts into each tile's first triangle, and launch 3 writes each tile's triangles at that offset, ranked by a
//   warp scan of the per-cube counts.  The output order is the cube's linear index, then the table's triangle order, so it
//   depends on nothing but the volume; there are no atomics and the launches can be captured in a CUDA graph.
//
// Every float operation is a round-to-nearest intrinsic in the order the comments give (no contraction into FMAs), so a
// float32 numpy restatement matches bit for bit.
#include "common.cuh"
#include <cmath>
#include <cstdint>

namespace demon {
namespace {

constexpr int kFuseThreads = 256;
constexpr int kFuseChunk = 64;        // frames whose cameras are staged in shared memory at a time
constexpr int kCam = 16;              // fx, fy, cx, cy, R row-major (9), t (3)
constexpr int kMcThreads = 256;
constexpr int kMcWarps = kMcThreads / 32;
constexpr int kMcRounds = 8;
constexpr int kMcTile = kMcThreads * kMcRounds;   // round j of thread i handles cube tile * kMcTile + j * kMcThreads + i
constexpr int kScanThreads = 1024;

// ---- TSDF integration -------------------------------------------------------------------------------------------------
// Frame f updates voxel X = origin + voxel_size * (i, j, k):  X_c = R X + t, u = fx x/z + cx, v = fy y/z + cy, pixel
// (floor(u), floor(v)) (the pixel-centre-at +0.5 convention of the point clouds and the depth ratios).  The frame is skipped
// when z <= 0, the pixel is outside the image, d is not finite or not > 0, or sdf = d - z < -trunc; otherwise
// f = min(1, sdf / trunc), tsdf = (tsdf W + f) / (W + 1), colour likewise, W = W + 1.
template <bool kColor>
__global__ void __launch_bounds__(kFuseThreads) tsdf_integrate_kernel(
    float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color, int nx, int ny, long nvox, float ox, float oy,
    float oz, float vs, float trunc, const float* __restrict__ depth, const float* __restrict__ K, const float* __restrict__ R,
    const float* __restrict__ t, const uint8_t* __restrict__ image, int n, int h, int w) {
  __shared__ float cam[kFuseChunk][kCam];
  const long vox = (long)blockIdx.x * kFuseThreads + threadIdx.x;
  const bool active = vox < nvox;
  float s = 0.0f, W = 0.0f, c0 = 0.0f, c1 = 0.0f, c2 = 0.0f;
  float X0 = 0.0f, X1 = 0.0f, X2 = 0.0f;
  if (active) {
    s = tsdf[vox];
    W = weight[vox];
    if (kColor) {
      c0 = color[3 * vox];
      c1 = color[3 * vox + 1];
      c2 = color[3 * vox + 2];
    }
    const long plane = (long)nx * ny;
    const int k = (int)(vox / plane);
    const long r = vox - (long)k * plane;
    const int j = (int)(r / nx), i = (int)(r - (long)j * nx);
    X0 = fadd(ox, fmul(vs, (float)i));
    X1 = fadd(oy, fmul(vs, (float)j));
    X2 = fadd(oz, fmul(vs, (float)k));
  }
  const float fw = (float)w, fh = (float)h;
  const long hw = (long)h * w;
  for (int f0 = 0; f0 < n; f0 += kFuseChunk) {
    const int m = min(kFuseChunk, n - f0);
    __syncthreads();   // the previous chunk's cameras are no longer read
    for (int q = threadIdx.x; q < m * kCam; q += kFuseThreads) {
      const int fr = q / kCam, e = q - fr * kCam;
      const long g = f0 + fr;
      float val;
      if (e < 4) val = __ldg(K + 9 * g + (e == 0 ? 0 : e == 1 ? 4 : e == 2 ? 2 : 5));
      else if (e < 13) val = __ldg(R + 9 * g + (e - 4));
      else val = __ldg(t + 3 * g + (e - 13));
      cam[fr][e] = val;
    }
    __syncthreads();
    if (!active) continue;
    for (int fr = 0; fr < m; ++fr) {
      const float* cm = cam[fr];
      const float z = fadd(fadd(fadd(fmul(cm[10], X0), fmul(cm[11], X1)), fmul(cm[12], X2)), cm[15]);
      if (!(z > 0.0f)) continue;
      const float x = fadd(fadd(fadd(fmul(cm[4], X0), fmul(cm[5], X1)), fmul(cm[6], X2)), cm[13]);
      const float y = fadd(fadd(fadd(fmul(cm[7], X0), fmul(cm[8], X1)), fmul(cm[9], X2)), cm[14]);
      const float u = fadd(fdiv(fmul(cm[0], x), z), cm[2]);
      const float v = fadd(fdiv(fmul(cm[1], y), z), cm[3]);
      if (!(u >= 0.0f && u < fw && v >= 0.0f && v < fh)) continue;   // floor(u) in [0, w) and floor(v) in [0, h)
      const long p = (long)(f0 + fr) * hw + (long)(int)v * w + (int)u;
      const float d = __ldg(depth + p);
      if (!(isfinite(d) && d > 0.0f)) continue;
      const float sdf = fsub(d, z);
      if (sdf < -trunc) continue;
      const float fv = fminf(1.0f, fdiv(sdf, trunc));
      const float W1 = fadd(W, 1.0f);
      s = fdiv(fadd(fmul(s, W), fv), W1);
      if (kColor) {
        const uint8_t* px = image + 3 * p;
        c0 = fdiv(fadd(fmul(c0, W), (float)__ldg(px)), W1);
        c1 = fdiv(fadd(fmul(c1, W), (float)__ldg(px + 1)), W1);
        c2 = fdiv(fadd(fmul(c2, W), (float)__ldg(px + 2)), W1);
      }
      W = W1;
    }
  }
  if (active) {
    tsdf[vox] = s;
    weight[vox] = W;
    if (kColor) {
      color[3 * vox] = c0;
      color[3 * vox + 1] = c1;
      color[3 * vox + 2] = c2;
    }
  }
}

// ---- marching cubes ---------------------------------------------------------------------------------------------------
// Corner q of cube (i, j, k) is voxel (i, j, k) + kCorner[q]; bit q of the case is set when its tsdf is < 0.
__constant__ int8_t kCorner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
// The corners of each of the 12 edges, the one with the lower grid coordinate first: a vertex is interpolated from that
// corner, so the cubes that share an edge compute the same vertex bit for bit.
__constant__ int8_t kEdge[12][2] = {{0, 1}, {1, 2}, {3, 2}, {0, 3}, {4, 5}, {5, 6}, {7, 6}, {4, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
// The standard 256-case Lorensen-Cline triangle table (edges of each triangle, -1 ends the list).
__constant__ int8_t kTriTable[256][16] = {
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 8, 3, 9, 8, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 2, 10, 0, 2, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 8, 3, 2, 10, 8, 10, 9, 8, -1, -1, -1, -1, -1, -1, -1},
    {3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 11, 2, 8, 11, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 11, 2, 1, 9, 11, 9, 8, 11, -1, -1, -1, -1, -1, -1, -1},
    {3, 10, 1, 11, 10, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 10, 1, 0, 8, 10, 8, 11, 10, -1, -1, -1, -1, -1, -1, -1},
    {3, 9, 0, 3, 11, 9, 11, 10, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 3, 0, 7, 3, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 1, 9, 4, 7, 1, 7, 3, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 4, 7, 3, 0, 4, 1, 2, 10, -1, -1, -1, -1, -1, -1, -1},
    {9, 2, 10, 9, 0, 2, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4, -1, -1, -1, -1},
    {8, 4, 7, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 4, 7, 11, 2, 4, 2, 0, 4, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 1, 8, 4, 7, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
    {4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1, -1, -1, -1, -1},
    {3, 10, 1, 3, 11, 10, 7, 8, 4, -1, -1, -1, -1, -1, -1, -1},
    {1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4, -1, -1, -1, -1},
    {4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3, -1, -1, -1, -1},
    {4, 7, 11, 4, 11, 9, 9, 11, 10, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 5, 4, 1, 5, 0, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 5, 4, 8, 3, 5, 3, 1, 5, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 1, 2, 10, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
    {5, 2, 10, 5, 4, 2, 4, 0, 2, -1, -1, -1, -1, -1, -1, -1},
    {2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8, -1, -1, -1, -1},
    {9, 5, 4, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 11, 2, 0, 8, 11, 4, 9, 5, -1, -1, -1, -1, -1, -1, -1},
    {0, 5, 4, 0, 1, 5, 2, 3, 11, -1, -1, -1, -1, -1, -1, -1},
    {2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5, -1, -1, -1, -1},
    {10, 3, 11, 10, 1, 3, 9, 5, 4, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10, -1, -1, -1, -1},
    {5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3, -1, -1, -1, -1},
    {5, 4, 8, 5, 8, 10, 10, 8, 11, -1, -1, -1, -1, -1, -1, -1},
    {9, 7, 8, 5, 7, 9, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 3, 0, 9, 5, 3, 5, 7, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 7, 8, 0, 1, 7, 1, 5, 7, -1, -1, -1, -1, -1, -1, -1},
    {1, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 7, 8, 9, 5, 7, 10, 1, 2, -1, -1, -1, -1, -1, -1, -1},
    {10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3, -1, -1, -1, -1},
    {8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2, -1, -1, -1, -1},
    {2, 10, 5, 2, 5, 3, 3, 5, 7, -1, -1, -1, -1, -1, -1, -1},
    {7, 9, 5, 7, 8, 9, 3, 11, 2, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11, -1, -1, -1, -1},
    {2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7, -1, -1, -1, -1},
    {11, 2, 1, 11, 1, 7, 7, 1, 5, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11, -1, -1, -1, -1},
    {5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0, -1},
    {11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0, -1},
    {11, 10, 5, 7, 11, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 1, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 8, 3, 1, 9, 8, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 5, 2, 6, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 5, 1, 2, 6, 3, 0, 8, -1, -1, -1, -1, -1, -1, -1},
    {9, 6, 5, 9, 0, 6, 0, 2, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8, -1, -1, -1, -1},
    {2, 3, 11, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 0, 8, 11, 2, 0, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11, -1, -1, -1, -1},
    {6, 3, 11, 6, 5, 3, 5, 1, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6, -1, -1, -1, -1},
    {3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9, -1, -1, -1, -1},
    {6, 5, 9, 6, 9, 11, 11, 9, 8, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 3, 0, 4, 7, 3, 6, 5, 10, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 5, 10, 6, 8, 4, 7, -1, -1, -1, -1, -1, -1, -1},
    {10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4, -1, -1, -1, -1},
    {6, 1, 2, 6, 5, 1, 4, 7, 8, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7, -1, -1, -1, -1},
    {8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6, -1, -1, -1, -1},
    {7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9, -1},
    {3, 11, 2, 7, 8, 4, 10, 6, 5, -1, -1, -1, -1, -1, -1, -1},
    {5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11, -1, -1, -1, -1},
    {0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6, -1, -1, -1, -1},
    {9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6, -1},
    {8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6, -1, -1, -1, -1},
    {5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11, -1},
    {0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7, -1},
    {6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9, -1, -1, -1, -1},
    {10, 4, 9, 6, 4, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 10, 6, 4, 9, 10, 0, 8, 3, -1, -1, -1, -1, -1, -1, -1},
    {10, 0, 1, 10, 6, 0, 6, 4, 0, -1, -1, -1, -1, -1, -1, -1},
    {8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10, -1, -1, -1, -1},
    {1, 4, 9, 1, 2, 4, 2, 6, 4, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4, -1, -1, -1, -1},
    {0, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 3, 2, 8, 2, 4, 4, 2, 6, -1, -1, -1, -1, -1, -1, -1},
    {10, 4, 9, 10, 6, 4, 11, 2, 3, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6, -1, -1, -1, -1},
    {3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10, -1, -1, -1, -1},
    {6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1, -1},
    {9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3, -1, -1, -1, -1},
    {8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1, -1},
    {3, 11, 6, 3, 6, 0, 0, 6, 4, -1, -1, -1, -1, -1, -1, -1},
    {6, 4, 8, 11, 6, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 10, 6, 7, 8, 10, 8, 9, 10, -1, -1, -1, -1, -1, -1, -1},
    {0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10, -1, -1, -1, -1},
    {10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0, -1, -1, -1, -1},
    {10, 6, 7, 10, 7, 1, 1, 7, 3, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7, -1, -1, -1, -1},
    {2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9, -1},
    {7, 8, 0, 7, 0, 6, 6, 0, 2, -1, -1, -1, -1, -1, -1, -1},
    {7, 3, 2, 6, 7, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7, -1, -1, -1, -1},
    {2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7, -1},
    {1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11, -1},
    {11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1, -1, -1, -1, -1},
    {8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6, -1},
    {0, 9, 1, 11, 6, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0, -1, -1, -1, -1},
    {7, 11, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 8, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 9, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 1, 9, 8, 3, 1, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
    {10, 1, 2, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 3, 0, 8, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
    {2, 9, 0, 2, 10, 9, 6, 11, 7, -1, -1, -1, -1, -1, -1, -1},
    {6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8, -1, -1, -1, -1},
    {7, 2, 3, 6, 2, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {7, 0, 8, 7, 6, 0, 6, 2, 0, -1, -1, -1, -1, -1, -1, -1},
    {2, 7, 6, 2, 3, 7, 0, 1, 9, -1, -1, -1, -1, -1, -1, -1},
    {1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6, -1, -1, -1, -1},
    {10, 7, 6, 10, 1, 7, 1, 3, 7, -1, -1, -1, -1, -1, -1, -1},
    {10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8, -1, -1, -1, -1},
    {0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7, -1, -1, -1, -1},
    {7, 6, 10, 7, 10, 8, 8, 10, 9, -1, -1, -1, -1, -1, -1, -1},
    {6, 8, 4, 11, 8, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 6, 11, 3, 0, 6, 0, 4, 6, -1, -1, -1, -1, -1, -1, -1},
    {8, 6, 11, 8, 4, 6, 9, 0, 1, -1, -1, -1, -1, -1, -1, -1},
    {9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6, -1, -1, -1, -1},
    {6, 8, 4, 6, 11, 8, 2, 10, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6, -1, -1, -1, -1},
    {4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9, -1, -1, -1, -1},
    {10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3, -1},
    {8, 2, 3, 8, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1},
    {0, 4, 2, 4, 6, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8, -1, -1, -1, -1},
    {1, 9, 4, 1, 4, 2, 2, 4, 6, -1, -1, -1, -1, -1, -1, -1},
    {8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1, -1, -1, -1, -1},
    {10, 1, 0, 10, 0, 6, 6, 0, 4, -1, -1, -1, -1, -1, -1, -1},
    {4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3, -1},
    {10, 9, 4, 6, 10, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 5, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 4, 9, 5, 11, 7, 6, -1, -1, -1, -1, -1, -1, -1},
    {5, 0, 1, 5, 4, 0, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
    {11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5, -1, -1, -1, -1},
    {9, 5, 4, 10, 1, 2, 7, 6, 11, -1, -1, -1, -1, -1, -1, -1},
    {6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5, -1, -1, -1, -1},
    {7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2, -1, -1, -1, -1},
    {3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6, -1},
    {7, 2, 3, 7, 6, 2, 5, 4, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7, -1, -1, -1, -1},
    {3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0, -1, -1, -1, -1},
    {6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8, -1},
    {9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7, -1, -1, -1, -1},
    {1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4, -1},
    {4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10, -1},
    {7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10, -1, -1, -1, -1},
    {6, 9, 5, 6, 11, 9, 11, 8, 9, -1, -1, -1, -1, -1, -1, -1},
    {3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5, -1, -1, -1, -1},
    {0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11, -1, -1, -1, -1},
    {6, 11, 3, 6, 3, 5, 5, 3, 1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6, -1, -1, -1, -1},
    {0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10, -1},
    {11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5, -1},
    {6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3, -1, -1, -1, -1},
    {5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2, -1, -1, -1, -1},
    {9, 5, 6, 9, 6, 0, 0, 6, 2, -1, -1, -1, -1, -1, -1, -1},
    {1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8, -1},
    {1, 5, 6, 2, 1, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6, -1},
    {10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0, -1, -1, -1, -1},
    {0, 3, 8, 5, 6, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {10, 5, 6, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 5, 10, 7, 5, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {11, 5, 10, 11, 7, 5, 8, 3, 0, -1, -1, -1, -1, -1, -1, -1},
    {5, 11, 7, 5, 10, 11, 1, 9, 0, -1, -1, -1, -1, -1, -1, -1},
    {10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1, -1, -1, -1, -1},
    {11, 1, 2, 11, 7, 1, 7, 5, 1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11, -1, -1, -1, -1},
    {9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7, -1, -1, -1, -1},
    {7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2, -1},
    {2, 5, 10, 2, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1},
    {8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5, -1, -1, -1, -1},
    {9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2, -1, -1, -1, -1},
    {9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2, -1},
    {1, 3, 5, 3, 7, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 7, 0, 7, 1, 1, 7, 5, -1, -1, -1, -1, -1, -1, -1},
    {9, 0, 3, 9, 3, 5, 5, 3, 7, -1, -1, -1, -1, -1, -1, -1},
    {9, 8, 7, 5, 9, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {5, 8, 4, 5, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1},
    {5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0, -1, -1, -1, -1},
    {0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5, -1, -1, -1, -1},
    {10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4, -1},
    {2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8, -1, -1, -1, -1},
    {0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11, -1},
    {0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5, -1},
    {9, 4, 5, 2, 11, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4, -1, -1, -1, -1},
    {5, 10, 2, 5, 2, 4, 4, 2, 0, -1, -1, -1, -1, -1, -1, -1},
    {3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9, -1},
    {5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2, -1, -1, -1, -1},
    {8, 4, 5, 8, 5, 3, 3, 5, 1, -1, -1, -1, -1, -1, -1, -1},
    {0, 4, 5, 1, 0, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5, -1, -1, -1, -1},
    {9, 4, 5, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 11, 7, 4, 9, 11, 9, 10, 11, -1, -1, -1, -1, -1, -1, -1},
    {0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11, -1, -1, -1, -1},
    {1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11, -1, -1, -1, -1},
    {3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4, -1},
    {4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2, -1, -1, -1, -1},
    {9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3, -1},
    {11, 7, 4, 11, 4, 2, 2, 4, 0, -1, -1, -1, -1, -1, -1, -1},
    {11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4, -1, -1, -1, -1},
    {2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9, -1, -1, -1, -1},
    {9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7, -1},
    {3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10, -1},
    {1, 10, 2, 8, 7, 4, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 1, 4, 1, 7, 7, 1, 3, -1, -1, -1, -1, -1, -1, -1},
    {4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1, -1, -1, -1, -1},
    {4, 0, 3, 7, 4, 3, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {4, 8, 7, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {9, 10, 8, 10, 11, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 9, 3, 9, 11, 11, 9, 10, -1, -1, -1, -1, -1, -1, -1},
    {0, 1, 10, 0, 10, 8, 8, 10, 11, -1, -1, -1, -1, -1, -1, -1},
    {3, 1, 10, 11, 3, 10, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 2, 11, 1, 11, 9, 9, 11, 8, -1, -1, -1, -1, -1, -1, -1},
    {3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9, -1, -1, -1, -1},
    {0, 2, 11, 8, 0, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {3, 2, 11, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 10, 10, 8, 9, -1, -1, -1, -1, -1, -1, -1},
    {9, 10, 2, 0, 9, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8, -1, -1, -1, -1},
    {1, 10, 2, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {1, 3, 8, 9, 1, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 9, 1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {0, 3, 8, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
    {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1},
};

struct Volume {
  const float* tsdf;
  const float* weight;
  int nx, ny, cx, cy;   // voxels and cubes along x and y
  long ncubes;
  // the case of cube c, or -1 when a corner has weight 0 (or c is past the last cube)
  __device__ int cube_case(long c, int& i, int& j, int& k) const {
    if (c >= ncubes) return -1;
    const long plane = (long)cx * cy;
    k = (int)(c / plane);
    const long r = c - (long)k * plane;
    j = (int)(r / cx);
    i = (int)(r - (long)j * cx);
    int ci = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const long o = ((long)(k + kCorner[q][2]) * ny + (j + kCorner[q][1])) * nx + (i + kCorner[q][0]);
      if (!(__ldg(weight + o) > 0.0f)) return -1;
      ci |= (__ldg(tsdf + o) < 0.0f) << q;
    }
    return ci;
  }
};

__device__ __forceinline__ int tri_count(int ci) {
  if (ci < 0) return 0;
  int m = 0;
  while (m < 5 && kTriTable[ci][3 * m] >= 0) ++m;
  return m;
}

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(Volume vol, int* __restrict__ tile_counts) {
  __shared__ int s_warp[kMcWarps];
  const long base = (long)blockIdx.x * kMcTile + threadIdx.x;
  int c = 0;
  for (int r = 0; r < kMcRounds; ++r) {
    int i, j, k;
    c += tri_count(vol.cube_case(base + r * kMcThreads, i, j, k));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
#pragma unroll
    for (int q = 0; q < kMcWarps; ++q) s += s_warp[q];
    tile_counts[blockIdx.x] = s;
  }
}

// One CTA: tile_first[t] = the triangles of tiles 0..t-1, and *total = all of them.
__global__ void __launch_bounds__(kScanThreads) mc_offsets_kernel(const int* __restrict__ tile_counts, int tiles,
                                                                  int64_t* __restrict__ tile_first, int64_t* __restrict__ total) {
  __shared__ int64_t s_sum[kScanThreads];
  const int seg = (tiles + kScanThreads - 1) / kScanThreads;
  const int b = threadIdx.x * seg, e = min(tiles, b + seg);
  int64_t s = 0;
  for (int q = b; q < e; ++q) s += tile_counts[q];
  s_sum[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {   // 1024 additions: not worth a tree
    int64_t run = 0;
    for (int q = 0; q < kScanThreads; ++q) {
      const int64_t v = s_sum[q];
      s_sum[q] = run;
      run += v;
    }
    *total = run;
  }
  __syncthreads();
  int64_t run = s_sum[threadIdx.x];
  for (int q = b; q < e; ++q) {
    tile_first[q] = run;
    run += tile_counts[q];
  }
}

template <bool kColor>
__global__ void __launch_bounds__(kMcThreads) mc_scatter_kernel(Volume vol, const float* __restrict__ color, float ox, float oy, float oz,
                                                                 float vs, const int64_t* __restrict__ tile_first,
                                                                 float* __restrict__ vertices, uint8_t* __restrict__ colors_out,
                                                                 int* __restrict__ faces) {
  __shared__ int s_warp[kMcWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long base = (long)blockIdx.x * kMcTile + threadIdx.x;
  long row = tile_first[blockIdx.x];   // first triangle of round r in this tile
  const float org[3] = {ox, oy, oz};
  for (int r = 0; r < kMcRounds; ++r) {
    int i = 0, j = 0, k = 0;
    const int ci = vol.cube_case(base + r * kMcThreads, i, j, k);
    const int cnt = tri_count(ci);
    int incl = cnt;   // inclusive scan of the counts over the warp's lanes
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    __syncthreads();   // s_warp of the previous round has been read
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int q = 0; q < kMcWarps; ++q) {
      const int v = s_warp[q];
      total += v;
      before += q < warp ? v : 0;
    }
    if (cnt) {
      const int g[3] = {i, j, k};
      long tri = row + before + incl - cnt;
      for (int m = 0; m < cnt; ++m, ++tri) {
        for (int e3 = 0; e3 < 3; ++e3) {
          const int edge = kTriTable[ci][3 * m + e3];
          const int qa = kEdge[edge][0], qb = kEdge[edge][1];
          long oa = 0, ob = 0;
          float pa[3], pb[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const int ia = g[a] + kCorner[qa][a], ib = g[a] + kCorner[qb][a];
            pa[a] = fadd(org[a], fmul(vs, (float)ia));
            pb[a] = fadd(org[a], fmul(vs, (float)ib));
          }
          oa = ((long)(k + kCorner[qa][2]) * vol.ny + (j + kCorner[qa][1])) * vol.nx + (i + kCorner[qa][0]);
          ob = ((long)(k + kCorner[qb][2]) * vol.ny + (j + kCorner[qb][1])) * vol.nx + (i + kCorner[qb][0]);
          const float fa = __ldg(vol.tsdf + oa), fb = __ldg(vol.tsdf + ob);
          const float mu = fdiv(fa, fsub(fa, fb));   // fa and fb lie on either side of 0, so fa - fb != 0
          const long vtx = 3 * tri + e3;
#pragma unroll
          for (int a = 0; a < 3; ++a) vertices[3 * vtx + a] = fadd(pa[a], fmul(mu, fsub(pb[a], pa[a])));
          if (kColor) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
              const float ca = __ldg(color + 3 * oa + a), cb = __ldg(color + 3 * ob + a);
              const int q = __float2int_rn(fadd(ca, fmul(mu, fsub(cb, ca))));   // half to even
              colors_out[3 * vtx + a] = (uint8_t)min(255, max(0, q));
            }
          }
          faces[vtx] = (int)vtx;
        }
      }
    }
    row += total;
  }
}

long mc_tiles(int nx, int ny, int nz) {
  const long ncubes = (long)(nx - 1) * (ny - 1) * (nz - 1);
  return (ncubes + kMcTile - 1) / kMcTile;
}

// every volume entry: a non-empty box of at most 2^31 - 1 voxels, and a vertex index of every possible triangle fits int32
int check_volume(const char* name, int nx, int ny, int nz) {
  DEMON_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "%s: the volume needs at least 2 voxels along each axis, got %dx%dx%d", name, nx, ny, nz);
  const long ncubes = (long)(nx - 1) * (ny - 1) * (nz - 1);
  DEMON_REQUIRE((long)nx * ny * nz < (1L << 31) && 15 * ncubes < (1L << 31), "%s: volume %dx%dx%d is too large", name, nx, ny, nz);
  return DEMON_OK;
}

Volume make_volume(const float* tsdf, const float* weight, int nx, int ny, int nz) {
  return Volume{tsdf, weight, nx, ny, nx - 1, ny - 1, (long)(nx - 1) * (ny - 1) * (nz - 1)};
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int demon_tsdf_integrate_f32(float* tsdf, float* weight, float* color, int nx, int ny, int nz, const float* origin, float voxel_size,
                             float trunc, const float* depth, const float* K, const float* R, const float* t, const uint8_t* image,
                             int n, int h, int w, void* stream) {
  if (int rc = check_volume("tsdf_integrate", nx, ny, nz)) return rc;
  DEMON_REQUIRE(n >= 0 && h >= 1 && w >= 1 && (long)h * w < (1L << 24), "tsdf_integrate: bad size %d frames of %dx%d", n, h, w);
  DEMON_REQUIRE(origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]),
                "tsdf_integrate: the origin must be finite");
  DEMON_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0f && std::isfinite(trunc) && trunc > 0.0f,
                "tsdf_integrate: voxel_size and trunc must be finite and > 0, got %g and %g", voxel_size, trunc);
  DEMON_REQUIRE(!color == !image, "tsdf_integrate: color and image go together");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(tsdf && weight && depth && K && R && t, "tsdf_integrate: null pointer");
  const long nvox = (long)nx * ny * nz;
  const unsigned blocks = (unsigned)((nvox + kFuseThreads - 1) / kFuseThreads);
  if (color)
    tsdf_integrate_kernel<true><<<blocks, kFuseThreads, 0, (cudaStream_t)stream>>>(
        tsdf, weight, color, nx, ny, nvox, origin[0], origin[1], origin[2], voxel_size, trunc, depth, K, R, t, image, n, h, w);
  else
    tsdf_integrate_kernel<false><<<blocks, kFuseThreads, 0, (cudaStream_t)stream>>>(
        tsdf, weight, nullptr, nx, ny, nvox, origin[0], origin[1], origin[2], voxel_size, trunc, depth, K, R, t, nullptr, n, h, w);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int64_t demon_marching_cubes_scratch_bytes(int nx, int ny, int nz) {
  if (check_volume("marching_cubes_scratch_bytes", nx, ny, nz)) return 0;
  return mc_tiles(nx, ny, nz) * (int64_t)(sizeof(int64_t) + sizeof(int));
}

int demon_marching_cubes_count_f32(const float* tsdf, const float* weight, int nx, int ny, int nz, void* scratch, int64_t* triangles,
                                   void* stream) {
  if (int rc = check_volume("marching_cubes_count", nx, ny, nz)) return rc;
  DEMON_REQUIRE(tsdf && weight && scratch && triangles, "marching_cubes_count: null pointer");
  const int tiles = (int)mc_tiles(nx, ny, nz);
  int64_t* tile_first = static_cast<int64_t*>(scratch);   // scratch: tile_first [tiles], tile_counts [tiles]
  int* tile_counts = reinterpret_cast<int*>(tile_first + tiles);
  mc_count_kernel<<<tiles, kMcThreads, 0, (cudaStream_t)stream>>>(make_volume(tsdf, weight, nx, ny, nz), tile_counts);
  DEMON_LAUNCH_CHECK();
  mc_offsets_kernel<<<1, kScanThreads, 0, (cudaStream_t)stream>>>(tile_counts, tiles, tile_first, triangles);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_marching_cubes_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                             float voxel_size, const void* scratch, float* vertices, uint8_t* colors, int* faces, void* stream) {
  if (int rc = check_volume("marching_cubes", nx, ny, nz)) return rc;
  DEMON_REQUIRE(origin && std::isfinite(voxel_size) && voxel_size > 0.0f, "marching_cubes: bad origin or voxel_size %g", voxel_size);
  DEMON_REQUIRE(!color == !colors, "marching_cubes: color and colors go together");
  DEMON_REQUIRE(tsdf && weight && scratch && vertices && faces, "marching_cubes: null pointer");
  const int tiles = (int)mc_tiles(nx, ny, nz);
  const Volume vol = make_volume(tsdf, weight, nx, ny, nz);
  const int64_t* tile_first = static_cast<const int64_t*>(scratch);
  if (color)
    mc_scatter_kernel<true><<<tiles, kMcThreads, 0, (cudaStream_t)stream>>>(vol, color, origin[0], origin[1], origin[2], voxel_size,
                                                                           tile_first, vertices, colors, faces);
  else
    mc_scatter_kernel<false><<<tiles, kMcThreads, 0, (cudaStream_t)stream>>>(vol, nullptr, origin[0], origin[1], origin[2], voxel_size,
                                                                            tile_first, vertices, nullptr, faces);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // extern "C"
