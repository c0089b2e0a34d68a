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
// * the sparse volume: 8x8x8 voxel blocks in a hash table.  sparse_allocate_kernel inserts, one thread per pixel, the blocks
//   around each pixel's band cell; the new keys are gathered, sorted by the caller and committed in that order; the
//   integration and marching cubes run the dense code above on every block (tsdf_integrate_frames, SparseVolume).
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
struct VoxelState {
  float s, W, c0, c1, c2;
};

// One frame's update of one voxel; cm is the frame's staged camera and p0 the frame's first pixel.
template <bool kColor>
__device__ __forceinline__ void tsdf_update(const float* cm, float X0, float X1, float X2, float trunc, const float* __restrict__ depth,
                                            const uint8_t* __restrict__ image, long p0, int w, float fw, float fh, VoxelState& st) {
  const float z = fadd(fadd(fadd(fmul(cm[10], X0), fmul(cm[11], X1)), fmul(cm[12], X2)), cm[15]);
  if (!(z > 0.0f)) return;
  const float x = fadd(fadd(fadd(fmul(cm[4], X0), fmul(cm[5], X1)), fmul(cm[6], X2)), cm[13]);
  const float y = fadd(fadd(fadd(fmul(cm[7], X0), fmul(cm[8], X1)), fmul(cm[9], X2)), cm[14]);
  const float u = fadd(fdiv(fmul(cm[0], x), z), cm[2]);
  const float v = fadd(fdiv(fmul(cm[1], y), z), cm[3]);
  if (!(u >= 0.0f && u < fw && v >= 0.0f && v < fh)) return;   // floor(u) in [0, w) and floor(v) in [0, h)
  const long p = p0 + (long)(int)v * w + (int)u;
  const float d = __ldg(depth + p);
  if (!(isfinite(d) && d > 0.0f)) return;
  const float sdf = fsub(d, z);
  if (sdf < -trunc) return;
  const float fv = fminf(1.0f, fdiv(sdf, trunc));
  const float W1 = fadd(st.W, 1.0f);
  st.s = fdiv(fadd(fmul(st.s, st.W), fv), W1);
  if (kColor) {
    const uint8_t* px = image + 3 * p;
    st.c0 = fdiv(fadd(fmul(st.c0, st.W), (float)__ldg(px)), W1);
    st.c1 = fdiv(fadd(fmul(st.c1, st.W), (float)__ldg(px + 1)), W1);
    st.c2 = fdiv(fadd(fmul(st.c2, st.W), (float)__ldg(px + 2)), W1);
  }
  st.W = W1;
}

// The n frames of a call, in order, on the state of the thread's voxel X (every thread of the CTA calls this: it stages the
// cameras of kFuseChunk frames at a time in shared memory).
template <bool kColor>
__device__ __forceinline__ void tsdf_integrate_frames(bool active, float X0, float X1, float X2, float trunc, const float* __restrict__ depth,
                                                      const float* __restrict__ K, const float* __restrict__ R, const float* __restrict__ t,
                                                      const uint8_t* __restrict__ image, int n, int h, int w, VoxelState& st) {
  __shared__ float cam[kFuseChunk][kCam];
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
    for (int fr = 0; fr < m; ++fr) tsdf_update<kColor>(cam[fr], X0, X1, X2, trunc, depth, image, (long)(f0 + fr) * hw, w, fw, fh, st);
  }
}

template <bool kColor>
__device__ __forceinline__ void load_state(const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ color,
                                           long vox, VoxelState& st) {
  st.s = tsdf[vox];
  st.W = weight[vox];
  if (kColor) {
    st.c0 = color[3 * vox];
    st.c1 = color[3 * vox + 1];
    st.c2 = color[3 * vox + 2];
  }
}

template <bool kColor>
__device__ __forceinline__ void store_state(float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color, long vox,
                                            const VoxelState& st) {
  tsdf[vox] = st.s;
  weight[vox] = st.W;
  if (kColor) {
    color[3 * vox] = st.c0;
    color[3 * vox + 1] = st.c1;
    color[3 * vox + 2] = st.c2;
  }
}

template <bool kColor>
__global__ void __launch_bounds__(kFuseThreads) tsdf_integrate_kernel(
    float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color, int nx, int ny, long nvox, float ox, float oy,
    float oz, float vs, float trunc, const float* __restrict__ depth, const float* __restrict__ K, const float* __restrict__ R,
    const float* __restrict__ t, const uint8_t* __restrict__ image, int n, int h, int w) {
  const long vox = (long)blockIdx.x * kFuseThreads + threadIdx.x;
  const bool active = vox < nvox;
  VoxelState st = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
  float X0 = 0.0f, X1 = 0.0f, X2 = 0.0f;
  if (active) {
    load_state<kColor>(tsdf, weight, color, vox, st);
    const long plane = (long)nx * ny;
    const int k = (int)(vox / plane);
    const long r = vox - (long)k * plane;
    const int j = (int)(r / nx), i = (int)(r - (long)j * nx);
    X0 = fadd(ox, fmul(vs, (float)i));
    X1 = fadd(oy, fmul(vs, (float)j));
    X2 = fadd(oz, fmul(vs, (float)k));
  }
  tsdf_integrate_frames<kColor>(active, X0, X1, X2, trunc, depth, K, R, t, image, n, h, w, st);
  if (active) store_state<kColor>(tsdf, weight, color, vox, st);
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

// The cubes of the dense box: cube c has its lower corner at voxel (i, j, k), i fastest.
struct DenseVolume {
  const float* tsdf;
  const float* weight;
  int nx, ny, cx, cy;   // voxels and cubes along x and y
  long ncubes;
  struct Cube {
    int g[3];   // grid coordinate of corner 0
  };
  __device__ bool locate(long c, Cube& cb) const {
    if (c >= ncubes) return false;
    const long plane = (long)cx * cy;
    const int k = (int)(c / plane);
    const long r = c - (long)k * plane;
    const int j = (int)(r / cx);
    cb.g[0] = (int)(r - (long)j * cx);
    cb.g[1] = j;
    cb.g[2] = k;
    return true;
  }
  // the state index of corner q
  __device__ long corner(const Cube& cb, int q) const {
    return ((long)(cb.g[2] + kCorner[q][2]) * ny + (cb.g[1] + kCorner[q][1])) * nx + (cb.g[0] + kCorner[q][0]);
  }
};

// The cubes of the hashed blocks: cube c has its lower corner at local voxel c % 512 (x fastest) of block c / 512, and
// its corners past the block's last voxel lie in the +x, +y, +z neighbours nbr[8 b + (dx | dy << 1 | dz << 2)].
struct SparseVolume {
  const float* tsdf;
  const float* weight;
  const int* blocks;   // [m,3] block coordinates
  const int* nbr;      // [m,8] pool index of block b + (dx, dy, dz), or -1
  long ncubes;
  struct Cube {
    int b;      // pool index
    int l[3];   // local voxel of corner 0
    int g[3];   // grid coordinate of corner 0: 8 * block + l
  };
  __device__ bool locate(long c, Cube& cb) const {
    if (c >= ncubes) return false;
    cb.b = (int)(c >> 9);
    const int r = (int)(c & 511);
    cb.l[0] = r & 7;
    cb.l[1] = (r >> 3) & 7;
    cb.l[2] = r >> 6;
#pragma unroll
    for (int a = 0; a < 3; ++a) cb.g[a] = 8 * __ldg(blocks + 3 * cb.b + a) + cb.l[a];
    return true;
  }
  // the state index of corner q, or -1 when its block is not allocated
  __device__ long corner(const Cube& cb, int q) const {
    const int x = cb.l[0] + kCorner[q][0], y = cb.l[1] + kCorner[q][1], z = cb.l[2] + kCorner[q][2];
    const int nb = (x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2);
    const int blk = nb ? __ldg(nbr + 8 * cb.b + nb) : cb.b;
    if (blk < 0) return -1;
    return ((long)blk << 9) + ((z & 7) << 6) + ((y & 7) << 3) + (x & 7);
  }
};

// the case of cube c, or -1 when a corner is not stored or has weight 0 (or c is past the last cube)
template <class V>
__device__ __forceinline__ int cube_case(const V& vol, long c, typename V::Cube& cb) {
  if (!vol.locate(c, cb)) return -1;
  int ci = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const long o = vol.corner(cb, q);
    if (o < 0 || !(__ldg(vol.weight + o) > 0.0f)) return -1;
    ci |= (__ldg(vol.tsdf + o) < 0.0f) << q;
  }
  return ci;
}

__device__ __forceinline__ int tri_count(int ci) {
  if (ci < 0) return 0;
  int m = 0;
  while (m < 5 && kTriTable[ci][3 * m] >= 0) ++m;
  return m;
}

template <class V>
__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(V vol, int* __restrict__ tile_counts) {
  __shared__ int s_warp[kMcWarps];
  const long base = (long)blockIdx.x * kMcTile + threadIdx.x;
  int c = 0;
  for (int r = 0; r < kMcRounds; ++r) {
    typename V::Cube cb;
    c += tri_count(cube_case(vol, base + r * kMcThreads, cb));
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

template <bool kColor, class V>
__global__ void __launch_bounds__(kMcThreads) mc_scatter_kernel(V vol, const float* __restrict__ color, float ox, float oy, float oz,
                                                                 float vs, const int64_t* __restrict__ tile_first,
                                                                 float* __restrict__ vertices, uint8_t* __restrict__ colors_out,
                                                                 int* __restrict__ faces) {
  __shared__ int s_warp[kMcWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long base = (long)blockIdx.x * kMcTile + threadIdx.x;
  long row = tile_first[blockIdx.x];   // first triangle of round r in this tile
  const float org[3] = {ox, oy, oz};
  for (int r = 0; r < kMcRounds; ++r) {
    typename V::Cube cb;
    const int ci = cube_case(vol, base + r * kMcThreads, cb);
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
      long tri = row + before + incl - cnt;
      for (int m = 0; m < cnt; ++m, ++tri) {
        for (int e3 = 0; e3 < 3; ++e3) {
          const int edge = kTriTable[ci][3 * m + e3];
          const int qa = kEdge[edge][0], qb = kEdge[edge][1];
          float pa[3], pb[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const int ia = cb.g[a] + kCorner[qa][a], ib = cb.g[a] + kCorner[qb][a];
            pa[a] = fadd(org[a], fmul(vs, (float)ia));
            pb[a] = fadd(org[a], fmul(vs, (float)ib));
          }
          const long oa = vol.corner(cb, qa), ob = vol.corner(cb, qb);
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

DenseVolume make_volume(const float* tsdf, const float* weight, int nx, int ny, int nz) {
  return DenseVolume{tsdf, weight, nx, ny, nx - 1, ny - 1, (long)(nx - 1) * (ny - 1) * (nz - 1)};
}

// ---- sparse volume: voxel blocks in a hash table -------------------------------------------------------------------------
// Block (bx, by, bz), |b| <= kMaxBlockCoord per axis, holds voxels 8 b + (0..7) in the pool at its index: tsdf and weight
// [m,8,8,8] (z, y, x; x fastest), colour [m,8,8,8,3].  The table maps the packed key of a block to its pool index, by open
// addressing with linear probing over `capacity` (a power of 2) slots: key -1 marks an empty slot, value -1 a block
// inserted by the running call's allocation and not yet given a pool index.
constexpr int kSparseThreads = 256;
constexpr int kMaxBlockCoord = DEMON_SPARSE_TSDF_MAX_COORD;
constexpr int kMaxSpan = DEMON_SPARSE_TSDF_MAX_SPAN;
constexpr unsigned long long kEmptyKey = ~0ull;
// counters[]: 0 occupied slots, 1 the table reached half its capacity, 2 skipped pixels, 3 the gather's cursor
enum { kOccupied = 0, kOverflow = 1, kSkipped = 2, kCursor = 3 };

__device__ __forceinline__ unsigned long long block_key(int bx, int by, int bz) {
  const unsigned long long o = 1ull << 20;
  return ((unsigned long long)(bz + o) << 42) | ((unsigned long long)(by + o) << 21) | (unsigned long long)(bx + o);
}

__device__ __forceinline__ int key_coord(unsigned long long key, int a) { return (int)((key >> (21 * a)) & ((1u << 21) - 1)) - (1 << 20); }

__device__ __forceinline__ long key_slot(unsigned long long key, long mask) {   // the splitmix64 finaliser
  key ^= key >> 30;
  key *= 0xbf58476d1ce4e5b9ull;
  key ^= key >> 27;
  key *= 0x94d049bb133111ebull;
  key ^= key >> 31;
  return (long)(key & (unsigned long long)mask);
}

// the slot of key, or -1 (the table is not written while this runs)
__device__ __forceinline__ long find_slot(const unsigned long long* __restrict__ keys, long mask, unsigned long long key) {
  for (long s = key_slot(key, mask);; s = (s + 1) & mask) {
    const unsigned long long k = __ldg(keys + s);
    if (k == key) return s;
    if (k == kEmptyKey) return -1;
  }
}

// Inserts key unless present.  A thread takes one of the `limit` slots the table may fill before it claims an empty one, so
// the table never holds more than `limit` keys and always has an empty slot to end a probe; false when none is left.
__device__ __forceinline__ bool insert_key(unsigned long long* keys, long mask, unsigned long long key, unsigned long long* occupied,
                                           unsigned long long limit) {
  bool reserved = false;
  for (long s = key_slot(key, mask);; s = (s + 1) & mask) {
    unsigned long long k = *(volatile unsigned long long*)(keys + s);
    if (k == kEmptyKey) {
      if (!reserved) {
        if (atomicAdd(occupied, 1ull) >= limit) return false;
        reserved = true;
      }
      k = atomicCAS(keys + s, kEmptyKey, key);
      if (k == kEmptyKey) return true;
    }
    if (k == key) {
      if (reserved) atomicAdd(occupied, ~0ull);   // give the slot back
      return true;
    }
  }
}

// The world-space AABB of a pixel's band cell, point by point.
struct Cell {
  const float* R;
  float t0, t1, t2;
  float lo0 = INFINITY, lo1 = INFINITY, lo2 = INFINITY, hi0 = -INFINITY, hi1 = -INFINITY, hi2 = -INFINITY;
  bool finite = true;
  __device__ __forceinline__ void axis(float X, float& lo, float& hi) {
    finite = finite && isfinite(X);
    lo = fminf(lo, X);
    hi = fmaxf(hi, X);
  }
  // camera point (x, y, z) -> X = R^T ((x, y, z) - t)
  __device__ __forceinline__ void add(float x, float y, float z) {
    const float e0 = fsub(x, t0), e1 = fsub(y, t1), e2 = fsub(z, t2);
    axis(fadd(fadd(fmul(__ldg(R), e0), fmul(__ldg(R + 3), e1)), fmul(__ldg(R + 6), e2)), lo0, hi0);
    axis(fadd(fadd(fmul(__ldg(R + 1), e0), fmul(__ldg(R + 4), e1)), fmul(__ldg(R + 7), e2)), lo1, hi1);
    axis(fadd(fadd(fmul(__ldg(R + 2), e0), fmul(__ldg(R + 5), e1)), fmul(__ldg(R + 8), e2)), lo2, hi2);
  }
};

// The blocks [b0, b1] along one axis of the AABB [lo, hi] widened by 2 voxels; false past the key range or kMaxSpan.
__device__ __forceinline__ bool block_range(float lo, float hi, float o, float vs, int& b0, int& b1) {
  const float fl = floorf(fmul(fsub(fdiv(fsub(lo, o), vs), 2.0f), 0.125f));
  const float fh = floorf(fmul(fadd(fdiv(fsub(hi, o), vs), 2.0f), 0.125f));
  if (!(fl >= (float)-kMaxBlockCoord && fh <= (float)kMaxBlockCoord)) return false;
  b0 = (int)fl;
  b1 = (int)fh;
  return b1 - b0 < kMaxSpan;
}

// One thread per pixel of every frame: the pixel's band cell (its pixel square between camera z d - trunc and d + trunc,
// the near face replaced by the camera centre when d - trunc <= 0) in world space, its AABB widened by 2 voxels, and every
// block that AABB overlaps.  The float operations, in this order:
//   zf = d + trunc, zn = d - trunc;  for the corners (u, v) in {px, px+1} x {py, py+1}: a = (u - cx) / fx, b = (v - cy) / fy,
//   points (a zf, b zf, zf) and, when zn > 0, (a zn, b zn, zn);  when zn <= 0 the point (0, 0, 0);
//   world X_i = (R_0i (x - t_0) + R_1i (y - t_1)) + R_2i (z - t_2);  lo, hi = the min and max over the points;
//   block range floor(((lo - o) / vs - 2) * 0.125) .. floor(((hi - o) / vs + 2) * 0.125).
// A pixel with a non-finite point, a range past +-kMaxBlockCoord or more than kMaxSpan blocks along an axis is skipped.
__global__ void __launch_bounds__(kSparseThreads) sparse_allocate_kernel(
    unsigned long long* __restrict__ keys, long mask, unsigned long long limit, unsigned long long* __restrict__ counters, float ox, float oy,
    float oz, float vs, float trunc, const float* __restrict__ depth, const float* __restrict__ K, const float* __restrict__ R,
    const float* __restrict__ t, long npix, int h, int w) {
  const long p = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (p >= npix) return;
  const float d = __ldg(depth + p);
  if (!(isfinite(d) && d > 0.0f)) return;
  const long hw = (long)h * w;
  const int f = (int)(p / hw);
  const int pix = (int)(p - (long)f * hw), py = pix / w, px = pix - py * w;
  const float fx = __ldg(K + 9 * f), cx = __ldg(K + 9 * f + 2), fy = __ldg(K + 9 * f + 4), cy = __ldg(K + 9 * f + 5);
  Cell cell;
  cell.R = R + 9 * f;
  cell.t0 = __ldg(t + 3 * f);
  cell.t1 = __ldg(t + 3 * f + 1);
  cell.t2 = __ldg(t + 3 * f + 2);
  const float zf = fadd(d, trunc), zn = fsub(d, trunc);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float a = fdiv(fsub((float)(px + (c & 1)), cx), fx), b = fdiv(fsub((float)(py + (c >> 1)), cy), fy);
    cell.add(fmul(a, zf), fmul(b, zf), zf);
    if (zn > 0.0f) cell.add(fmul(a, zn), fmul(b, zn), zn);
  }
  if (!(zn > 0.0f)) cell.add(0.0f, 0.0f, 0.0f);
  int b0x, b1x, b0y, b1y, b0z, b1z;
  const bool ok = cell.finite && block_range(cell.lo0, cell.hi0, ox, vs, b0x, b1x) && block_range(cell.lo1, cell.hi1, oy, vs, b0y, b1y) &&
                  block_range(cell.lo2, cell.hi2, oz, vs, b0z, b1z);
  if (!ok) {
    atomicAdd(counters + kSkipped, 1ull);
    return;
  }
  for (int bz = b0z; bz <= b1z; ++bz)
    for (int by = b0y; by <= b1y; ++by)
      for (int bx = b0x; bx <= b1x; ++bx)
        if (!insert_key(keys, mask, block_key(bx, by, bz), counters + kOccupied, limit)) {
          counters[kOverflow] = 1ull;
          return;
        }
}

// Moves every entry of the old table into the new, empty one and counts them.
__global__ void __launch_bounds__(kSparseThreads) sparse_rehash_kernel(const unsigned long long* __restrict__ old_keys,
                                                                       const int* __restrict__ old_values, long old_capacity,
                                                                       unsigned long long* __restrict__ keys, int* __restrict__ values,
                                                                       long mask, unsigned long long* __restrict__ counters) {
  const long s = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (s >= old_capacity) return;
  const unsigned long long key = old_keys[s];
  if (key == kEmptyKey) return;
  for (long q = key_slot(key, mask);; q = (q + 1) & mask)
    if (atomicCAS(keys + q, kEmptyKey, key) == kEmptyKey) {
      values[q] = old_values[s];
      atomicAdd(counters + kOccupied, 1ull);
      return;
    }
}

// The keys without a pool index, in slot-claiming order (the caller sorts them).
__global__ void __launch_bounds__(kSparseThreads) sparse_gather_kernel(const unsigned long long* __restrict__ keys,
                                                                       const int* __restrict__ values, long capacity,
                                                                       unsigned long long* __restrict__ counters, int64_t* __restrict__ out) {
  const long s = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (s >= capacity) return;
  const unsigned long long key = keys[s];
  if (key != kEmptyKey && values[s] < 0) out[atomicAdd(counters + kCursor, 1ull)] = (int64_t)key;
}

// Key i of the sorted new keys gets pool index first + i.
__global__ void __launch_bounds__(kSparseThreads) sparse_commit_kernel(const unsigned long long* __restrict__ keys, int* __restrict__ values,
                                                                       long mask, const int64_t* __restrict__ sorted, int count, int first,
                                                                       int* __restrict__ blocks) {
  const int i = blockIdx.x * kSparseThreads + threadIdx.x;
  if (i >= count) return;
  const unsigned long long key = (unsigned long long)sorted[i];
  values[find_slot(keys, mask, key)] = first + i;
#pragma unroll
  for (int a = 0; a < 3; ++a) blocks[3 * (long)(first + i) + a] = key_coord(key, a);
}

// One thread per voxel of every block: the dense kernel's frame loop at voxel 8 b + l.
template <bool kColor>
__global__ void __launch_bounds__(kFuseThreads) sparse_tsdf_integrate_kernel(
    float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color, const int* __restrict__ blocks, long nvox, float ox,
    float oy, float oz, float vs, float trunc, const float* __restrict__ depth, const float* __restrict__ K, const float* __restrict__ R,
    const float* __restrict__ t, const uint8_t* __restrict__ image, int n, int h, int w) {
  const long vox = (long)blockIdx.x * kFuseThreads + threadIdx.x;
  const bool active = vox < nvox;
  VoxelState st = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
  float X0 = 0.0f, X1 = 0.0f, X2 = 0.0f;
  if (active) {
    load_state<kColor>(tsdf, weight, color, vox, st);
    const long b = vox >> 9;
    const int l = (int)(vox & 511);
    X0 = fadd(ox, fmul(vs, (float)(8 * __ldg(blocks + 3 * b) + (l & 7))));
    X1 = fadd(oy, fmul(vs, (float)(8 * __ldg(blocks + 3 * b + 1) + ((l >> 3) & 7))));
    X2 = fadd(oz, fmul(vs, (float)(8 * __ldg(blocks + 3 * b + 2) + (l >> 6))));
  }
  tsdf_integrate_frames<kColor>(active, X0, X1, X2, trunc, depth, K, R, t, image, n, h, w, st);
  if (active) store_state<kColor>(tsdf, weight, color, vox, st);
}

// nbr[8 b + q] = the pool index of block b + (q & 1, q >> 1 & 1, q >> 2), or -1.
__global__ void __launch_bounds__(kSparseThreads) sparse_neighbours_kernel(const unsigned long long* __restrict__ keys,
                                                                           const int* __restrict__ values, long mask,
                                                                           const int* __restrict__ blocks, int m, int* __restrict__ nbr) {
  const long e = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (e >= 8L * m) return;
  const long b = e >> 3;
  const int q = (int)(e & 7);
  const int bx = blocks[3 * b] + (q & 1), by = blocks[3 * b + 1] + ((q >> 1) & 1), bz = blocks[3 * b + 2] + (q >> 2);
  long s = -1;
  if (bx <= kMaxBlockCoord && by <= kMaxBlockCoord && bz <= kMaxBlockCoord) s = find_slot(keys, mask, block_key(bx, by, bz));
  nbr[e] = s < 0 ? -1 : __ldg(values + s);
}

int check_table(const char* name, const void* keys, const void* values, int64_t capacity) {
  DEMON_REQUIRE(keys && values, "%s: null table", name);
  DEMON_REQUIRE(capacity >= 2 && (capacity & (capacity - 1)) == 0 && capacity <= (1LL << 40),
                "%s: the table capacity must be a power of 2, got %lld", name, (long long)capacity);
  return DEMON_OK;
}

int check_frames(const char* name, const float* origin, float voxel_size, float trunc, int n, int h, int w) {
  DEMON_REQUIRE(n >= 0 && h >= 1 && w >= 1 && (long)h * w < (1L << 24), "%s: bad size %d frames of %dx%d", name, n, h, w);
  DEMON_REQUIRE(origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]), "%s: the origin must be finite",
                name);
  DEMON_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0f && std::isfinite(trunc) && trunc > 0.0f,
                "%s: voxel_size and trunc must be finite and > 0, got %g and %g", name, voxel_size, trunc);
  return DEMON_OK;
}

int64_t sparse_mc_tiles(int m) { return ((int64_t)m * 512 + kMcTile - 1) / kMcTile; }

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
  const DenseVolume vol = make_volume(tsdf, weight, nx, ny, nz);
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

int demon_sparse_tsdf_rehash(const int64_t* old_keys, const int* old_values, int64_t old_capacity, int64_t* keys, int* values,
                             int64_t capacity, int64_t* counters, void* stream) {
  if (int rc = check_table("sparse_tsdf_rehash", keys, values, capacity)) return rc;
  DEMON_REQUIRE(counters && old_capacity >= 0 && old_capacity <= capacity / 2 && (old_capacity == 0 || (old_keys && old_values)),
                "sparse_tsdf_rehash: bad old table of %lld slots for %lld", (long long)old_capacity, (long long)capacity);
  cudaStream_t st = (cudaStream_t)stream;
  DEMON_CHECK_CUDA(cudaMemsetAsync(keys, 0xff, capacity * sizeof(int64_t), st));
  DEMON_CHECK_CUDA(cudaMemsetAsync(values, 0xff, capacity * sizeof(int), st));
  DEMON_CHECK_CUDA(cudaMemsetAsync(counters, 0, 4 * sizeof(int64_t), st));
  if (old_capacity == 0) return DEMON_OK;
  sparse_rehash_kernel<<<(unsigned)ceil_div64(old_capacity, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(old_keys), old_values, old_capacity, reinterpret_cast<unsigned long long*>(keys), values,
      capacity - 1, reinterpret_cast<unsigned long long*>(counters));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_allocate_f32(int64_t* keys, const int* values, int64_t capacity, int64_t* counters, const float* origin,
                                   float voxel_size, float trunc, const float* depth, const float* K, const float* R, const float* t,
                                   int n, int h, int w, void* stream) {
  if (int rc = check_table("sparse_tsdf_allocate", keys, values, capacity)) return rc;
  if (int rc = check_frames("sparse_tsdf_allocate", origin, voxel_size, trunc, n, h, w)) return rc;
  DEMON_REQUIRE(counters, "sparse_tsdf_allocate: null counters");
  cudaStream_t st = (cudaStream_t)stream;
  DEMON_CHECK_CUDA(cudaMemsetAsync(counters + kOverflow, 0, 2 * sizeof(int64_t), st));
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && K && R && t, "sparse_tsdf_allocate: null pointer");
  const long npix = (long)n * h * w;
  sparse_allocate_kernel<<<(unsigned)ceil_div64(npix, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<unsigned long long*>(keys), capacity - 1, (unsigned long long)(capacity / 2),
      reinterpret_cast<unsigned long long*>(counters), origin[0], origin[1], origin[2], voxel_size, trunc, depth, K, R, t, npix, h, w);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_gather_new(const int64_t* keys, const int* values, int64_t capacity, int64_t* counters, int64_t* new_keys,
                                 void* stream) {
  if (int rc = check_table("sparse_tsdf_gather_new", keys, values, capacity)) return rc;
  DEMON_REQUIRE(counters && new_keys, "sparse_tsdf_gather_new: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  DEMON_CHECK_CUDA(cudaMemsetAsync(counters + kCursor, 0, sizeof(int64_t), st));
  sparse_gather_kernel<<<(unsigned)ceil_div64(capacity, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), values, capacity, reinterpret_cast<unsigned long long*>(counters), new_keys);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_commit(const int64_t* keys, int* values, int64_t capacity, const int64_t* sorted_keys, int count, int first,
                             int* blocks, void* stream) {
  if (int rc = check_table("sparse_tsdf_commit", keys, values, capacity)) return rc;
  DEMON_REQUIRE(count >= 0 && first >= 0 && (int64_t)first + count < (1LL << 31), "sparse_tsdf_commit: bad count %d at %d", count, first);
  if (count == 0) return DEMON_OK;
  DEMON_REQUIRE(sorted_keys && blocks, "sparse_tsdf_commit: null pointer");
  sparse_commit_kernel<<<ceil_div(count, kSparseThreads), kSparseThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned long long*>(keys), values, capacity - 1, sorted_keys, count, first, blocks);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_integrate_f32(float* tsdf, float* weight, float* color, const int* blocks, int m, const float* origin, float voxel_size,
                                    float trunc, const float* depth, const float* K, const float* R, const float* t, const uint8_t* image,
                                    int n, int h, int w, void* stream) {
  if (int rc = check_frames("sparse_tsdf_integrate", origin, voxel_size, trunc, n, h, w)) return rc;
  DEMON_REQUIRE(m >= 0, "sparse_tsdf_integrate: bad block count %d", m);
  DEMON_REQUIRE(!color == !image, "sparse_tsdf_integrate: color and image go together");
  if (n == 0 || m == 0) return DEMON_OK;
  DEMON_REQUIRE(tsdf && weight && blocks && depth && K && R && t, "sparse_tsdf_integrate: null pointer");
  const long nvox = 512L * m;
  const unsigned grid = (unsigned)((nvox + kFuseThreads - 1) / kFuseThreads);
  if (color)
    sparse_tsdf_integrate_kernel<true><<<grid, kFuseThreads, 0, (cudaStream_t)stream>>>(
        tsdf, weight, color, blocks, nvox, origin[0], origin[1], origin[2], voxel_size, trunc, depth, K, R, t, image, n, h, w);
  else
    sparse_tsdf_integrate_kernel<false><<<grid, kFuseThreads, 0, (cudaStream_t)stream>>>(
        tsdf, weight, nullptr, blocks, nvox, origin[0], origin[1], origin[2], voxel_size, trunc, depth, K, R, t, nullptr, n, h, w);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int64_t demon_sparse_tsdf_mesh_scratch_bytes(int m) {
  if (m < 1) return 0;
  return sparse_mc_tiles(m) * (int64_t)(sizeof(int64_t) + sizeof(int)) + 8LL * m * sizeof(int);
}

int demon_sparse_tsdf_mesh_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, const int64_t* keys, const int* values,
                                     int64_t capacity, void* scratch, int64_t* triangles, void* stream) {
  if (int rc = check_table("sparse_tsdf_mesh_count", keys, values, capacity)) return rc;
  DEMON_REQUIRE(m >= 1 && 512LL * m * 15 < (1LL << 40), "sparse_tsdf_mesh_count: bad block count %d", m);
  DEMON_REQUIRE(tsdf && weight && blocks && scratch && triangles, "sparse_tsdf_mesh_count: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = (int)sparse_mc_tiles(m);
  int64_t* tile_first = static_cast<int64_t*>(scratch);   // scratch: tile_first [tiles], tile_counts [tiles], nbr [m,8]
  int* tile_counts = reinterpret_cast<int*>(tile_first + tiles);
  int* nbr = tile_counts + tiles;
  sparse_neighbours_kernel<<<(unsigned)ceil_div64(8LL * m, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), values, capacity - 1, blocks, m, nbr);
  DEMON_LAUNCH_CHECK();
  mc_count_kernel<<<tiles, kMcThreads, 0, st>>>(SparseVolume{tsdf, weight, blocks, nbr, 512L * m}, tile_counts);
  DEMON_LAUNCH_CHECK();
  mc_offsets_kernel<<<1, kScanThreads, 0, st>>>(tile_counts, tiles, tile_first, triangles);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_mesh_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, const float* origin,
                               float voxel_size, const void* scratch, float* vertices, uint8_t* colors, int* faces, void* stream) {
  DEMON_REQUIRE(m >= 1 && 512LL * m * 15 < (1LL << 40), "sparse_tsdf_mesh: bad block count %d", m);
  DEMON_REQUIRE(origin && std::isfinite(voxel_size) && voxel_size > 0.0f, "sparse_tsdf_mesh: bad origin or voxel_size %g", voxel_size);
  DEMON_REQUIRE(!color == !colors, "sparse_tsdf_mesh: color and colors go together");
  DEMON_REQUIRE(tsdf && weight && blocks && scratch && vertices && faces, "sparse_tsdf_mesh: null pointer");
  const int tiles = (int)sparse_mc_tiles(m);
  const int64_t* tile_first = static_cast<const int64_t*>(scratch);
  const int* nbr = reinterpret_cast<const int*>(tile_first + tiles) + tiles;
  const SparseVolume vol{tsdf, weight, blocks, nbr, 512L * m};
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
