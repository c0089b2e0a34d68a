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
#include "tile_scan.cuh"
#include <climits>
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
constexpr int kSegWords = 48;   // the indexed mesh's segment of mask words: 8 * 8 * 8 voxels of 3 edges
constexpr int kSegBits = 32 * kSegWords;

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

// What a cube lookup at a grid coordinate (the ray caster's `at`) found.
enum CubeAt { kNoCube = 0, kStored = 1, kEmptyBlock = -1 };   // kEmptyBlock: corner 0's block is not allocated

// The cubes of the dense box: cube c has its lower corner at voxel (i, j, k), i fastest.
struct DenseVolume {
  const float* tsdf;
  const float* weight;
  int nx, ny, cx, cy, cz;   // voxels along x and y, cubes along x, y and z
  long ncubes;
  struct Cube {
    int g[3];   // grid coordinate of corner 0
    long s;     // the indexed mesh's segment: its first voxel
  };
  struct Cursor {};
  // the cube whose corner 0 is at grid coordinate c (integer-valued floats): stored when it lies inside the box
  __device__ int at(const float c[3], Cube& cb, Cursor&) const {
    if (!(c[0] >= 0.0f && c[0] < (float)cx && c[1] >= 0.0f && c[1] < (float)cy && c[2] >= 0.0f && c[2] < (float)cz)) return kNoCube;
#pragma unroll
    for (int a = 0; a < 3; ++a) cb.g[a] = (int)c[a];
    return kStored;
  }
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
  // indexed mesh: the bit of edge (corner q, axis a), 3 (linear index) + a
  __device__ long edge_bit(const Cube& cb, int q, int a) const { return 3 * corner(cb, q) + a; }
  // mask word t: its segment (512 voxels from cb.s) and the segment-local bit of its bit 0
  __device__ int word(long t, long& w, Cube& cb) const {
    w = t;
    const long s = t / kSegWords;
    cb.s = 512 * s;
    return 32 * (int)(t - s * kSegWords);
  }
  // g = the segment's voxel l
  __device__ void seg_voxel(int l, Cube& cb) const {
    const long v = cb.s + l, plane = (long)nx * ny;
    cb.g[2] = (int)(v / plane);
    const long r = v - (long)cb.g[2] * plane;
    cb.g[1] = (int)(r / nx);
    cb.g[0] = (int)(r - (long)cb.g[1] * nx);
  }
  // the state index of voxel g + d, or -1 outside the box
  __device__ long voxel(const Cube& cb, int dx, int dy, int dz) const {
    const int x = cb.g[0] + dx, y = cb.g[1] + dy, z = cb.g[2] + dz;
    if (x < 0 || x >= nx || y < 0 || y >= ny || z < 0 || z > cz) return -1;
    return ((long)z * ny + y) * nx + x;
  }
};

__device__ __forceinline__ unsigned long long block_key(int bx, int by, int bz);
__device__ __forceinline__ long find_slot(const unsigned long long* __restrict__ keys, long mask, unsigned long long key);

// The cubes of the hashed blocks first, first + 1, ...: cube c has its lower corner at local voxel c % 512 (x fastest) of
// block first + c / 512, and its corners past the block's last voxel lie in the +x, +y, +z neighbours
// nbr[8 (b - first) + (dx | dy << 1 | dz << 2)], which may be any block of the pool.
struct SparseVolume {
  const float* tsdf;
  const float* weight;
  const int* blocks;   // [m,3] block coordinates
  const int* nbr;      // [count,8] pool index of block b + (dx, dy, dz), or -1
  long ncubes;
  const unsigned long long* keys;   // the hash table, for `at` only
  const int* values;
  long mask;
  int first;           // the first block of the cubes `locate` enumerates
  const int* rank = nullptr;   // indexed mesh: the key rank of every pool block, its segment
  struct Cube {
    int b;      // pool index
    int l[3];   // local voxel of corner 0
    int g[3];   // grid coordinate of corner 0: 8 * block + l
  };
  // the block of the last `at` and its pool index (-1: not allocated), so the table is probed once per block a ray enters
  struct Cursor {
    int B[3] = {INT_MIN, INT_MIN, INT_MIN};
    int b = -1;
  };
  // the cube whose corner 0 is at grid coordinate c (integer-valued floats): stored when its block is allocated (its
  // corners in the neighbours are resolved by `corner`), kEmptyBlock with cur.B its block when that block is not
  __device__ int at(const float c[3], Cube& cb, Cursor& cur) const {
    constexpr float lo = -8.0f * DEMON_SPARSE_TSDF_MAX_COORD, hi = 8.0f * DEMON_SPARSE_TSDF_MAX_COORD + 7.0f;
    if (!(c[0] >= lo && c[0] <= hi && c[1] >= lo && c[1] <= hi && c[2] >= lo && c[2] <= hi)) return kNoCube;
    int B[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      cb.g[a] = (int)c[a];
      B[a] = cb.g[a] >> 3;   // floor(g / 8)
      cb.l[a] = cb.g[a] & 7;
    }
    if (B[0] != cur.B[0] || B[1] != cur.B[1] || B[2] != cur.B[2]) {
      const long s = find_slot(keys, mask, block_key(B[0], B[1], B[2]));
      cur.b = s < 0 ? -1 : __ldg(values + s);   // negative (new, or on the host): not stored
#pragma unroll
      for (int a = 0; a < 3; ++a) cur.B[a] = B[a];
    }
    cb.b = cur.b;
    return cur.b < 0 ? kEmptyBlock : kStored;
  }
  __device__ bool locate(long c, Cube& cb) const {
    if (c >= ncubes) return false;
    cb.b = first + (int)(c >> 9);
    seg_voxel((int)(c & 511), cb);
    return true;
  }
  // the state index of corner q, or -1 when its block is not allocated
  __device__ long corner(const Cube& cb, int q) const {
    const int x = cb.l[0] + kCorner[q][0], y = cb.l[1] + kCorner[q][1], z = cb.l[2] + kCorner[q][2];
    const int nb = (x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2);
    const int blk = nb ? __ldg(nbr + 8L * (cb.b - first) + nb) : cb.b;
    if (blk < 0) return -1;
    return ((long)blk << 9) + ((z & 7) << 6) + ((y & 7) << 3) + (x & 7);
  }
  // indexed mesh: the bit of edge (corner q, axis a) of a valid cube, in the segment of the block that holds the corner
  __device__ long edge_bit(const Cube& cb, int q, int a) const {
    const long o = corner(cb, q);
    return (long)__ldg(rank + (o >> 9)) * kSegBits + 3 * (o & 511) + a;
  }
  // mask word t of blocks first, first + 1, ...: the word of block b's segment, and the segment-local bit of its bit 0
  __device__ int word(long t, long& w, Cube& cb) const {
    const int k = (int)(t / kSegWords), i = (int)(t - (long)k * kSegWords);
    cb.b = first + k;
    w = (long)__ldg(rank + cb.b) * kSegWords + i;
    return 32 * i;
  }
  // corner 0 of cube (or voxel) l of block cb.b
  __device__ void seg_voxel(int l, Cube& cb) const {
    cb.l[0] = l & 7;
    cb.l[1] = (l >> 3) & 7;
    cb.l[2] = l >> 6;
#pragma unroll
    for (int a = 0; a < 3; ++a) cb.g[a] = 8 * __ldg(blocks + 3 * cb.b + a) + cb.l[a];
  }
  // the state index of voxel g + d (|d_i| <= 1, or d = e_a + e_i), or -1 when its block is not stored: the block itself,
  // its + neighbours through nbr, the others through the table
  __device__ long voxel(const Cube& cb, int dx, int dy, int dz) const {
    const int x = cb.l[0] + dx, y = cb.l[1] + dy, z = cb.l[2] + dz;
    const int sx = x >> 3, sy = y >> 3, sz = z >> 3;   // -1, 0 or 1
    int blk = cb.b;
    if (sx | sy | sz) {
      if (sx >= 0 && sy >= 0 && sz >= 0) {
        blk = __ldg(nbr + 8L * (cb.b - first) + (sx | (sy << 1) | (sz << 2)));
      } else {
        const int bx = (cb.g[0] >> 3) + sx, by = (cb.g[1] >> 3) + sy, bz = (cb.g[2] >> 3) + sz;
        constexpr int lim = DEMON_SPARSE_TSDF_MAX_COORD;
        if (bx < -lim || by < -lim || bz < -lim || bx > lim || by > lim || bz > lim) return -1;
        const long s = find_slot(keys, mask, block_key(bx, by, bz));
        blk = s < 0 ? -1 : __ldg(values + s);
      }
      if (blk < 0) return -1;
    }
    return ((long)blk << 9) + ((z & 7) << 6) + ((y & 7) << 3) + (x & 7);
  }
};

// SparseVolume whose `locate` enumerates the blocks order[0], order[1], ... (a permutation of first .. first+count-1):
// the indexed mesh's faces in key order.  A type of its own, so the soup's kernels do not carry the lookup.
struct KeyOrderVolume : SparseVolume {
  const int* order;
  __device__ bool locate(long c, Cube& cb) const {
    if (c >= ncubes) return false;
    cb.b = __ldg(order + (c >> 9));
    seg_voxel((int)(c & 511), cb);
    return true;
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

// The soup's output: corner e3 of triangle tri gets its own vertex 3 tri + e3, interpolated on the edge.
template <bool kColor>
struct SoupOut {
  const float* color;
  float org[3];
  float vs;
  float* vertices;
  uint8_t* colors_out;
  int* faces;
  template <class V>
  __device__ __forceinline__ void operator()(const V& vol, const typename V::Cube& cb, int edge, long tri, int e3) const {
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
};

template <class V, class Out>
__global__ void __launch_bounds__(kMcThreads) mc_scatter_kernel(V vol, Out out, const int64_t* __restrict__ tile_first) {
  __shared__ int s_warp[kMcWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long base = (long)blockIdx.x * kMcTile + threadIdx.x;
  long row = tile_first[blockIdx.x];   // first triangle of round r in this tile
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
      for (int m = 0; m < cnt; ++m, ++tri)
        for (int e3 = 0; e3 < 3; ++e3) out(vol, cb, kTriTable[ci][3 * m + e3], tri, e3);
    }
    row += total;
  }
}

template <bool kColor, class V>
void launch_soup(const V& vol, int tiles, const float* color, const float* origin, float vs, const int64_t* tile_first, float* vertices,
                 uint8_t* colors, int* faces, cudaStream_t st) {
  const SoupOut<kColor> out{color, {origin[0], origin[1], origin[2]}, vs, vertices, colors, faces};
  mc_scatter_kernel<<<tiles, kMcThreads, 0, st>>>(vol, out, tile_first);
}

// ---- indexed mesh: one vertex per surface edge -------------------------------------------------------------------------
// Edge (g, a) runs from voxel g to g + e_a.  Every edge has a bit: in a dense box bit 3 (linear index of g) + a; in a
// sparse volume bit 1536 rank + 3 (local linear index of g) + a, rank the key rank of the block that holds g.  So both
// storages are runs of 48-word segments (512 voxels of 3 edges), and the vertices are the set bits in ascending order.
//   1. edge_mark_kernel: every valid cube ORs the bits of its sign-changing edges (the edges its triangles use).  The
//      owner of a cube's edge is the cube's block or one of its +x, +y, +z neighbours; OR is order-free, so the masks
//      depend on the volume alone.
//   2. edge_count_kernel, tile_offsets_kernel, edge_base_kernel: each segment's popcount, their exclusive scan (the
//      segment's first vertex), and each word's first vertex (the segment's plus the popcounts of the words before it).
//   3. edge_vertex_kernel: one thread per word writes the vertex of each of its set bits at base[word] + popcount of the
//      bits below it.  mc_scatter_kernel with IndexOut writes each triangle corner's edge index the same way.
constexpr int kEdgeThreads = 256;
__constant__ int8_t kEdgeAxis[12] = {0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2};

template <class V>
__global__ void __launch_bounds__(kMcThreads) edge_mark_kernel(V vol, unsigned* __restrict__ masks) {
  typename V::Cube cb;
  const int ci = cube_case(vol, (long)blockIdx.x * kMcThreads + threadIdx.x, cb);
  if (ci <= 0 || ci == 255) return;
#pragma unroll 1
  for (int e = 0; e < 12; ++e) {
    const int qa = kEdge[e][0], qb = kEdge[e][1];
    if (((ci >> qa) ^ (ci >> qb)) & 1) {
      const long bit = vol.edge_bit(cb, qa, kEdgeAxis[e]);
      atomicOr(masks + (bit >> 5), 1u << (bit & 31));
    }
  }
}

// One warp per segment: the number of its set bits.
__global__ void __launch_bounds__(kEdgeThreads) edge_count_kernel(const unsigned* __restrict__ masks, int segs, int* __restrict__ counts) {
  const long s = ((long)blockIdx.x * kEdgeThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= segs) return;
  const unsigned* m = masks + s * kSegWords;
  int c = __popc(m[lane]) + (lane < kSegWords - 32 ? __popc(m[32 + lane]) : 0);
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) counts[s] = c;
}

// One warp per segment: base[w] = the first vertex of word w (int32: the caller refuses 2^31 vertices or more).
__global__ void __launch_bounds__(kEdgeThreads) edge_base_kernel(const unsigned* __restrict__ masks, int segs,
                                                                 const int64_t* __restrict__ seg_first, int* __restrict__ base) {
  const long s = ((long)blockIdx.x * kEdgeThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= segs) return;
  const unsigned* m = masks + s * kSegWords;
  const int p0 = __popc(m[lane]), p1 = lane < kSegWords - 32 ? __popc(m[32 + lane]) : 0;
  int i0 = p0, i1 = p1;   // inclusive scans over the lanes
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y0 = __shfl_up_sync(0xffffffffu, i0, o), y1 = __shfl_up_sync(0xffffffffu, i1, o);
    if (lane >= o) {
      i0 += y0;
      i1 += y1;
    }
  }
  const int all0 = __shfl_sync(0xffffffffu, i0, 31);
  const long first = seg_first[s];
  base[s * kSegWords + lane] = (int)(first + i0 - p0);
  if (lane < kSegWords - 32) base[s * kSegWords + 32 + lane] = (int)(first + all0 + i1 - p1);
}

// The index of the vertex of edge bit `bit`.
__device__ __forceinline__ int edge_index(const unsigned* __restrict__ masks, const int* __restrict__ base, long bit) {
  const long w = bit >> 5;
  return __ldg(base + w) + __popc(__ldg(masks + w) & ((1u << (bit & 31)) - 1u));
}

// The indexed mesh's faces: corner e3 of triangle tri is the index of its edge's vertex.
struct IndexOut {
  const unsigned* masks;
  const int* base;
  int* faces;
  template <class V>
  __device__ __forceinline__ void operator()(const V& vol, const typename V::Cube& cb, int edge, long tri, int e3) const {
    faces[3 * tri + e3] = edge_index(masks, base, vol.edge_bit(cb, kEdge[edge][0], kEdgeAxis[edge]));
  }
};

// The vertex of edge (g, a) and its colour and normal, with demon_tsdf_indexed_mesh_f32's float order.  cb holds g
// (`voxel` resolves g + d for |d_i| <= 1 and d = e_a + e_i); the edge's two voxels are stored with weight > 0.
template <bool kColor, bool kNormals, class V>
__device__ __forceinline__ void edge_vertex(const V& vol, const typename V::Cube& cb, int a, const float* __restrict__ color,
                                            const float org[3], float vs, long v, float* __restrict__ vertices,
                                            float* __restrict__ normals, uint8_t* __restrict__ colors_out) {
  const int ea[3] = {a == 0, a == 1, a == 2};
  const long oa = vol.voxel(cb, 0, 0, 0), ob = vol.voxel(cb, ea[0], ea[1], ea[2]);
  const float fa = __ldg(vol.tsdf + oa), fb = __ldg(vol.tsdf + ob);
  const float mu = fdiv(fa, fsub(fa, fb));
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float pa = fadd(org[i], fmul(vs, (float)cb.g[i])), pb = fadd(org[i], fmul(vs, (float)(cb.g[i] + ea[i])));
    vertices[3 * v + i] = fadd(pa, fmul(mu, fsub(pb, pa)));
  }
  if (kColor) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const float ca = __ldg(color + 3 * oa + i), cc = __ldg(color + 3 * ob + i);
      const int q = __float2int_rn(fadd(ca, fmul(mu, fsub(cc, ca))));
      colors_out[3 * v + i] = (uint8_t)min(255, max(0, q));
    }
  }
  if (kNormals) {
    float n[3];
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      float d[2];
#pragma unroll
      for (int p = 0; p < 2; ++p) {   // central difference along i at g, then at g + e_a
        int hi[3] = {p * ea[0], p * ea[1], p * ea[2]}, lo[3] = {p * ea[0], p * ea[1], p * ea[2]};
        ++hi[i];
        --lo[i];
        const long oh = vol.voxel(cb, hi[0], hi[1], hi[2]), ol = vol.voxel(cb, lo[0], lo[1], lo[2]);
        ok = ok && oh >= 0 && ol >= 0 && __ldg(vol.weight + oh) > 0.0f && __ldg(vol.weight + ol) > 0.0f;
        d[p] = ok ? fsub(__ldg(vol.tsdf + oh), __ldg(vol.tsdf + ol)) : 0.0f;
      }
      n[i] = fadd(d[0], fmul(mu, fsub(d[1], d[0])));
    }
    const float len = __fsqrt_rn(fadd(fadd(fmul(n[0], n[0]), fmul(n[1], n[1])), fmul(n[2], n[2])));
    ok = ok && len > 0.0f;
#pragma unroll
    for (int i = 0; i < 3; ++i) normals[3 * v + i] = ok ? fdiv(n[i], len) : __int_as_float(0x7fffffff);
  }
}

// One thread per mask word of the voxels `vol.word_voxel` enumerates: the vertex of each set bit.
template <bool kColor, bool kNormals, class V>
__global__ void __launch_bounds__(kEdgeThreads) edge_vertex_kernel(V vol, long words, const unsigned* __restrict__ masks,
                                                                   const int* __restrict__ base, const float* __restrict__ color, float ox,
                                                                   float oy, float oz, float vs, float* __restrict__ vertices,
                                                                   float* __restrict__ normals, uint8_t* __restrict__ colors_out) {
  const long t = (long)blockIdx.x * kEdgeThreads + threadIdx.x;
  if (t >= words) return;
  long w;
  typename V::Cube cb;
  int lb0 = vol.word(t, w, cb);   // the word's global index, and the segment-local bit of its bit 0
  unsigned bitsw = __ldg(masks + w);
  if (!bitsw) return;
  int v = __ldg(base + w);
  const float org[3] = {ox, oy, oz};
  while (bitsw) {
    const int j = __ffs(bitsw) - 1;
    bitsw &= bitsw - 1;
    const int lb = lb0 + j, l = lb / 3, a = lb - 3 * l;
    vol.seg_voxel(l, cb);
    edge_vertex<kColor, kNormals>(vol, cb, a, color, org, vs, v++, vertices, normals, colors_out);
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
  return DenseVolume{tsdf, weight, nx, ny, nx - 1, ny - 1, nz - 1, (long)(nx - 1) * (ny - 1) * (nz - 1)};
}

// ---- sparse volume: voxel blocks in a hash table -------------------------------------------------------------------------
// Block (bx, by, bz), |b| <= kMaxBlockCoord per axis, holds voxels 8 b + (0..7) in the pool at its index: tsdf and weight
// [m,8,8,8] (z, y, x; x fastest), colour [m,8,8,8,3].  The table maps the packed key of a block to its pool index, by open
// addressing with linear probing over `capacity` (a power of 2) slots: key -1 marks an empty slot.  A value >= 0 is the
// block's pool index, -1 a block inserted by the running call's allocation and not yet given a pool index, and -2 - s a
// block streamed out to host slot s (SparseTsdfVolume's max_device_blocks): every reader below takes a negative value
// as "not stored on the device".
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

// Inserts key unless present; false when the table would hold more than `limit` keys.  `occupied` counts each key once,
// after the CAS that inserted it: counting every thread that meets an empty slot (many race on each new key) would raise
// overflows the keys do not cause.  Slots only go from empty to full, so an empty slot on the probe means the key is
// absent, and with `limit` keys counted already a new one overflows.  So a launch overflows exactly when the table's keys
// and the new ones are more than `limit` = capacity/2, and the table's size follows from the key count alone.  An
// overflowing launch may insert past `limit` before every thread sees the count, so the probe is bounded by the table's
// size and, every 32 slots, ends once more than `limit` keys are counted (the launch has overflowed then, whatever the
// key); the host rehashes into a doubled table before anything else reads it.  In a launch that does not overflow the
// count never passes `limit`, so that check ends no probe.
__device__ __forceinline__ bool insert_key(unsigned long long* keys, long mask, unsigned long long key, unsigned long long* occupied,
                                           unsigned long long limit) {
  long s = key_slot(key, mask);
  for (long probes = 0; probes <= mask; ++probes, s = (s + 1) & mask) {
    if ((probes & 31) == 31 && *(volatile unsigned long long*)occupied > limit) return false;
    unsigned long long k = *(volatile unsigned long long*)(keys + s);
    if (k == kEmptyKey) {
      if (*(volatile unsigned long long*)occupied >= limit) return false;
      k = atomicCAS(keys + s, kEmptyKey, key);
      if (k == kEmptyKey) return atomicAdd(occupied, 1ull) < limit;
    }
    if (k == key) return true;
  }
  return false;
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
  if (key != kEmptyKey && values[s] == -1) out[atomicAdd(counters + kCursor, 1ull)] = (int64_t)key;
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

// nbr[8 (b - first) + q] = the pool index of block b + (q & 1, q >> 1 & 1, q >> 2), or -1, for blocks first .. first+count-1.
__global__ void __launch_bounds__(kSparseThreads) sparse_neighbours_kernel(const unsigned long long* __restrict__ keys,
                                                                           const int* __restrict__ values, long mask,
                                                                           const int* __restrict__ blocks, int first, int count,
                                                                           int* __restrict__ nbr) {
  const long e = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (e >= 8L * count) return;
  const long b = first + (e >> 3);
  const int q = (int)(e & 7);
  const int bx = blocks[3 * b] + (q & 1), by = blocks[3 * b + 1] + ((q >> 1) & 1), bz = blocks[3 * b + 2] + (q >> 2);
  long s = -1;
  if (bx <= kMaxBlockCoord && by <= kMaxBlockCoord && bz <= kMaxBlockCoord) s = find_slot(keys, mask, block_key(bx, by, bz));
  const int v = s < 0 ? -1 : __ldg(values + s);
  nbr[e] = v < 0 ? -1 : v;   // a block on the host is not stored
}

// ---- ray casting ------------------------------------------------------------------------------------------------------
// One thread per pixel of every frame marches its ray through the volume with trilinear lookups (the rule is in
// include/demon_b200.h, demon_tsdf_raycast_f32).  The cube lookups are the volume's `at` and `corner`, so both storages run
// the same march; the sparse volume probes its hash table only when the ray enters another block, and jumps over the
// samples of a block that is not allocated (raycast_skip).
constexpr int kRayThreads = 128;
constexpr int kMaxSamples = 1 << 24;   // every sample index is exact in float

__device__ __forceinline__ float lerp_rn(float a, float b, float w) { return fadd(a, fmul(w, fsub(b, a))); }

// The trilinear value of field v (element ch of `stride`) over the corners o of a cube at weights w: x first, then y, then z.
__device__ __forceinline__ float trilinear(const float* __restrict__ v, const long o[8], const float w[3], int stride, int ch) {
  auto f = [&](int q) { return __ldg(v + stride * o[q] + ch); };
  const float y0 = lerp_rn(f(0), f(1), w[0]), y1 = lerp_rn(f(3), f(2), w[0]);
  const float y2 = lerp_rn(f(4), f(5), w[0]), y3 = lerp_rn(f(7), f(6), w[0]);
  return lerp_rn(lerp_rn(y0, y1, w[1]), lerp_rn(y2, y3, w[1]), w[2]);
}

// The grid coordinate of world point X: g = (X - origin) / voxel_size.
struct Grid {
  float o[3];
  float vs;
  __device__ __forceinline__ void coord(const float X[3], float g[3]) const {
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a] = fdiv(fsub(X[a], o[a]), vs);
  }
};

// The cube of world point X: its corners' state indices o and weights w when all 8 are stored with weight > 0
// (kStored); otherwise what `at` found, with kNoCube for a corner of weight 0 or in a missing neighbour.
template <class V>
__device__ __forceinline__ int cube_at(const V& vol, typename V::Cursor& cur, const Grid& gr, const float X[3], long o[8], float w[3]) {
  float g[3], c[3];
  gr.coord(X, g);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    c[a] = floorf(g[a]);
    w[a] = fsub(g[a], c[a]);
  }
  typename V::Cube cb;
  const int r = vol.at(c, cb, cur);
  if (r != kStored) return r;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    o[q] = vol.corner(cb, q);
    if (o[q] < 0 || !(__ldg(vol.weight + o[q]) > 0.0f)) return kNoCube;
  }
  return kStored;
}

template <class V>
__device__ __forceinline__ bool field_at(const V& vol, typename V::Cursor& cur, const Grid& gr, const float X[3], float& f) {
  long o[8];
  float w[3];
  if (cube_at(vol, cur, gr, X, o, w) != kStored) return false;
  f = trilinear(vol.tsdf, o, w, 1, 0);
  return true;
}

// The march's sample k: z_k = near + k delta, X = C + z_k D.
struct Ray {
  float C[3], D[3], near, delta;
  __device__ __forceinline__ float z(int k) const { return fadd(near, fmul((float)k, delta)); }
  __device__ __forceinline__ void point(float z, float X[3]) const {
#pragma unroll
    for (int a = 0; a < 3; ++a) X[a] = fadd(C[a], fmul(z, D[a]));
  }
};

// Sample k's corner 0 lies in block cur.B, which is not allocated: the last sample to evaluate before the ray leaves it.
// Every grid coordinate of a sample is monotonic in k (each step is a rounded monotonic operation), so the samples in
// cur.B are consecutive; a float estimate of the block's exit is checked against the rule's own arithmetic, and k itself
// is returned when the estimate's sample is not in cur.B.
__device__ __forceinline__ int raycast_skip(const SparseVolume::Cursor& cur, const Ray& ray, const Grid& gr, int k) {
  float zexit = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (ray.D[a] == 0.0f) continue;
    const int face = 8 * (cur.B[a] + (ray.D[a] > 0.0f ? 1 : 0));
    zexit = fminf(zexit, (gr.o[a] + gr.vs * (float)face - ray.C[a]) / ray.D[a]);
  }
  const float ke = floorf((zexit - ray.near) / ray.delta) - 1.0f;   // a sample or so short of the exit
  if (!(ke > (float)(k + 1) && ke < (float)kMaxSamples)) return k;
  const int kc = (int)ke;
  float X[3], g[3];
  ray.point(ray.z(kc), X);
  gr.coord(X, g);
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (!(floorf(g[a]) >= 8.0f * (float)cur.B[a] && floorf(g[a]) < 8.0f * (float)cur.B[a] + 8.0f)) return k;
  return kc;
}
__device__ __forceinline__ int raycast_skip(const DenseVolume::Cursor&, const Ray&, const Grid&, int k) { return k; }

template <class V, bool kColor>
__global__ void __launch_bounds__(kRayThreads) raycast_kernel(V vol, const float* __restrict__ color, Grid gr, const float* __restrict__ K,
                                                              const float* __restrict__ R, const float* __restrict__ t,
                                                              const float* __restrict__ near, const float* __restrict__ far, float step,
                                                              long nrays, int h, int w, float* __restrict__ depth,
                                                              float* __restrict__ normals, uint8_t* __restrict__ colors) {
  const long p = (long)blockIdx.x * kRayThreads + threadIdx.x;
  if (p >= nrays) return;
  const long hw = (long)h * w;
  const int f = (int)(p / hw);
  const int pix = (int)(p - (long)f * hw), py = pix / w, px = pix - py * w;
  const float* Rf = R + 9 * f;
  const float a = fdiv(fsub(fadd((float)px, 0.5f), __ldg(K + 9 * f + 2)), __ldg(K + 9 * f));
  const float b = fdiv(fsub(fadd((float)py, 0.5f), __ldg(K + 9 * f + 5)), __ldg(K + 9 * f + 4));
  Ray ray;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    ray.D[i] = fadd(fadd(fmul(__ldg(Rf + i), a), fmul(__ldg(Rf + 3 + i), b)), __ldg(Rf + 6 + i));
    ray.C[i] = -fadd(fadd(fmul(__ldg(Rf + i), __ldg(t + 3 * f)), fmul(__ldg(Rf + 3 + i), __ldg(t + 3 * f + 1))),
                     fmul(__ldg(Rf + 6 + i), __ldg(t + 3 * f + 2)));
  }
  ray.near = __ldg(near + f);
  ray.delta = fdiv(fmul(step, gr.vs), __fsqrt_rn(fadd(fadd(fmul(a, a), fmul(b, b)), 1.0f)));
  const float zfar = __ldg(far + f);
  typename V::Cursor cur;
  float zhit = NAN, fprev = 0.0f, zprev = 0.0f;
  bool vprev = false;
  for (int k = 0; ray.near >= 0.0f && k < kMaxSamples; ++k) {
    const float z = ray.z(k);
    if (!(z <= zfar)) break;
    bool valid = false;
    float fk = 0.0f;
    if (z > 0.0f) {
      float X[3], o_w[3];
      long o[8];
      ray.point(z, X);
      const int r = cube_at(vol, cur, gr, X, o, o_w);
      if (r == kStored) {
        valid = true;
        fk = trilinear(vol.tsdf, o, o_w, 1, 0);
      } else if (r == kEmptyBlock) {
        k = raycast_skip(cur, ray, gr, k);   // samples up to the new k are in the same empty block
      }
    }
    if (valid && vprev && fprev >= 0.0f && fk < 0.0f) {
      zhit = fadd(zprev, fmul(ray.delta, fdiv(fprev, fsub(fprev, fk))));
      break;
    }
    vprev = valid;
    fprev = fk;
    zprev = z;
  }
  depth[p] = zhit;
  const bool hit = zhit == zhit;
  float Xs[3];
  ray.point(zhit, Xs);
  if (normals) {
    float n[3] = {NAN, NAN, NAN};
    if (hit) {
      float grad[3];
      bool ok = true;
#pragma unroll
      for (int ax = 0; ax < 3 && ok; ++ax) {
        float Xp[3] = {Xs[0], Xs[1], Xs[2]}, Xm[3] = {Xs[0], Xs[1], Xs[2]}, fp, fm;
        Xp[ax] = fadd(Xs[ax], gr.vs);
        Xm[ax] = fsub(Xs[ax], gr.vs);
        ok = field_at(vol, cur, gr, Xp, fp) && field_at(vol, cur, gr, Xm, fm);
        grad[ax] = fsub(fp, fm);
      }
      if (ok) {
#pragma unroll
        for (int r = 0; r < 3; ++r)
          n[r] = fadd(fadd(fmul(__ldg(Rf + 3 * r), grad[0]), fmul(__ldg(Rf + 3 * r + 1), grad[1])), fmul(__ldg(Rf + 3 * r + 2), grad[2]));
        const float len = __fsqrt_rn(fadd(fadd(fmul(n[0], n[0]), fmul(n[1], n[1])), fmul(n[2], n[2])));
#pragma unroll
        for (int r = 0; r < 3; ++r) n[r] = fdiv(n[r], len);
      }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) normals[((long)f * 3 + r) * hw + pix] = n[r];
  }
  if (kColor) {
    int q[3] = {0, 0, 0};
    long o[8];
    float o_w[3];
    if (hit && cube_at(vol, cur, gr, Xs, o, o_w) == kStored) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) q[ch] = min(255, max(0, __float2int_rn(trilinear(color, o, o_w, 3, ch))));   // half to even
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) colors[3 * p + ch] = (uint8_t)q[ch];
  }
}

// far[f] = the largest camera z of the 8 corners 8 B + (0 or 8) of every block B: one thread per block, a warp maximum
// per frame, then an atomicMax on the order-preserving integer image of the float (far is zeroed first).
__device__ __forceinline__ unsigned ordered_bits(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(kSparseThreads) sparse_far_kernel(const int* __restrict__ blocks, int m, Grid gr, const float* __restrict__ R,
                                                                    const float* __restrict__ t, int n, unsigned* __restrict__ far_bits) {
  const int b = blockIdx.x * kSparseThreads + threadIdx.x;
  float X[2][3];
  if (b < m) {
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int e = 0; e < 2; ++e) X[e][a] = fadd(gr.o[a], fmul(gr.vs, (float)(8 * __ldg(blocks + 3 * b + a) + 8 * e)));
  }
  for (int f = 0; f < n; ++f) {
    float zmax = -INFINITY;
    if (b < m) {
      const float* Rf = R + 9 * f;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float z = fadd(fadd(fadd(fmul(__ldg(Rf + 6), X[q & 1][0]), fmul(__ldg(Rf + 7), X[(q >> 1) & 1][1])),
                                  fmul(__ldg(Rf + 8), X[q >> 2][2])),
                             __ldg(t + 3 * f + 2));
        zmax = fmaxf(zmax, z);
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) zmax = fmaxf(zmax, __shfl_xor_sync(0xffffffffu, zmax, o));
    if ((threadIdx.x & 31) == 0 && zmax > -INFINITY) atomicMax(far_bits + f, ordered_bits(zmax));
  }
}

__global__ void sparse_far_decode_kernel(float* far, int n) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const unsigned u = reinterpret_cast<const unsigned*>(far)[f];
  far[f] = __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}


// ---- streaming blocks between the device and host memory (SparseTsdfVolume's max_device_blocks) -----------------------
// The reach rule decides which blocks a call's cameras can touch; the evict and restore kernels move whole blocks between
// pool slots and host slots of mapped pinned memory (zero-copy: one warp per block, coalesced 16-byte accesses over the
// PCIe link) and rewrite the blocks' table values in the same pass.  The rule is in include/demon_b200.h
// (demon_sparse_tsdf_reach_f32) and its guarantee in DESIGN.md §3.9.
constexpr int kDepthTile = 8;
constexpr int kMoveThreads = 256;

// tiles[f, ty, tx] = the largest finite depth > 0 of the tile's pixels, -inf when there is none.
__global__ void __launch_bounds__(kSparseThreads) sparse_depth_tiles_kernel(const float* __restrict__ depth, int n, int h, int w, int th,
                                                                            int tw, float* __restrict__ tiles) {
  const long e = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (e >= (long)n * th * tw) return;
  const int f = (int)(e / ((long)th * tw));
  const int r = (int)(e - (long)f * th * tw), ty = r / tw, tx = r - ty * tw;
  const float* df = depth + (long)f * h * w;
  float mx = -INFINITY;
  for (int y = kDepthTile * ty; y < min(h, kDepthTile * ty + kDepthTile); ++y)
    for (int x = kDepthTile * tx; x < min(w, kDepthTile * tx + kDepthTile); ++x) {
      const float d = __ldg(df + (long)y * w + x);
      if (isfinite(d) && d > 0.0f) mx = fmaxf(mx, d);
    }
  tiles[e] = mx;
}

// One thread per block and frame: out[b] = mark when frame f reaches block b (the rule of demon_sparse_tsdf_reach_f32).
__global__ void __launch_bounds__(kSparseThreads) sparse_reach_kernel(const int* __restrict__ blocks, int m, Grid gr, float trunc,
                                                                      const float* __restrict__ tiles, const float* __restrict__ K,
                                                                      const float* __restrict__ R, const float* __restrict__ t, int n,
                                                                      int h, int w, int* __restrict__ out, int mark) {
  const long e = (long)blockIdx.x * kSparseThreads + threadIdx.x;
  if (e >= (long)m * n) return;
  const int f = (int)(e / m), b = (int)(e - (long)f * m);
  float lo[3], hi[3];
  const float tr2 = fadd(trunc, trunc);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int g = 8 * __ldg(blocks + 3 * b + a);
    lo[a] = fsub(fadd(gr.o[a], fmul(gr.vs, (float)(g - 3))), tr2);
    hi[a] = fadd(fadd(gr.o[a], fmul(gr.vs, (float)(g + 10))), tr2);
  }
  const float* Rf = R + 9 * f;
  const float* tf = t + 3 * f;
  const float fx = __ldg(K + 9 * f), cx = __ldg(K + 9 * f + 2), fy = __ldg(K + 9 * f + 4), cy = __ldg(K + 9 * f + 5);
  float zmin = INFINITY, zmax = -INFINITY, umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
  bool behind = false;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float X0 = (q & 1) ? hi[0] : lo[0], X1 = (q & 2) ? hi[1] : lo[1], X2 = (q & 4) ? hi[2] : lo[2];
    const float z = fadd(fadd(fadd(fmul(__ldg(Rf + 6), X0), fmul(__ldg(Rf + 7), X1)), fmul(__ldg(Rf + 8), X2)), __ldg(tf + 2));
    zmin = fminf(zmin, z);
    zmax = fmaxf(zmax, z);
    if (!(z > gr.vs)) {
      behind = true;
      continue;
    }
    const float x = fadd(fadd(fadd(fmul(__ldg(Rf), X0), fmul(__ldg(Rf + 1), X1)), fmul(__ldg(Rf + 2), X2)), __ldg(tf));
    const float y = fadd(fadd(fadd(fmul(__ldg(Rf + 3), X0), fmul(__ldg(Rf + 4), X1)), fmul(__ldg(Rf + 5), X2)), __ldg(tf + 1));
    const float u = fadd(fdiv(fmul(fx, x), z), cx), v = fadd(fdiv(fmul(fy, y), z), cy);
    umin = fminf(umin, u);
    umax = fmaxf(umax, u);
    vmin = fminf(vmin, v);
    vmax = fmaxf(vmax, v);
  }
  if (!(zmax > gr.vs)) return;   // wholly behind the camera
  int x0 = 0, x1 = w - 1, y0 = 0, y1 = h - 1;
  if (behind) {
    zmin = 0.0f;
  } else {
    const float u0 = floorf(umin) - 1.0f, u1 = floorf(umax) + 1.0f, v0 = floorf(vmin) - 1.0f, v1 = floorf(vmax) + 1.0f;
    if (!(u1 >= 0.0f && u0 <= (float)(w - 1) && v1 >= 0.0f && v0 <= (float)(h - 1))) return;
    x0 = (int)fmaxf(u0, 0.0f);
    x1 = (int)fminf(u1, (float)(w - 1));
    y0 = (int)fmaxf(v0, 0.0f);
    y1 = (int)fminf(v1, (float)(h - 1));
  }
  const int tw = (w + kDepthTile - 1) / kDepthTile, th = (h + kDepthTile - 1) / kDepthTile;
  const float* T = tiles + (long)f * th * tw;
  for (int ty = y0 / kDepthTile; ty <= y1 / kDepthTile; ++ty)
    for (int tx = x0 / kDepthTile; tx <= x1 / kDepthTile; ++tx)
      if (fadd(__ldg(T + ty * tw + tx), trunc) >= zmin) {
        out[b] = mark;
        return;
      }
}

// Warp i moves pool block src[i] to host slot slots[i] and gives its key the value -2 - slots[i].
__global__ void __launch_bounds__(kMoveThreads) sparse_evict_kernel(const float4* __restrict__ tsdf, const float4* __restrict__ weight,
                                                                    const float4* __restrict__ color, const int* __restrict__ blocks,
                                                                    const int* __restrict__ stamps, const unsigned long long* __restrict__ keys,
                                                                    int* __restrict__ values, long mask, const int* __restrict__ src,
                                                                    const int* __restrict__ slots, int count, float4* __restrict__ htsdf,
                                                                    float4* __restrict__ hweight, float4* __restrict__ hcolor,
                                                                    int* __restrict__ hblocks, int* __restrict__ hstamps) {
  const int i = (int)(((long)blockIdx.x * kMoveThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= count) return;
  const long s = __ldg(src + i), d = __ldg(slots + i);
  for (int j = lane; j < 128; j += 32) {
    htsdf[128 * d + j] = __ldg(tsdf + 128 * s + j);
    hweight[128 * d + j] = __ldg(weight + 128 * s + j);
  }
  if (color)
    for (int j = lane; j < 384; j += 32) hcolor[384 * d + j] = __ldg(color + 384 * s + j);
  if (lane < 3) hblocks[3 * d + lane] = __ldg(blocks + 3 * s + lane);
  if (lane == 0) {
    hstamps[d] = __ldg(stamps + s);
    const long sl = find_slot(keys, mask, block_key(__ldg(blocks + 3 * s), __ldg(blocks + 3 * s + 1), __ldg(blocks + 3 * s + 2)));
    if (sl >= 0) values[sl] = -2 - (int)d;
  }
}

// Warp i moves host slot slots[i] to pool block dst[i]: its coordinates, optionally its stamp, and its table value.
__global__ void __launch_bounds__(kMoveThreads) sparse_restore_kernel(const float4* __restrict__ htsdf, const float4* __restrict__ hweight,
                                                                      const float4* __restrict__ hcolor, const int* __restrict__ hblocks,
                                                                      const int* __restrict__ slots, const int* __restrict__ dst, int count,
                                                                      float4* __restrict__ tsdf, float4* __restrict__ weight,
                                                                      float4* __restrict__ color, int* __restrict__ blocks,
                                                                      int* __restrict__ stamps, int stamp,
                                                                      const unsigned long long* __restrict__ keys, int* __restrict__ values,
                                                                      long mask) {
  const int i = (int)(((long)blockIdx.x * kMoveThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= count) return;
  const long s = __ldg(slots + i), d = __ldg(dst + i);
  for (int j = lane; j < 128; j += 32) {
    tsdf[128 * d + j] = htsdf[128 * s + j];
    weight[128 * d + j] = hweight[128 * s + j];
  }
  if (color)
    for (int j = lane; j < 384; j += 32) color[384 * d + j] = hcolor[384 * s + j];
  if (lane < 3) blocks[3 * d + lane] = __ldg(hblocks + 3 * s + lane);
  if (lane == 0) {
    if (stamps) stamps[d] = stamp;
    if (keys) {
      const long sl = find_slot(keys, mask, block_key(__ldg(hblocks + 3 * s), __ldg(hblocks + 3 * s + 1), __ldg(hblocks + 3 * s + 2)));
      if (sl >= 0) values[sl] = (int)d;
    }
  }
}

// values[key of block b] = b for blocks first .. first+count-1, inserting the key when the table lacks it.
__global__ void __launch_bounds__(kSparseThreads) sparse_index_kernel(unsigned long long* __restrict__ keys, int* __restrict__ values,
                                                                      long mask, const int* __restrict__ blocks, int first, int count) {
  const int i = blockIdx.x * kSparseThreads + threadIdx.x;
  if (i >= count) return;
  const long b = (long)first + i;
  const unsigned long long key = block_key(blocks[3 * b], blocks[3 * b + 1], blocks[3 * b + 2]);
  for (long q = key_slot(key, mask);; q = (q + 1) & mask) {
    unsigned long long k = *(volatile unsigned long long*)(keys + q);
    if (k == kEmptyKey) k = atomicCAS(keys + q, kEmptyKey, key);
    if (k == kEmptyKey || k == key) {
      values[q] = (int)b;
      return;
    }
  }
}

// The device address of mapped pinned host memory, or an error for memory the device cannot reach.
int mapped(const char* name, const void* p, void** dev) {
  if (!p) {
    *dev = nullptr;
    return DEMON_OK;
  }
  cudaPointerAttributes at;
  DEMON_CHECK_CUDA(cudaPointerGetAttributes(&at, p));
  DEMON_REQUIRE(at.type == cudaMemoryTypeHost && at.devicePointer, "%s: the host store must be pinned host memory the device can map", name);
  *dev = at.devicePointer;
  return DEMON_OK;
}

int check_raycast(const char* name, const float* origin, float voxel_size, float step, int n, int h, int w) {
  DEMON_REQUIRE(n >= 0 && h >= 1 && w >= 1 && (long)h * w < (1L << 24), "%s: bad size %d frames of %dx%d", name, n, h, w);
  DEMON_REQUIRE(origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]), "%s: the origin must be finite",
                name);
  DEMON_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0f, "%s: voxel_size must be finite and > 0, got %g", name, voxel_size);
  DEMON_REQUIRE(std::isfinite(step) && step > 0.0f && step <= 1.0f, "%s: step must be in (0, 1], got %g", name, step);
  return DEMON_OK;
}

template <class V>
int launch_raycast(const V& vol, const float* color, const float* origin, float voxel_size, const float* K, const float* R, const float* t,
                   const float* near, const float* far, float step, int n, int h, int w, float* depth, float* normals, uint8_t* colors,
                   cudaStream_t st) {
  const long nrays = (long)n * h * w;
  const Grid gr{{origin[0], origin[1], origin[2]}, voxel_size};
  const unsigned grid = (unsigned)ceil_div64(nrays, kRayThreads);
  if (colors)
    raycast_kernel<V, true><<<grid, kRayThreads, 0, st>>>(vol, color, gr, K, R, t, near, far, step, nrays, h, w, depth, normals, colors);
  else
    raycast_kernel<V, false><<<grid, kRayThreads, 0, st>>>(vol, nullptr, gr, K, R, t, near, far, step, nrays, h, w, depth, normals, nullptr);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
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

int check_range(const char* name, int m, int first, int count) {
  DEMON_REQUIRE(m >= 1 && first >= 0 && count >= 1 && (int64_t)first + count <= m && 512LL * count * 15 < (1LL << 40),
                "%s: bad blocks %d..%d of %d", name, first, first + count - 1, m);
  return DEMON_OK;
}

// The neighbour table of blocks first .. first+count-1 into the sparse mesh scratch (tile_first [tiles], tile_counts
// [tiles], nbr [count,8]); returns nbr.
int* sparse_range_neighbours(const int* blocks, int first, int count, const int64_t* keys, const int* values, int64_t capacity, void* scratch,
                             cudaStream_t st) {
  const int tiles = (int)sparse_mc_tiles(count);
  int* nbr = reinterpret_cast<int*>(static_cast<int64_t*>(scratch) + tiles) + tiles;
  sparse_neighbours_kernel<<<(unsigned)ceil_div64(8LL * count, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), values, capacity - 1, blocks, first, count, nbr);
  return nbr;
}

// Marching cubes, step 1, on the cubes of blocks first .. first+count-1 enumerated in pool order or, with `order`, in
// the order order[0], order[1], ... (a permutation of first .. first+count-1).
int sparse_range_count(const char* name, const float* tsdf, const float* weight, const int* blocks, int m, int first, int count,
                       const int* order, const int64_t* keys, const int* values, int64_t capacity, void* scratch, int64_t* triangles,
                       cudaStream_t st) {
  if (int rc = check_table(name, keys, values, capacity)) return rc;
  if (int rc = check_range(name, m, first, count)) return rc;
  DEMON_REQUIRE(tsdf && weight && blocks && scratch && triangles, "%s: null pointer", name);
  const int tiles = (int)sparse_mc_tiles(count);
  int64_t* tile_first = static_cast<int64_t*>(scratch);
  int* tile_counts = reinterpret_cast<int*>(tile_first + tiles);
  const int* nbr = sparse_range_neighbours(blocks, first, count, keys, values, capacity, scratch, st);
  DEMON_LAUNCH_CHECK();
  const SparseVolume vol{tsdf, weight, blocks, nbr, 512L * count, nullptr, nullptr, 0, first};
  if (order)
    mc_count_kernel<<<tiles, kMcThreads, 0, st>>>(KeyOrderVolume{vol, order}, tile_counts);
  else
    mc_count_kernel<<<tiles, kMcThreads, 0, st>>>(vol, tile_counts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(tile_counts, tiles, tile_first, triangles);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// The indexed mesh, step 2: each segment's vertex count, their scan (the total into *vertices) and each word's first
// vertex.  scratch: seg_first int64 [segs], counts int [segs].
int edge_scan(const unsigned* masks, int segs, void* scratch, int* base, int64_t* vertices, cudaStream_t st) {
  int64_t* seg_first = static_cast<int64_t*>(scratch);
  int* counts = reinterpret_cast<int*>(seg_first + segs);
  const unsigned grid = (unsigned)ceil_div64(32LL * segs, kEdgeThreads);
  edge_count_kernel<<<grid, kEdgeThreads, 0, st>>>(masks, segs, counts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(counts, segs, seg_first, vertices);
  DEMON_LAUNCH_CHECK();
  edge_base_kernel<<<grid, kEdgeThreads, 0, st>>>(masks, segs, seg_first, base);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

template <class V>
int launch_edge_vertices(const V& vol, long words, const unsigned* masks, const int* base, const float* color, const float* origin, float vs,
                         float* vertices, float* normals, uint8_t* colors, cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(words, kEdgeThreads);
#define DEMON_EDGE_VERTICES(C, N)                                                                                               \
  edge_vertex_kernel<C, N><<<grid, kEdgeThreads, 0, st>>>(vol, words, masks, base, color, origin[0], origin[1], origin[2], vs, vertices, \
                                                          normals, colors)
  if (color && normals) DEMON_EDGE_VERTICES(true, true);
  else if (color) DEMON_EDGE_VERTICES(true, false);
  else if (normals) DEMON_EDGE_VERTICES(false, true);
  else DEMON_EDGE_VERTICES(false, false);
#undef DEMON_EDGE_VERTICES
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// The dense indexed mesh's segments (512 voxels each) and its scratch: tile_first int64 [tiles], seg_first int64 [segs],
// seg counts int [segs], tile_counts int [tiles], masks [segs,48], base [segs,48].
long dense_segs(int nx, int ny, int nz) { return ((long)nx * ny * nz + 511) / 512; }

struct DenseEdgeScratch {
  int64_t* tile_first;
  int* tile_counts;
  void* scan;   // seg_first, then the counts
  unsigned* masks;
  int* base;
  DenseEdgeScratch(void* scratch, int tiles, long segs) {
    tile_first = static_cast<int64_t*>(scratch);
    int64_t* seg_first = tile_first + tiles;
    scan = seg_first;
    // edge_scan's counts follow seg_first; tile_counts follow those
    tile_counts = reinterpret_cast<int*>(seg_first + segs) + segs;
    masks = reinterpret_cast<unsigned*>(tile_counts + tiles);
    base = reinterpret_cast<int*>(masks + segs * kSegWords);
  }
};

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
  tile_offsets_kernel<<<1, kScanThreads, 0, (cudaStream_t)stream>>>(tile_counts, tiles, tile_first, triangles);
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
    launch_soup<true>(vol, tiles, color, origin, voxel_size, tile_first, vertices, colors, faces, (cudaStream_t)stream);
  else
    launch_soup<false>(vol, tiles, nullptr, origin, voxel_size, tile_first, vertices, nullptr, faces, (cudaStream_t)stream);
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

int demon_sparse_tsdf_mesh_range_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count,
                                           const int64_t* keys, const int* values, int64_t capacity, void* scratch, int64_t* triangles,
                                           void* stream) {
  return sparse_range_count("sparse_tsdf_mesh_count", tsdf, weight, blocks, m, first, count, nullptr, keys, values, capacity, scratch,
                            triangles, (cudaStream_t)stream);
}

int demon_sparse_tsdf_mesh_range_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, int first,
                                     int count, const float* origin, float voxel_size, const void* scratch, float* vertices, uint8_t* colors,
                                     int* faces, void* stream) {
  DEMON_REQUIRE(m >= 1 && first >= 0 && count >= 1 && (int64_t)first + count <= m && 512LL * count * 15 < (1LL << 40),
                "sparse_tsdf_mesh: bad blocks %d..%d of %d", first, first + count - 1, m);
  DEMON_REQUIRE(origin && std::isfinite(voxel_size) && voxel_size > 0.0f, "sparse_tsdf_mesh: bad origin or voxel_size %g", voxel_size);
  DEMON_REQUIRE(!color == !colors, "sparse_tsdf_mesh: color and colors go together");
  DEMON_REQUIRE(tsdf && weight && blocks && scratch && vertices && faces, "sparse_tsdf_mesh: null pointer");
  const int tiles = (int)sparse_mc_tiles(count);
  const int64_t* tile_first = static_cast<const int64_t*>(scratch);
  const int* nbr = reinterpret_cast<const int*>(tile_first + tiles) + tiles;
  const SparseVolume vol{tsdf, weight, blocks, nbr, 512L * count, nullptr, nullptr, 0, first};
  if (color)
    launch_soup<true>(vol, tiles, color, origin, voxel_size, tile_first, vertices, colors, faces, (cudaStream_t)stream);
  else
    launch_soup<false>(vol, tiles, nullptr, origin, voxel_size, tile_first, vertices, nullptr, faces, (cudaStream_t)stream);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_mesh_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, const int64_t* keys, const int* values,
                                     int64_t capacity, void* scratch, int64_t* triangles, void* stream) {
  return demon_sparse_tsdf_mesh_range_count_f32(tsdf, weight, blocks, m, 0, m, keys, values, capacity, scratch, triangles, stream);
}

int demon_sparse_tsdf_mesh_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, const float* origin,
                               float voxel_size, const void* scratch, float* vertices, uint8_t* colors, int* faces, void* stream) {
  return demon_sparse_tsdf_mesh_range_f32(tsdf, weight, color, blocks, m, 0, m, origin, voxel_size, scratch, vertices, colors, faces, stream);
}

int demon_tsdf_raycast_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                           float voxel_size, const float* K, const float* R, const float* t, const float* near, const float* far, float step,
                           int n, int h, int w, float* depth, float* normals, uint8_t* colors, void* stream) {
  if (int rc = check_volume("tsdf_raycast", nx, ny, nz)) return rc;
  if (int rc = check_raycast("tsdf_raycast", origin, voxel_size, step, n, h, w)) return rc;
  DEMON_REQUIRE(color || !colors, "tsdf_raycast: colors need a colour volume");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(tsdf && weight && K && R && t && near && far && depth, "tsdf_raycast: null pointer");
  return launch_raycast(make_volume(tsdf, weight, nx, ny, nz), color, origin, voxel_size, K, R, t, near, far, step, n, h, w, depth, normals,
                        colors, (cudaStream_t)stream);
}

int64_t demon_sparse_tsdf_raycast_scratch_bytes(int m) { return m < 1 ? 0 : 8LL * m * sizeof(int); }

int demon_sparse_tsdf_far_f32(const int* blocks, int m, const float* origin, float voxel_size, const float* R, const float* t, int n, float* far,
                              void* stream) {
  DEMON_REQUIRE(m >= 1 && n >= 0, "sparse_tsdf_far: bad block count %d or frame count %d", m, n);
  DEMON_REQUIRE(origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]) && std::isfinite(voxel_size) &&
                    voxel_size > 0.0f,
                "sparse_tsdf_far: bad origin or voxel_size %g", voxel_size);
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(blocks && R && t && far, "sparse_tsdf_far: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  DEMON_CHECK_CUDA(cudaMemsetAsync(far, 0, n * sizeof(float), st));
  const Grid gr{{origin[0], origin[1], origin[2]}, voxel_size};
  sparse_far_kernel<<<ceil_div(m, kSparseThreads), kSparseThreads, 0, st>>>(blocks, m, gr, R, t, n, reinterpret_cast<unsigned*>(far));
  DEMON_LAUNCH_CHECK();
  sparse_far_decode_kernel<<<ceil_div(n, 256), 256, 0, st>>>(far, n);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_raycast_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, const int64_t* keys,
                                  const int* values, int64_t capacity, void* scratch, const float* origin, float voxel_size, const float* K,
                                  const float* R, const float* t, const float* near, const float* far, float step, int n, int h, int w,
                                  float* depth, float* normals, uint8_t* colors, void* stream) {
  if (int rc = check_table("sparse_tsdf_raycast", keys, values, capacity)) return rc;
  if (int rc = check_raycast("sparse_tsdf_raycast", origin, voxel_size, step, n, h, w)) return rc;
  DEMON_REQUIRE(m >= 1 && 512LL * m < (1LL << 40), "sparse_tsdf_raycast: bad block count %d", m);
  DEMON_REQUIRE(color || !colors, "sparse_tsdf_raycast: colors need a colour volume");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(tsdf && weight && blocks && scratch && K && R && t && near && far && depth, "sparse_tsdf_raycast: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int* nbr = static_cast<int*>(scratch);   // scratch: nbr [m,8]
  sparse_neighbours_kernel<<<(unsigned)ceil_div64(8LL * m, kSparseThreads), kSparseThreads, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), values, capacity - 1, blocks, 0, m, nbr);
  DEMON_LAUNCH_CHECK();
  const SparseVolume vol{tsdf, weight, blocks, nbr, 512L * m, reinterpret_cast<const unsigned long long*>(keys), values, (long)capacity - 1, 0};
  return launch_raycast(vol, color, origin, voxel_size, K, R, t, near, far, step, n, h, w, depth, normals, colors, st);
}

int demon_sparse_tsdf_depth_tiles_f32(const float* depth, int n, int h, int w, float* tiles, void* stream) {
  DEMON_REQUIRE(n >= 0 && h >= 1 && w >= 1 && (long)h * w < (1L << 24), "sparse_tsdf_depth_tiles: bad size %d frames of %dx%d", n, h, w);
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && tiles, "sparse_tsdf_depth_tiles: null pointer");
  const int th = ceil_div(h, kDepthTile), tw = ceil_div(w, kDepthTile);
  sparse_depth_tiles_kernel<<<(unsigned)ceil_div64((int64_t)n * th * tw, kSparseThreads), kSparseThreads, 0, (cudaStream_t)stream>>>(
      depth, n, h, w, th, tw, tiles);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_reach_f32(const int* blocks, int m, const float* origin, float voxel_size, float trunc, const float* tiles, const float* K,
                                const float* R, const float* t, int n, int h, int w, int* out, int mark, void* stream) {
  DEMON_REQUIRE(m >= 0 && n >= 0 && h >= 1 && w >= 1 && (long)h * w < (1L << 24), "sparse_tsdf_reach: bad size %d blocks, %d frames of %dx%d",
                m, n, h, w);
  DEMON_REQUIRE(origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]) && std::isfinite(voxel_size) &&
                    voxel_size > 0.0f && std::isfinite(trunc) && trunc >= 0.0f,
                "sparse_tsdf_reach: bad origin, voxel_size %g or trunc %g", voxel_size, trunc);
  if (m == 0 || n == 0) return DEMON_OK;
  DEMON_REQUIRE(blocks && tiles && K && R && t && out, "sparse_tsdf_reach: null pointer");
  const Grid gr{{origin[0], origin[1], origin[2]}, voxel_size};
  sparse_reach_kernel<<<(unsigned)ceil_div64((int64_t)m * n, kSparseThreads), kSparseThreads, 0, (cudaStream_t)stream>>>(
      blocks, m, gr, trunc, tiles, K, R, t, n, h, w, out, mark);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_evict(const float* tsdf, const float* weight, const float* color, const int* blocks, const int* stamps, const int64_t* keys,
                            int* values, int64_t capacity, const int* src, const int* slots, int count, float* host_tsdf, float* host_weight,
                            float* host_color, int* host_blocks, int* host_stamps, void* stream) {
  if (int rc = check_table("sparse_tsdf_evict", keys, values, capacity)) return rc;
  DEMON_REQUIRE(count >= 0, "sparse_tsdf_evict: bad count %d", count);
  DEMON_REQUIRE(!color == !host_color, "sparse_tsdf_evict: color and host_color go together");
  if (count == 0) return DEMON_OK;
  DEMON_REQUIRE(tsdf && weight && blocks && stamps && src && slots && host_tsdf && host_weight && host_blocks && host_stamps,
                "sparse_tsdf_evict: null pointer");
  void *ht, *hw, *hc;
  if (int rc = mapped("sparse_tsdf_evict", host_tsdf, &ht)) return rc;
  if (int rc = mapped("sparse_tsdf_evict", host_weight, &hw)) return rc;
  if (int rc = mapped("sparse_tsdf_evict", host_color, &hc)) return rc;
  sparse_evict_kernel<<<(unsigned)ceil_div64(32LL * count, kMoveThreads), kMoveThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(tsdf), reinterpret_cast<const float4*>(weight), reinterpret_cast<const float4*>(color), blocks, stamps,
      reinterpret_cast<const unsigned long long*>(keys), values, capacity - 1, src, slots, count, static_cast<float4*>(ht),
      static_cast<float4*>(hw), static_cast<float4*>(hc), host_blocks, host_stamps);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_restore(const float* host_tsdf, const float* host_weight, const float* host_color, const int* host_blocks, const int* slots,
                              const int* dst, int count, float* tsdf, float* weight, float* color, int* blocks, int* stamps, int stamp,
                              const int64_t* keys, int* values, int64_t capacity, void* stream) {
  if (keys) {
    if (int rc = check_table("sparse_tsdf_restore", keys, values, capacity)) return rc;
  }
  DEMON_REQUIRE(count >= 0, "sparse_tsdf_restore: bad count %d", count);
  DEMON_REQUIRE(!color == !host_color, "sparse_tsdf_restore: color and host_color go together");
  if (count == 0) return DEMON_OK;
  DEMON_REQUIRE(host_tsdf && host_weight && host_blocks && slots && dst && tsdf && weight && blocks, "sparse_tsdf_restore: null pointer");
  void *ht, *hw, *hc;
  if (int rc = mapped("sparse_tsdf_restore", host_tsdf, &ht)) return rc;
  if (int rc = mapped("sparse_tsdf_restore", host_weight, &hw)) return rc;
  if (int rc = mapped("sparse_tsdf_restore", host_color, &hc)) return rc;
  sparse_restore_kernel<<<(unsigned)ceil_div64(32LL * count, kMoveThreads), kMoveThreads, 0, (cudaStream_t)stream>>>(
      static_cast<const float4*>(ht), static_cast<const float4*>(hw), static_cast<const float4*>(hc), host_blocks, slots, dst, count,
      reinterpret_cast<float4*>(tsdf), reinterpret_cast<float4*>(weight), reinterpret_cast<float4*>(color), blocks, stamps, stamp,
      reinterpret_cast<const unsigned long long*>(keys), values, keys ? capacity - 1 : 0);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_index(int64_t* keys, int* values, int64_t capacity, const int* blocks, int first, int count, void* stream) {
  if (int rc = check_table("sparse_tsdf_index", keys, values, capacity)) return rc;
  DEMON_REQUIRE(first >= 0 && count >= 0 && (int64_t)first + count < (1LL << 31) && count < capacity, "sparse_tsdf_index: bad blocks %d + %d",
                first, count);
  if (count == 0) return DEMON_OK;
  DEMON_REQUIRE(blocks, "sparse_tsdf_index: null pointer");
  sparse_index_kernel<<<ceil_div(count, kSparseThreads), kSparseThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<unsigned long long*>(keys), values, capacity - 1, blocks, first, count);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int64_t demon_tsdf_indexed_mesh_scratch_bytes(int nx, int ny, int nz) {
  if (check_volume("tsdf_indexed_mesh_scratch_bytes", nx, ny, nz)) return 0;
  const long segs = dense_segs(nx, ny, nz);
  return mc_tiles(nx, ny, nz) * (int64_t)(sizeof(int64_t) + sizeof(int)) + segs * (int64_t)(sizeof(int64_t) + sizeof(int)) +
         segs * kSegWords * (int64_t)(sizeof(unsigned) + sizeof(int));
}

int demon_tsdf_indexed_mesh_count_f32(const float* tsdf, const float* weight, int nx, int ny, int nz, void* scratch, int64_t* counts,
                                      void* stream) {
  if (int rc = check_volume("tsdf_indexed_mesh_count", nx, ny, nz)) return rc;
  DEMON_REQUIRE(tsdf && weight && scratch && counts, "tsdf_indexed_mesh_count: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = (int)mc_tiles(nx, ny, nz);
  const long segs = dense_segs(nx, ny, nz);
  const DenseEdgeScratch sc(scratch, tiles, segs);
  const DenseVolume vol = make_volume(tsdf, weight, nx, ny, nz);
  DEMON_CHECK_CUDA(cudaMemsetAsync(sc.masks, 0, segs * kSegWords * sizeof(unsigned), st));
  edge_mark_kernel<<<(unsigned)ceil_div64(vol.ncubes, kMcThreads), kMcThreads, 0, st>>>(vol, sc.masks);
  DEMON_LAUNCH_CHECK();
  if (int rc = edge_scan(sc.masks, (int)segs, sc.scan, sc.base, counts, st)) return rc;
  mc_count_kernel<<<tiles, kMcThreads, 0, st>>>(vol, sc.tile_counts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(sc.tile_counts, tiles, sc.tile_first, counts + 1);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_tsdf_indexed_mesh_f32(const float* tsdf, const float* weight, const float* color, int nx, int ny, int nz, const float* origin,
                                float voxel_size, const void* scratch, float* vertices, float* normals, uint8_t* colors, int* faces,
                                void* stream) {
  if (int rc = check_volume("tsdf_indexed_mesh", nx, ny, nz)) return rc;
  DEMON_REQUIRE(origin && std::isfinite(voxel_size) && voxel_size > 0.0f, "tsdf_indexed_mesh: bad origin or voxel_size %g", voxel_size);
  DEMON_REQUIRE(!color == !colors, "tsdf_indexed_mesh: color and colors go together");
  DEMON_REQUIRE(tsdf && weight && scratch && vertices && faces, "tsdf_indexed_mesh: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = (int)mc_tiles(nx, ny, nz);
  const long segs = dense_segs(nx, ny, nz);
  const DenseEdgeScratch sc(const_cast<void*>(scratch), tiles, segs);
  const DenseVolume vol = make_volume(tsdf, weight, nx, ny, nz);
  if (int rc = launch_edge_vertices(vol, segs * kSegWords, sc.masks, sc.base, color, origin, voxel_size, vertices, normals, colors, st))
    return rc;
  mc_scatter_kernel<<<tiles, kMcThreads, 0, st>>>(vol, IndexOut{sc.masks, sc.base, faces}, sc.tile_first);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int64_t demon_sparse_tsdf_edge_scan_bytes(int blocks) { return blocks < 1 ? 0 : (int64_t)blocks * (int64_t)(sizeof(int64_t) + sizeof(int)); }

int demon_sparse_tsdf_edge_mark_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count, const int64_t* keys,
                                    const int* values, int64_t capacity, const int* rank, void* scratch, uint32_t* masks, void* stream) {
  if (int rc = check_table("sparse_tsdf_edge_mark", keys, values, capacity)) return rc;
  if (int rc = check_range("sparse_tsdf_edge_mark", m, first, count)) return rc;
  DEMON_REQUIRE(tsdf && weight && blocks && rank && scratch && masks, "sparse_tsdf_edge_mark: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int* nbr = sparse_range_neighbours(blocks, first, count, keys, values, capacity, scratch, st);
  DEMON_LAUNCH_CHECK();
  SparseVolume vol{tsdf, weight, blocks, nbr, 512L * count, nullptr, nullptr, 0, first};
  vol.rank = rank;
  edge_mark_kernel<<<(unsigned)ceil_div64(vol.ncubes, kMcThreads), kMcThreads, 0, st>>>(vol, masks);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sparse_tsdf_edge_scan(const uint32_t* masks, int blocks, void* scratch, int* base, int64_t* vertices, void* stream) {
  DEMON_REQUIRE(blocks >= 1, "sparse_tsdf_edge_scan: bad block count %d", blocks);
  DEMON_REQUIRE(masks && scratch && base && vertices, "sparse_tsdf_edge_scan: null pointer");
  return edge_scan(masks, blocks, scratch, base, vertices, (cudaStream_t)stream);
}

int demon_sparse_tsdf_indexed_mesh_range_count_f32(const float* tsdf, const float* weight, const int* blocks, int m, int first, int count,
                                                   const int* order, const int64_t* keys, const int* values, int64_t capacity, void* scratch,
                                                   int64_t* triangles, void* stream) {
  return sparse_range_count("sparse_tsdf_indexed_mesh_count", tsdf, weight, blocks, m, first, count, order, keys, values, capacity, scratch,
                            triangles, (cudaStream_t)stream);
}

int demon_sparse_tsdf_indexed_mesh_range_f32(const float* tsdf, const float* weight, const float* color, const int* blocks, int m, int first,
                                             int count, const int* order, const int64_t* keys, const int* values, int64_t capacity,
                                             const int* rank, const uint32_t* masks, const int* base, const float* origin, float voxel_size,
                                             const void* scratch, float* vertices, float* normals, uint8_t* colors, int* faces,
                                             void* stream) {
  if (int rc = check_table("sparse_tsdf_indexed_mesh", keys, values, capacity)) return rc;
  if (int rc = check_range("sparse_tsdf_indexed_mesh", m, first, count)) return rc;
  DEMON_REQUIRE(origin && std::isfinite(voxel_size) && voxel_size > 0.0f, "sparse_tsdf_indexed_mesh: bad origin or voxel_size %g", voxel_size);
  DEMON_REQUIRE(!color == !colors, "sparse_tsdf_indexed_mesh: color and colors go together");
  DEMON_REQUIRE(tsdf && weight && blocks && rank && masks && base && scratch, "sparse_tsdf_indexed_mesh: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = (int)sparse_mc_tiles(count);
  const int64_t* tile_first = static_cast<const int64_t*>(scratch);
  const int* nbr = reinterpret_cast<const int*>(tile_first + tiles) + tiles;
  SparseVolume vol{tsdf, weight, blocks, nbr, 512L * count, reinterpret_cast<const unsigned long long*>(keys), values, (long)capacity - 1,
                   first};
  vol.rank = rank;
  if (vertices) {
    if (int rc = launch_edge_vertices(vol, (long)kSegWords * count, masks, base, color, origin, voxel_size, vertices, normals, colors, st))
      return rc;
  }
  if (faces) {
    if (order)
      mc_scatter_kernel<<<tiles, kMcThreads, 0, st>>>(KeyOrderVolume{vol, order}, IndexOut{masks, base, faces}, tile_first);
    else
      mc_scatter_kernel<<<tiles, kMcThreads, 0, st>>>(vol, IndexOut{masks, base, faces}, tile_first);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

}  // extern "C"
