// Point clouds of depth maps on the device: compute_point_cloud_from_depthmap (python/depthmotionnet/vis_cython.pyx:24-173)
// for n views, bit for bit.  The .pyx keeps the valid pixels (finite and > 0) in row-major order and emits the point
// R^T (K^-1 (x+.5, y+.5, 1) d - t), the normal rotated by R^T and the colour of each; every float operation here is the
// .pyx's float32 C operation in its order, with round-to-nearest intrinsics (no contraction into FMAs).
//
// The compaction is deterministic: launch 1 counts the valid pixels of every 2048-pixel tile into the caller's scratch;
// launch 2 gives each tile its start (the sum of the counts of the tiles before it in its sample) and ranks the tile's
// valid pixels by ballots, so an output row depends only on the pixel order, never on scheduling.
#include "common.cuh"
#include "geometry.cuh"
#include <cstdint>

namespace demon {
namespace {

constexpr int kVisThreads = 256;
constexpr int kVisWarps = kVisThreads / 32;
constexpr int kVisRounds = 8;
constexpr int kVisTile = kVisThreads * kVisRounds;   // round j of thread i reads pixel tile * kVisTile + j * kVisThreads + i
constexpr int kVisMaxSide = 8192;

long vis_tiles(int h, int w) { return ((long)h * w + kVisTile - 1) / kVisTile; }

// the .pyx's predicate (:55, 88, 107) on pixel p of one view; d is the camera z it tests (1/inverse depth with kInverse,
// as visualize_prediction's `depth = 1/inverse_depth`, vis.py:246)
template <bool kInverse>
__device__ __forceinline__ bool vis_valid(const float* __restrict__ depth, long p, long hw, float& d) {
  if (p >= hw) return false;
  d = __ldg(depth + p);
  if (kInverse) d = fdiv(1.0f, d);
  return isfinite(d) && d > 0.0f;
}

template <bool kInverse>
__global__ void __launch_bounds__(kVisThreads) point_cloud_count_kernel(const float* __restrict__ depth, long hw, int tiles,
                                                                        int* __restrict__ tile_counts) {
  __shared__ int s_warp[kVisWarps];
  const int n = blockIdx.y, tile = blockIdx.x;
  const float* dn = depth + (long)n * hw;
  const long base = (long)tile * kVisTile + threadIdx.x;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kVisRounds; ++j) {
    float d;
    c += vis_valid<kInverse>(dn, base + j * kVisThreads, hw, d) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
#pragma unroll
    for (int k = 0; k < kVisWarps; ++k) s += s_warp[k];
    tile_counts[(long)n * tiles + tile] = s;
  }
}

template <bool kInverse>
__global__ void __launch_bounds__(kVisThreads) point_cloud_scatter_kernel(
    const float* __restrict__ depth, const float* __restrict__ K, const float* __restrict__ R, const float* __restrict__ t,
    const float* __restrict__ normals, const uint8_t* __restrict__ colors, const float* __restrict__ image, int h, int w, int tiles,
    const int* __restrict__ tile_counts, float* __restrict__ points, float* __restrict__ normals_out, uint8_t* __restrict__ colors_out,
    int* __restrict__ counts) {
  __shared__ float cam[16];   // K[0,0], K[1,1], K[0,2], K[1,2], R row-major (9), t (3) of this sample
  __shared__ int s_cnt[kVisRounds][kVisWarps];
  __shared__ int s_prev[kVisWarps];
  const int n = blockIdx.y, tile = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < 9) {
    cam[4 + threadIdx.x] = R[9 * n + threadIdx.x];
  } else if (threadIdx.x < 12) {
    cam[13 + threadIdx.x - 9] = t[3 * n + threadIdx.x - 9];
  } else if (threadIdx.x < 16) {
    const int k = threadIdx.x - 12;
    cam[k] = K[9 * n + (k == 0 ? 0 : k == 1 ? 4 : k == 2 ? 2 : 5)];
  }
  int prev = 0;   // valid pixels of the tiles before this one
  for (int k = threadIdx.x; k < tile; k += kVisThreads) prev += tile_counts[(long)n * tiles + k];
#pragma unroll
  for (int o = 16; o; o >>= 1) prev += __shfl_xor_sync(0xffffffffu, prev, o);
  if (lane == 0) s_prev[warp] = prev;

  const long hw = (long)h * w;
  const float* dn = depth + (long)n * hw;
  const long base = (long)tile * kVisTile + threadIdx.x;
  float d[kVisRounds];
  unsigned ballot[kVisRounds];
#pragma unroll
  for (int j = 0; j < kVisRounds; ++j) {
    d[j] = 0.0f;
    ballot[j] = __ballot_sync(0xffffffffu, vis_valid<kInverse>(dn, base + j * kVisThreads, hw, d[j]));
    if (lane == 0) s_cnt[j][warp] = __popc(ballot[j]);
  }
  __syncthreads();

  int row = 0;   // output row of the first valid pixel of round j in this tile
#pragma unroll
  for (int k = 0; k < kVisWarps; ++k) row += s_prev[k];
  const float inv_fx = fdiv(1.0f, cam[0]), inv_fy = fdiv(1.0f, cam[1]);   // .pyx:41-42 multiplies by these
  const float cx = cam[2], cy = cam[3];
  const float* Rm = cam + 4;
  const float* tv = cam + 13;
  const unsigned lanes_below = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < kVisRounds; ++j) {
    int before = 0, total = 0;
#pragma unroll
    for (int k = 0; k < kVisWarps; ++k) {
      const int c = s_cnt[j][k];
      total += c;
      before += k < warp ? c : 0;
    }
    if ((ballot[j] >> lane) & 1u) {
      const long p = base + j * kVisThreads;
      const long o = ((long)n * hw + row + before + __popc(ballot[j] & lanes_below)) * 3;
      const int y = (int)(p / w), x = (int)(p - (long)y * w);
      const float dd = d[j];
      // .pyx:67-72: tmp = (d*((x+0.5) - cx)*inv_fx - t0, d*((y+0.5) - cy)*inv_fy - t1, d - t2), X = R^T tmp
      const float tmp0 = fsub(fmul(fmul(dd, fsub(fadd((float)x, 0.5f), cx)), inv_fx), tv[0]);
      const float tmp1 = fsub(fmul(fmul(dd, fsub(fadd((float)y, 0.5f), cy)), inv_fy), tv[1]);
      const float tmp2 = fsub(dd, tv[2]);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        points[o + c] = fadd(fadd(fmul(Rm[c], tmp0), fmul(Rm[3 + c], tmp1)), fmul(Rm[6 + c], tmp2));
      if (normals) {   // .pyx:86-99, the same rotation without the translation
        const float* nn = normals + (long)n * 3 * hw + p;
        const float n0 = __ldg(nn), n1 = __ldg(nn + hw), n2 = __ldg(nn + 2 * hw);
#pragma unroll
        for (int c = 0; c < 3; ++c) normals_out[o + c] = fadd(fadd(fmul(Rm[c], n0), fmul(Rm[3 + c], n1)), fmul(Rm[6 + c], n2));
      }
      if (colors) {   // .pyx:103-113: planar uint8 copied as is
        const uint8_t* cc = colors + (long)n * 3 * hw + p;
#pragma unroll
        for (int c = 0; c < 3; ++c) colors_out[o + c] = __ldg(cc + c * hw);
      } else if (image) {
        // ((image+0.5)*255).astype(np.uint8) (vis.py:276): two float32 operations, then numpy's cast, which on x86 keeps
        // the low byte of cvttss2si (NaN, infinities and values out of int32 range give 0x80000000, so 0)
        const float* im = image + (long)n * 3 * hw + p;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          colors_out[o + c] = (uint8_t)(cvtt_x86(fmul(fadd(__ldg(im + c * hw), 0.5f), 255.0f)) & 0xff);
      }
    }
    row += total;
  }
  if (tile == tiles - 1 && threadIdx.x == 0) counts[n] = row;
}

template <bool kInverse>
int point_cloud(const float* depth, const float* K, const float* R, const float* t, const float* normals, const uint8_t* colors,
                const float* image, int n, int h, int w, void* scratch, float* points, float* normals_out, uint8_t* colors_out,
                int* counts, void* stream) {
  DEMON_REQUIRE(n >= 0 && n <= 65535 && h >= 1 && w >= 1 && h <= kVisMaxSide && w <= kVisMaxSide,
                "point_cloud: bad size %d views of %dx%d (1..%d per side, up to 65535 views)", n, h, w, kVisMaxSide);
  DEMON_REQUIRE(!(colors && image), "point_cloud: pass uint8 colors or a float image, not both");
  DEMON_REQUIRE(!normals == !normals_out, "point_cloud: normals and normals_out go together");
  DEMON_REQUIRE(!(colors || image) == !colors_out, "point_cloud: colors_out goes with colors or image");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && K && R && t && scratch && points && counts, "point_cloud: null pointer");
  const long hw = (long)h * w;
  const int tiles = (int)vis_tiles(h, w);
  int* tile_counts = static_cast<int*>(scratch);
  const dim3 grid((unsigned)tiles, (unsigned)n);
  point_cloud_count_kernel<kInverse><<<grid, kVisThreads, 0, (cudaStream_t)stream>>>(depth, hw, tiles, tile_counts);
  DEMON_LAUNCH_CHECK();
  point_cloud_scatter_kernel<kInverse><<<grid, kVisThreads, 0, (cudaStream_t)stream>>>(
      depth, K, R, t, normals, colors, image, h, w, tiles, tile_counts, points, normals_out, colors_out, counts);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int64_t demon_point_cloud_scratch_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return (int64_t)n * vis_tiles(h, w) * (int64_t)sizeof(int);
}

int demon_point_cloud_f32(const float* depth, const float* K, const float* R, const float* t, const float* normals,
                          const uint8_t* colors, const float* image, int n, int h, int w, void* scratch, float* points,
                          float* normals_out, uint8_t* colors_out, int* counts, void* stream) {
  return point_cloud<false>(depth, K, R, t, normals, colors, image, n, h, w, scratch, points, normals_out, colors_out, counts, stream);
}

int demon_point_cloud_inverse_f32(const float* inverse_depth, const float* K, const float* R, const float* t, const float* normals,
                                  const uint8_t* colors, const float* image, int n, int h, int w, void* scratch, float* points,
                                  float* normals_out, uint8_t* colors_out, int* counts, void* stream) {
  return point_cloud<true>(inverse_depth, K, R, t, normals, colors, image, n, h, w, scratch, points, normals_out, colors_out, counts,
                           stream);
}

}  // extern "C"
