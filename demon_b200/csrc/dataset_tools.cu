// The compute of the reference's dataset tools (python/depthmotionnet/dataset_tools) on the device, bit for bit:
//
// * sharpness_kernel: measure_sharpness (helpers.py:23-31), np.var(laplace(grey)) of a batch of uint8 RGB frames.  Grey
//   is Pillow's convert('L'), the Laplacian scipy's [1,-2,1] per axis with half-sample symmetric edges (an exact integer),
//   and the variance numpy's: two pairwise sums over the flattened float32 array (pairwise_leaf / pairwise_subtree below).
//   One CTA per frame; the Laplacian is recomputed from the frame's bytes in both passes, never stored.
// * sun3d_depth_kernel: sun3d_utils.read_depth's arithmetic on the decoded uint16 PNG, and each frame's count of valid
//   (finite, > 0) depths.
// * depth_ratio_kernel: _compute_depth_ratios (view_tools_cython.pyx:107-159) for a batch of ordered view pairs, as a
//   ratio map or only as the two counts check_depth_consistency (view_tools.py:62-94) needs from it.
//
// Float arithmetic uses common.cuh's round-to-nearest helpers, so nothing is contracted into FMAs.
#include "common.cuh"
#include "view_projection.cuh"
#include <cstdint>

namespace demon {
namespace {

// ---- numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src, float32) -----------------------------------
// pairwise(a, n): n < 8 adds sequentially; n <= 128 keeps eight strided accumulators, combines them as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and adds the n % 8 tail sequentially; larger n splits at n2 = n/2 - (n/2) % 8 and
// returns pairwise(a, n2) + pairwise(a + n2, n - n2).  The tree depends on n alone.
constexpr int kPairwiseBlock = 128;
__host__ __device__ inline int pairwise_split(int n) {
  const int n2 = n / 2;
  return n2 - n2 % 8;
}

constexpr int kSharpThreads = 512;
constexpr int kSharpDepth = 9;   // 2^9 = kSharpThreads: the top nine levels of the tree are combined across the CTA
static_assert((1 << kSharpDepth) == kSharpThreads, "one thread per depth-9 node");
constexpr int kSharpMaxPixels = 1 << 24;   // n must be exact in float32 for the mean's and the variance's division

struct Frame {
  const uint8_t* p;   // first byte of the frame
  long sy;            // row stride in bytes (pixel stride 3, channel stride 1)
  int h, w;
  __device__ int grey(int y, int x) const {   // Pillow's ImagingConvert RGB -> L (L24 rounding)
    const uint8_t* q = p + (long)y * sy + 3 * x;
    return ((int)__ldg(q) * 19595 + (int)__ldg(q + 1) * 38470 + (int)__ldg(q + 2) * 7471 + 0x8000) >> 16;
  }
  // scipy.ndimage.laplace(mode='reflect'): [1,-2,1] along y plus along x, index -1 -> 0 and n -> n-1; exact in any precision
  __device__ float laplace(int y, int x) const {
    const int c = grey(y, x);
    const int ym = y > 0 ? y - 1 : 0, yp = y < h - 1 ? y + 1 : h - 1;
    const int xm = x > 0 ? x - 1 : 0, xp = x < w - 1 ? x + 1 : w - 1;
    return (float)((grey(ym, x) + grey(yp, x) - 2 * c) + (grey(y, xm) + grey(y, xp) - 2 * c));
  }
};

// element i of the array numpy sums: the Laplacian in pass 1, (lap - mean)^2 in pass 2 (x = arr - mean; x *= x)
template <bool kSquares>
struct Elements {
  Frame f;
  float mean;
  int x, y;   // cursor: the next element, in row-major order
  __device__ void seek(int i) {
    y = i / f.w;
    x = i - y * f.w;
  }
  __device__ float next() {
    float v = f.laplace(y, x);
    if (++x == f.w) x = 0, ++y;
    if (kSquares) {
      const float dv = fsub(v, mean);
      v = fmul(dv, dv);
    }
    return v;
  }
};

template <bool kSquares>
__device__ float pairwise_leaf(Elements<kSquares>& e, int off, int n) {
  e.seek(off);
  if (n < 8) {
    float res = 0.0f;
    for (int i = 0; i < n; ++i) res = fadd(res, e.next());
    return res;
  }
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = e.next();
  int i = 8;
  for (; i < n - n % 8; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = fadd(r[j], e.next());
  }
  float res = fadd(fadd(fadd(r[0], r[1]), fadd(r[2], r[3])), fadd(fadd(r[4], r[5]), fadd(r[6], r[7])));
  for (; i < n; ++i) res = fadd(res, e.next());
  return res;
}

// pairwise(a + off, n) by a post-order walk with an explicit stack: each entry is an internal node whose left sum is
// pending (have_left = 0) or done, and it remembers its right child.
template <bool kSquares>
__device__ float pairwise_subtree(Elements<kSquares>& e, int off, int n) {
  constexpr int kMaxDepth = 32;   // n < 2^24 halves to 128 in fewer than 20 levels
  int right_off[kMaxDepth], right_n[kMaxDepth];
  float left[kMaxDepth];
  bool have_left[kMaxDepth];
  int sp = 0;
  for (;;) {
    while (n > kPairwiseBlock) {
      const int n2 = pairwise_split(n);
      right_off[sp] = off + n2;
      right_n[sp] = n - n2;
      have_left[sp] = false;
      ++sp;
      n = n2;
    }
    float v = pairwise_leaf(e, off, n);
    while (sp > 0 && have_left[sp - 1]) {
      v = fadd(left[sp - 1], v);
      --sp;
    }
    if (sp == 0) return v;
    have_left[sp - 1] = true;
    left[sp - 1] = v;
    off = right_off[sp - 1];
    n = right_n[sp - 1];
  }
}

// The whole tree over the CTA: thread t follows the bits of t (most significant first, 0 = left) down from the root for
// kSharpDepth levels or until it reaches a leaf at depth `stop`; the node it reaches is owned by the thread whose path
// below `stop` is all left turns, which sums it alone.  The levels above are combined in shared memory, deepest first.
template <bool kSquares>
__device__ float pairwise_cta(Elements<kSquares>& e, int total, float* s_val) {
  const int t = threadIdx.x;
  int off = 0, n = total, stop = 0;
  while (stop < kSharpDepth && n > kPairwiseBlock) {
    const int n2 = pairwise_split(n);
    if ((t >> (kSharpDepth - 1 - stop)) & 1) {
      off += n2;
      n -= n2;
    } else {
      n = n2;
    }
    ++stop;
  }
  const bool owner = (t & ((1 << (kSharpDepth - stop)) - 1)) == 0;
  s_val[t] = owner ? pairwise_subtree(e, off, n) : 0.0f;
  __syncthreads();
  for (int s = kSharpDepth - 1; s >= 0; --s) {
    const int stride = 1 << (kSharpDepth - 1 - s);
    // thread t (low kSharpDepth - s bits zero) holds the depth-s node on its path; it is internal iff stop > s
    if ((t & (2 * stride - 1)) == 0 && stop > s) s_val[t] = fadd(s_val[t], s_val[t + stride]);
    __syncthreads();
  }
  const float root = s_val[0];
  __syncthreads();   // s_val is reused by the next pass
  return root;
}

__global__ void __launch_bounds__(kSharpThreads) sharpness_kernel(const uint8_t* __restrict__ images, long stride_n, long stride_y,
                                                                  int h, int w, float* __restrict__ out) {
  __shared__ float s_val[kSharpThreads];
  const Frame f{images + (long)blockIdx.x * stride_n, stride_y, h, w};
  const int total = h * w;
  const float count = (float)total;   // exact: total < 2^24
  Elements<false> lap{f, 0.0f, 0, 0};
  const float mean = fdiv(pairwise_cta(lap, total, s_val), count);
  Elements<true> sq{f, mean, 0, 0};
  const float var = fdiv(pairwise_cta(sq, total, s_val), count);
  if (threadIdx.x == 0) out[blockIdx.x] = var;
}

// ---- SUN3D depth ----------------------------------------------------------------------------------------------------
constexpr int kDepthThreads = 256;
constexpr int kDepthPerThread = 8;

__global__ void __launch_bounds__(kDepthThreads) sun3d_depth_kernel(const uint16_t* __restrict__ raw, long hw,
                                                                    float* __restrict__ depth,
                                                                    unsigned long long* __restrict__ valid) {
  __shared__ int s_warp[kDepthThreads / 32];
  const long base = (long)blockIdx.y * hw;
  int c = 0;
#pragma unroll
  for (int k = 0; k < kDepthPerThread; ++k) {
    const long i = ((long)blockIdx.x * kDepthPerThread + k) * kDepthThreads + threadIdx.x;
    if (i < hw) {
      const unsigned d = __ldg(raw + base + i);
      const unsigned s = ((d >> 3) | (d << 13)) & 0xffffu;   // (depth_uint16 >> 3) | (depth_uint16 << 13) in uint16
      const float z = __double2float_rn(__ddiv_rn((double)s, 1000.0));   // (depth_shifted / 1000).astype(np.float32)
      depth[base + i] = z;
      c += z > 0.0f ? 1 : 0;   // every value is finite
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
#pragma unroll
    for (int k = 0; k < kDepthThreads / 32; ++k) s += s_warp[k];
    if (s) atomicAdd(valid + blockIdx.y, (unsigned long long)s);
  }
}

// ---- depth ratios -----------------------------------------------------------------------------------------------------
constexpr int kRatioThreads = 256;
constexpr int kRatioPerThread = 4;
constexpr int kRatioTile = kRatioThreads * kRatioPerThread;

// _compute_depth_ratios at pixel (x, y) of view 1 (depth d) against view 2's depth d2 [h*w]: NaN where the .pyx leaves NaN.
// x2 = max(0, min(w, round(u))) uses Python's round (half to even) and may equal w; the .pyx then reads flat element
// y2*w + x2 without a bounds check: the next row's first pixel, or past the array (undefined) when that is >= h*w, which
// stays NaN here (DESIGN.md §7).
__device__ __forceinline__ float depth_ratio(float d, int x, int y, int h, int w, const float* K, const float* RT, const float* t,
                                             const float* P, const float* __restrict__ d2map) {
  float u, v, z;
  if (!(isfinite(d) && d > 0.0f && project_into_view2(d, x, y, K, RT, t, P, u, v, z))) return __int_as_float(0x7fc00000);
  if (!(u > 0.0f && v > 0.0f && u < (float)w && v < (float)h)) return __int_as_float(0x7fc00000);
  const int x2 = min(w, (int)rintf(u)), y2 = min(h, (int)rintf(v));   // u, v > 0: the max(0, .) never binds
  const long flat = (long)y2 * w + x2;
  if (flat >= (long)h * w) return __int_as_float(0x7fc00000);
  const float d2 = __ldg(d2map + flat);
  if (!(d2 > 0.0f && isfinite(d2))) return __int_as_float(0x7fc00000);
  return fdiv(z, d2);
}

// grid (pairs, pixel tiles); kCounts: counts[2p] += finite ratios, counts[2p+1] += finite ratios with lo < r < hi
template <bool kCounts>
__global__ void __launch_bounds__(kRatioThreads) depth_ratio_kernel(const float* __restrict__ depth, const float* __restrict__ K,
                                                                    const float* __restrict__ R, const float* __restrict__ t,
                                                                    const float* __restrict__ P, int n_views, int h, int w,
                                                                    const int* __restrict__ pairs, float* __restrict__ ratios,
                                                                    float lo, float hi, unsigned long long* __restrict__ counts) {
  __shared__ float cam[33];   // K_i (9), R_i^T (9), t_i (3), P_j (12)
  __shared__ int s_cnt[2][kRatioThreads / 32];
  const long p = blockIdx.x;
  const int i = __ldg(pairs + 2 * p), j = __ldg(pairs + 2 * p + 1);
  const bool ok = i >= 0 && i < n_views && j >= 0 && j < n_views;   // checked on the host; a bad pair gives NaN / no counts
  if (ok) {
    if (threadIdx.x < 9) {
      const int r = threadIdx.x / 3, c = threadIdx.x % 3;
      cam[threadIdx.x] = K[9L * i + threadIdx.x];
      cam[9 + threadIdx.x] = R[9L * i + c * 3 + r];   // RT = R1.transpose() (.pyx:122)
    } else if (threadIdx.x < 12) {
      cam[18 + threadIdx.x - 9] = t[3L * i + threadIdx.x - 9];
    } else if (threadIdx.x < 24) {
      cam[21 + threadIdx.x - 12] = P[12L * j + threadIdx.x - 12];
    }
  }
  __syncthreads();
  const long hw = (long)h * w;
  const float* d1 = depth + (long)i * hw;
  const float* d2 = depth + (long)j * hw;
  int finite = 0, consistent = 0;
#pragma unroll
  for (int k = 0; k < kRatioPerThread; ++k) {
    const long q = (long)blockIdx.y * kRatioTile + k * kRatioThreads + threadIdx.x;
    if (q >= hw) break;
    float r = __int_as_float(0x7fc00000);
    if (ok) {
      const int y = (int)(q / w), x = (int)(q - (long)y * w);
      r = depth_ratio(__ldg(d1 + q), x, y, h, w, cam, cam + 9, cam + 18, cam + 21, d2);
    }
    if (kCounts) {
      const bool f = isfinite(r);   // a denormal d2 gives inf, which is not finite
      finite += f ? 1 : 0;
      consistent += (f && r > lo && r < hi) ? 1 : 0;
    } else {
      ratios[p * hw + q] = r;
    }
  }
  if (kCounts) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      finite += __shfl_xor_sync(0xffffffffu, finite, o);
      consistent += __shfl_xor_sync(0xffffffffu, consistent, o);
    }
    if ((threadIdx.x & 31) == 0) {
      s_cnt[0][threadIdx.x >> 5] = finite;
      s_cnt[1][threadIdx.x >> 5] = consistent;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
      int s = 0;
#pragma unroll
      for (int k = 0; k < kRatioThreads / 32; ++k) s += s_cnt[threadIdx.x][k];
      if (s) atomicAdd(counts + 2 * p + threadIdx.x, (unsigned long long)s);   // integer sums: order does not matter
    }
  }
}

template <bool kCounts>
int depth_ratios(const float* depth, const float* K, const float* R, const float* t, const float* P, int n_views, int h, int w,
                 const int* pairs, int n_pairs, float* ratios, float lo, float hi, int64_t* counts, void* stream) {
  const char* name = kCounts ? "depth_consistency_counts" : "depth_ratios";
  DEMON_REQUIRE(n_views >= 0 && n_pairs >= 0 && h >= 0 && w >= 0, "%s: bad size %d views of %dx%d, %d pairs", name, n_views, h, w,
                n_pairs);
  const long hw = (long)h * w;
  DEMON_REQUIRE(hw < kSharpMaxPixels, "%s: %dx%d pixels per view is too many (h*w must be below 2^24)", name, h, w);
  if (kCounts && n_pairs > 0) {
    DEMON_REQUIRE(counts, "%s: null pointer", name);
    DEMON_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 2 * n_pairs, (cudaStream_t)stream));
  }
  if (n_pairs == 0 || hw == 0) return DEMON_OK;
  DEMON_REQUIRE(n_views > 0, "%s: pairs without views", name);
  DEMON_REQUIRE(depth && K && R && t && P && pairs && (kCounts || ratios), "%s: null pointer", name);
  const dim3 grid((unsigned)n_pairs, (unsigned)((hw + kRatioTile - 1) / kRatioTile));
  depth_ratio_kernel<kCounts><<<grid, kRatioThreads, 0, (cudaStream_t)stream>>>(
      depth, K, R, t, P, n_views, h, w, pairs, ratios, lo, hi, reinterpret_cast<unsigned long long*>(counts));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int demon_sharpness_u8(const uint8_t* images, int64_t stride_n, int64_t stride_y, int n, int h, int w, float* out, void* stream) {
  DEMON_REQUIRE(n >= 0 && h >= 1 && w >= 1, "sharpness: bad size %d frames of %dx%d", n, h, w);
  DEMON_REQUIRE((long)h * w < kSharpMaxPixels, "sharpness: %dx%d pixels per frame is too many (h*w must be below 2^24)", h, w);
  DEMON_REQUIRE(stride_n >= 0 && stride_y >= 0, "sharpness: negative strides are not supported");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(images && out, "sharpness: null pointer");
  sharpness_kernel<<<(unsigned)n, kSharpThreads, 0, (cudaStream_t)stream>>>(images, stride_n, stride_y, h, w, out);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_sun3d_depth_u16(const uint16_t* raw, int n, int h, int w, float* depth, int64_t* valid_counts, void* stream) {
  DEMON_REQUIRE(n >= 0 && n <= 65535 && h >= 0 && w >= 0, "sun3d_depth: bad size %d frames of %dx%d (up to 65535 frames)", n, h, w);
  const long hw = (long)h * w;
  DEMON_REQUIRE(hw < (1L << 31), "sun3d_depth: %dx%d pixels per frame is too many", h, w);
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(valid_counts, "sun3d_depth: null pointer");
  DEMON_CHECK_CUDA(cudaMemsetAsync(valid_counts, 0, sizeof(int64_t) * n, (cudaStream_t)stream));
  if (hw == 0) return DEMON_OK;
  DEMON_REQUIRE(raw && depth, "sun3d_depth: null pointer");
  const long per_block = (long)kDepthThreads * kDepthPerThread;
  sun3d_depth_kernel<<<dim3((unsigned)((hw + per_block - 1) / per_block), (unsigned)n), kDepthThreads, 0, (cudaStream_t)stream>>>(
      raw, hw, depth, reinterpret_cast<unsigned long long*>(valid_counts));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_depth_ratios_f32(const float* depth, const float* K, const float* R, const float* t, const float* P, int n_views, int h, int w,
                           const int* pairs, int n_pairs, float* ratios, void* stream) {
  return depth_ratios<false>(depth, K, R, t, P, n_views, h, w, pairs, n_pairs, ratios, 0.0f, 0.0f, nullptr, stream);
}

int demon_depth_consistency_counts_f32(const float* depth, const float* K, const float* R, const float* t, const float* P, int n_views,
                                       int h, int w, const int* pairs, int n_pairs, float lo, float hi, int64_t* counts, void* stream) {
  return depth_ratios<true>(depth, K, R, t, P, n_views, h, w, pairs, n_pairs, nullptr, lo, hi, counts, stream);
}

}  // extern "C"
