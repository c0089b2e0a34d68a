// Resize of RGB uint8 images, bit for bit what Pillow's `Image.resize` returns for NEAREST, BILINEAR and BICUBIC
// (examples/example.py:15-22 resizes every input with it).
//
// The model, per axis resized from `in` to `out` samples (scale = in / out, all in double):
//   BILINEAR / BICUBIC  separable: a horizontal pass, then a vertical pass over its uint8 result; a pass whose axis keeps its
//                       size is skipped.  Output index i reads the inputs [lo, lo + cnt) with
//                         fs = max(scale, 1), support = r * fs (r = 1 triangle, 2 cubic a = -0.5), center = (i + 0.5) * scale,
//                         lo = max(trunc(center - support + 0.5), 0), cnt = min(trunc(center + support + 0.5), in) - lo,
//                         w_j = f(((lo + j) - center + 0.5) * (1 / fs)) / sum_j w_j  (the division skipped if the sum is 0),
//                         k_j = trunc(w_j * 2^22 + 0.5) (w_j >= 0) or trunc(w_j * 2^22 - 0.5) (w_j < 0),
//                         out = clamp((2^21 + sum_j k_j * v_j) >> 22, 0, 255) in int32.
//                       Pillow runs the vertical pass first instead when the source is more than 100 times taller than
//                       wide and the height shrinks (h > 100 w and oh < h); the kernel then works on the transposed image
//                       (swapped strides).
//   NEAREST             out[i] = in[trunc(x_i)], x_0 = scale / 2, x_{i+1} = x_i + scale: a running double sum, which is not
//                       always trunc((i + 0.5) * scale) (64 -> 48 differs).
// Every double operation is an _rn intrinsic so that nvcc contracts nothing into an FMA (DESIGN.md section 3.3).
//
// One CTA owns a tile of kTX x kTY output pixels of one image.  It walks the source rows its vertical support needs in
// chunks of kRows: the horizontal pass of a chunk goes to shared memory as uint8, the vertical pass accumulates the chunk
// into per-pixel int32 sums in registers (integer sums: chunking changes nothing).  The horizontal weights of the tile's
// columns are computed in chunks of kTaps taps, so shared memory is a fixed 25,728 bytes whatever the scale: at the largest
// downscale allowed (8192 -> 1, BICUBIC: 8192 taps per output sample) a tile makes 64 tap chunks per row chunk instead of
// one.  NEAREST and an unchanged axis are a single tap of weight 2^22, which reproduces the input byte exactly.
#include "images.cuh"

namespace demon {
namespace {

constexpr int kTX = 32;        // output columns per CTA (one warp lane each)
constexpr int kTY = 8;         // output rows per CTA (one warp each)
constexpr int kThreads = kTX * kTY;
constexpr int kRows = 64;      // source rows per chunk
constexpr int kTaps = 128;     // horizontal taps per weight chunk
constexpr int kPairs = kRows * kTX / kThreads;   // (source row, output column) pairs of a chunk per thread
constexpr int kOne = 1 << 22;  // 1.0 in the 22-fraction-bit fixed point of the weights
constexpr int kHalf = 1 << 21;
constexpr int kMaxSide = 8192;

// what one axis does
enum AxisFilter { kAxisNearest = 0, kAxisCopy = 1, kAxisTriangle = 2, kAxisCubic = 3 };

__device__ __forceinline__ double filter_value(int f, double x) {
  x = fabs(x);
  if (f == kAxisTriangle) return x < 1.0 ? fsub(1.0, x) : 0.0;
  if (x < 1.0) return fadd(fmul(fmul(fsub(fmul(1.5, x), 2.5), x), x), 1.0);         // ((a + 2) x - (a + 3)) x x + 1
  if (x < 2.0) return fmul(fsub(fmul(fadd(fmul(fsub(x, 5.0), x), 8.0), x), 4.0), -0.5);   // (((x - 5) x + 8) x - 4) a
  return 0.0;
}

struct AxisScale { double scale, support, ss; };

__device__ __forceinline__ AxisScale axis_scale(int f, int in, int out) {
  AxisScale a;
  a.scale = fdiv((double)in, (double)out);
  const double fs = fmax(a.scale, 1.0);
  a.support = fmul(f == kAxisTriangle ? 1.0 : 2.0, fs);
  a.ss = fdiv(1.0, fs);
  return a;
}

// unnormalised weight of input sample `src` for an output sample centred at `center`
__device__ __forceinline__ double raw_weight(int f, int src, double center, double ss) {
  return filter_value(f, fmul(fadd(fsub((double)src, center), 0.5), ss));
}

// fixed-point weight of input sample `src`; ww: the sum of the output sample's raw weights
__device__ __forceinline__ int tap_weight(int f, int src, double center, double ww, double ss) {
  if (f == kAxisNearest || f == kAxisCopy) return kOne;
  double w = raw_weight(f, src, center, ss);
  if (ww != 0.0) w = fdiv(w, ww);
  const double k = fmul(w, (double)kOne);
  return (int)(w < 0.0 ? fsub(k, 0.5) : fadd(k, 0.5));
}

// The taps of output samples [i0, i0 + count) of one axis (count <= 32), computed by one warp: lo, cnt and, for the
// convolution filters, the center and the weight sum.  Samples past `out` get cnt = 0.
__device__ void axis_setup(int f, int in, int out, int i0, int count, int lane, int* lo, int* cnt, double* center, double* ww) {
  if (f == kAxisNearest) {
    if (lane == 0) {
      const double scale = fdiv((double)in, (double)out);
      double x = fmul(scale, 0.5);
      for (int i = 0; i < i0 + count; ++i, x = fadd(x, scale)) {
        if (i < i0) continue;
        const bool valid = i < out;
        lo[i - i0] = valid ? min((int)x, in - 1) : 0;
        cnt[i - i0] = valid ? 1 : 0;
        center[i - i0] = 0.0;   // not read by tap_weight for a single tap, but every argument it gets is defined
        ww[i - i0] = 0.0;
      }
    }
    return;
  }
  if (lane >= count) return;
  const int i = i0 + lane;
  if (i >= out) { lo[lane] = 0; cnt[lane] = 0; center[lane] = 0.0; ww[lane] = 0.0; return; }
  if (f == kAxisCopy) { lo[lane] = i; cnt[lane] = 1; center[lane] = 0.0; ww[lane] = 0.0; return; }
  const AxisScale a = axis_scale(f, in, out);
  const double c = fmul(fadd((double)i, 0.5), a.scale);
  const int l = max((int)fadd(fsub(c, a.support), 0.5), 0);
  const int h = min((int)fadd(fadd(c, a.support), 0.5), in);
  double s = 0.0;
  for (int j = l; j < h; ++j) s = fadd(s, raw_weight(f, j, c, a.ss));
  lo[lane] = l; cnt[lane] = h - l; center[lane] = c; ww[lane] = s;
}

__device__ __forceinline__ unsigned char clip8(int v) { return (unsigned char)min(max(v >> 22, 0), 255); }

// grid (ceil(ow / kTX), ceil(oh / kTY), n); fx / fy: AxisFilter of the first (horizontal) / second (vertical) pass.
// sy / sx: source bytes between rows / pixels; dn / dy / dx: output bytes between images / rows / pixels.
__global__ void __launch_bounds__(kThreads) resize_u8_kernel(const unsigned char* __restrict__ src, long s_outer, long s_inner, int per,
                                                             long sy, long sx, int h, int w, unsigned char* __restrict__ dst, long dn,
                                                             long dy, long dx, int oh, int ow, int fx, int fy) {
  __shared__ int x_lo[kTX], x_cnt[kTX], y_lo[kTY], y_cnt[kTY];
  __shared__ double x_center[kTX], x_ww[kTX], y_center[kTY], y_ww[kTY];
  __shared__ int hk[kTX][kTaps + 1];                   // horizontal weights of one tap chunk (+1: lanes read one column each)
  __shared__ int vk[kTY][kRows];                       // vertical weights of the current row chunk
  __shared__ unsigned char rows[kRows][kTX * 3];       // horizontal pass of the current row chunk
  __shared__ unsigned char row_used[kRows];

  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY, z = blockIdx.z;
  const unsigned char* img = src + (long)(z / per) * s_outer + (long)(z % per) * s_inner;
  if (warp == 0) axis_setup(fx, w, ow, x0, kTX, lane, x_lo, x_cnt, x_center, x_ww);
  if (warp == 1) axis_setup(fy, h, oh, y0, kTY, lane, y_lo, y_cnt, y_center, y_ww);
  pdl_wait();
  __syncthreads();

  const double ssx = (fx >= kAxisTriangle) ? axis_scale(fx, w, ow).ss : 0.0;
  const double ssy = (fy >= kAxisTriangle) ? axis_scale(fy, h, oh).ss : 0.0;
  int max_cnt = 0, r0 = h, r1 = 0;
#pragma unroll
  for (int c = 0; c < kTX; ++c) max_cnt = max(max_cnt, x_cnt[c]);
#pragma unroll
  for (int y = 0; y < kTY; ++y)
    if (y_cnt[y] > 0) { r0 = min(r0, y_lo[y]); r1 = max(r1, y_lo[y] + y_cnt[y]); }
  const int tap_chunks = (max_cnt + kTaps - 1) / kTaps;
  auto fill_hk = [&](int j0) {
    for (int e = tid; e < kTX * kTaps; e += kThreads) {
      const int c = e / kTaps, j = e % kTaps;
      hk[c][j] = (j0 + j < x_cnt[c]) ? tap_weight(fx, x_lo[c] + j0 + j, x_center[c], x_ww[c], ssx) : 0;
    }
  };
  if (tap_chunks == 1) fill_hk(0);   // used after the first barrier of the row loop

  const int ty = warp, tx = lane;    // the output pixel whose vertical sums this thread keeps
  int acc[3] = {kHalf, kHalf, kHalf};
  for (int rc = r0; rc < r1; rc += kRows) {
    const int nrows = min(kRows, r1 - rc);
    for (int e = tid; e < kTY * kRows; e += kThreads) {
      const int y = e / kRows, i = e % kRows, r = rc + i;
      const bool in_support = i < nrows && r >= y_lo[y] && r < y_lo[y] + y_cnt[y];
      vk[y][i] = in_support ? tap_weight(fy, r, y_center[y], y_ww[y], ssy) : 0;
    }
    if (tid < kRows) {   // NEAREST reads a few of the rows its tile spans; the convolutions read all of them
      bool used = false;
#pragma unroll
      for (int y = 0; y < kTY; ++y) used |= (rc + tid >= y_lo[y] && rc + tid < y_lo[y] + y_cnt[y]);
      row_used[tid] = used && tid < nrows;
    }
    __syncthreads();

    // horizontal pass: thread (warp, lane) takes source rows warp, warp + kTY, ... of the chunk at output column lane
    int hacc[kPairs][3];
#pragma unroll
    for (int p = 0; p < kPairs; ++p) hacc[p][0] = hacc[p][1] = hacc[p][2] = kHalf;
    for (int t = 0; t < tap_chunks; ++t) {
      const int j0 = t * kTaps;
      if (tap_chunks > 1) { __syncthreads(); fill_hk(j0); __syncthreads(); }
      const int j1 = min(x_cnt[tx], j0 + kTaps);
#pragma unroll
      for (int p = 0; p < kPairs; ++p) {
        const int i = p * kTY + ty;
        if (!row_used[i]) continue;
        const unsigned char* px = img + (long)(rc + i) * sy + (long)(x_lo[tx] + j0) * sx;
        for (int j = j0; j < j1; ++j, px += sx) {
          const int k = hk[tx][j - j0];
          hacc[p][0] += k * (int)__ldg(px);
          hacc[p][1] += k * (int)__ldg(px + 1);
          hacc[p][2] += k * (int)__ldg(px + 2);
        }
      }
    }
#pragma unroll
    for (int p = 0; p < kPairs; ++p) {
      const int i = p * kTY + ty;
#pragma unroll
      for (int c = 0; c < 3; ++c) rows[i][tx * 3 + c] = clip8(hacc[p][c]);
    }
    __syncthreads();

    // vertical pass over the chunk
    const int i0 = max(y_lo[ty] - rc, 0), i1 = min(y_lo[ty] + y_cnt[ty] - rc, nrows);
    for (int i = i0; i < i1; ++i) {
      const int k = vk[ty][i];
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] += k * (int)rows[i][tx * 3 + c];
    }
    __syncthreads();
  }
  const int x = x0 + tx, y = y0 + ty;
  if (x < ow && y < oh) {
    unsigned char* o = dst + z * dn + y * dy + x * dx;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = clip8(acc[c]);
  }
}

}  // namespace

int resize_u8_check(int h, int w, int oh, int ow, int resample, const char* who) {
  DEMON_REQUIRE(h >= 1 && w >= 1 && h <= kMaxSide && w <= kMaxSide, "%s: source size %dx%d (width x height) outside 1..%d", who, w, h,
                kMaxSide);
  DEMON_REQUIRE(oh >= 1 && ow >= 1 && oh <= kMaxSide && ow <= kMaxSide, "%s: output size %dx%d (width x height) outside 1..%d", who, ow,
                oh, kMaxSide);
  DEMON_REQUIRE(resample == DEMON_RESAMPLE_NEAREST || resample == DEMON_RESAMPLE_BILINEAR || resample == DEMON_RESAMPLE_BICUBIC,
                "%s: resample %d is not NEAREST (0), BILINEAR (2) or BICUBIC (3)", who, resample);
  return DEMON_OK;
}

int resize_u8_launch(const uint8_t* src, int64_t s_outer, int64_t s_inner, int per, int64_t sy, int n, int h, int w, uint8_t* dst,
                     int oh, int ow, int resample, cudaStream_t stream) {
  if (n == 0) return DEMON_OK;
  const auto axis = [resample](int in, int out) {
    if (resample == DEMON_RESAMPLE_NEAREST) return (int)kAxisNearest;
    if (in == out) return (int)kAxisCopy;
    return resample == DEMON_RESAMPLE_BILINEAR ? (int)kAxisTriangle : (int)kAxisCubic;
  };
  const long dn = (long)oh * ow * 3;
  const bool convolve = resample != DEMON_RESAMPLE_NEAREST && w != ow && h != oh;
  if (convolve && h > 100L * w && oh < h)   // vertical pass first: the transposed image, horizontal pass first
    (void)launch_pdl(resize_u8_kernel, dim3(ceil_div(oh, kTX), ceil_div(ow, kTY), n), dim3(kThreads), 0, stream, src, (long)s_outer,
                     (long)s_inner, per, 3L, (long)sy, w, h, dst, dn, 3L, (long)ow * 3, ow, oh, axis(h, oh), axis(w, ow));
  else
    (void)launch_pdl(resize_u8_kernel, dim3(ceil_div(ow, kTX), ceil_div(oh, kTY), n), dim3(kThreads), 0, stream, src, (long)s_outer,
                     (long)s_inner, per, (long)sy, 3L, h, w, dst, dn, (long)ow * 3, 3L, oh, ow, axis(w, ow), axis(h, oh));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace demon

using namespace demon;

extern "C" {

int demon_resize_u8(const uint8_t* src, int64_t src_sn, int64_t src_sy, int n, int h, int w, uint8_t* dst, int oh, int ow, int resample,
                    void* stream) {
  DEMON_REQUIRE(src && dst, "resize_u8: null pointer");
  DEMON_REQUIRE(n >= 0 && n <= 65535, "resize_u8: n %d outside 0..65535", n);
  DEMON_REQUIRE(src_sn >= 0 && src_sy >= 0, "resize_u8: negative stride");
  int rc = resize_u8_check(h, w, oh, ow, resample, "resize_u8");
  if (rc) return rc;
  return resize_u8_launch(src, src_sn, 0, 1, src_sy, n, h, w, dst, oh, ow, resample, (cudaStream_t)stream);
}

}  // extern "C"
