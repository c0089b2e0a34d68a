// Resize of RGB uint8 images, bit for bit what Pillow's `Image.resize` returns for NEAREST, BILINEAR and BICUBIC
// (examples/example.py:15-22 resizes every input with it), and the windowed form behind adjust_intrinsics
// (dataset_tools/view_tools.py:97-172): resize with BILINEAR or LANCZOS, then crop with fill, in one pass.
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
//
// Windowed (IntrinsicsWindow): image z gets its own resize rw x rh, filter and window offset (x0, y0), computed by every
// thread from the image's intrinsics (window_of).  Output pixel (u, v) is resized pixel (x0 + u, y0 + v) when that lies in
// [0, rw) x [0, rh) and kFill otherwise.  A resized byte depends only on its own coordinates, so computing the window
// alone equals "resize all, then crop".  Only this instantiation compiles the LANCZOS branch:
//   lanczos(x) = (-3 <= x < 3) ? sinc(x) sinc(x / 3) : 0, sinc(x) = x == 0 ? 1 : sin(x pi) / (x pi), support 3,
// in Pillow's order of operations (Resample.c).  CUDA's double sin is within 2 ulp of the exact value rather than
// correctly rounded; tests/test_intrinsics.py shows that no quantised weight of the tested sizes can change by that.
#include "images.cuh"

#include <cmath>

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
enum AxisFilter { kAxisNearest = 0, kAxisCopy = 1, kAxisTriangle = 2, kAxisCubic = 3, kAxisLanczos = 4 };

__device__ __forceinline__ double sinc(double x) {
  if (x == 0.0) return 1.0;
  x = fmul(x, M_PI);
  return fdiv(sin(x), x);
}

template <bool kLanczos>
__device__ __forceinline__ double filter_value(int f, double x) {
  if (kLanczos && f == kAxisLanczos) return (-3.0 <= x && x < 3.0) ? fmul(sinc(x), sinc(fdiv(x, 3.0))) : 0.0;
  x = fabs(x);
  if (f == kAxisTriangle) return x < 1.0 ? fsub(1.0, x) : 0.0;
  if (x < 1.0) return fadd(fmul(fmul(fsub(fmul(1.5, x), 2.5), x), x), 1.0);         // ((a + 2) x - (a + 3)) x x + 1
  if (x < 2.0) return fmul(fsub(fmul(fadd(fmul(fsub(x, 5.0), x), 8.0), x), 4.0), -0.5);   // (((x - 5) x + 8) x - 4) a
  return 0.0;
}

struct AxisScale { double scale, support, ss; };

template <bool kLanczos>
__device__ __forceinline__ AxisScale axis_scale(int f, int in, int out) {
  AxisScale a;
  a.scale = fdiv((double)in, (double)out);
  const double fs = fmax(a.scale, 1.0);
  a.support = fmul(f == kAxisTriangle ? 1.0 : (kLanczos && f == kAxisLanczos ? 3.0 : 2.0), fs);
  a.ss = fdiv(1.0, fs);
  return a;
}

// unnormalised weight of input sample `src` for an output sample centred at `center`
template <bool kLanczos>
__device__ __forceinline__ double raw_weight(int f, int src, double center, double ss) {
  return filter_value<kLanczos>(f, fmul(fadd(fsub((double)src, center), 0.5), ss));
}

// fixed-point weight of input sample `src`; ww: the sum of the output sample's raw weights
template <bool kLanczos>
__device__ __forceinline__ int tap_weight(int f, int src, double center, double ww, double ss) {
  if (f == kAxisNearest || f == kAxisCopy) return kOne;
  double w = raw_weight<kLanczos>(f, src, center, ss);
  if (ww != 0.0) w = fdiv(w, ww);
  const double k = fmul(w, (double)kOne);
  return (int)(w < 0.0 ? fsub(k, 0.5) : fadd(k, 0.5));
}

// The taps of output samples [i0, i0 + count) of one axis (count <= 32), computed by one warp: lo, cnt and, for the
// convolution filters, the center and the weight sum.  Samples past `out` (windowed: or before 0) get cnt = 0.
template <bool kWindowed>
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
  if ((kWindowed && i < 0) || i >= out) { lo[lane] = 0; cnt[lane] = 0; center[lane] = 0.0; ww[lane] = 0.0; return; }
  if (f == kAxisCopy) { lo[lane] = i; cnt[lane] = 1; center[lane] = 0.0; ww[lane] = 0.0; return; }
  const AxisScale a = axis_scale<kWindowed>(f, in, out);
  const double c = fmul(fadd((double)i, 0.5), a.scale);
  const int l = max((int)fadd(fsub(c, a.support), 0.5), 0);
  const int h = min((int)fadd(fadd(c, a.support), 0.5), in);
  double s = 0.0;
  for (int j = l; j < h; ++j) s = fadd(s, raw_weight<kWindowed>(f, j, c, a.ss));
  lo[lane] = l; cnt[lane] = h - l; center[lane] = c; ww[lane] = s;
}

__device__ __forceinline__ unsigned char clip8(int v) { return (unsigned char)min(max(v >> 22, 0), 255); }

// The plain resize: every image of the batch is resized to oh x ow with the filters of the launch.
struct FullImage {
  static constexpr bool kWindowed = false;
};

// adjust_intrinsics: image z, with intrinsics K[z] = (fx, fy, cx, cy) in pixels, is resized and cropped so that it has the
// target intrinsics (fx, fy, cx, cy) and size ow x oh; status[z] = 0 (ok), 1 (fill was added), 2 (invalid: all fill).
struct IntrinsicsWindow {
  static constexpr bool kWindowed = true;
  const double* K;
  double fx, fy, cx, cy;
  unsigned char* status;
};

struct Window { int rw, rh, x0, y0, fx, fy, status; };

// The reference's arithmetic in IEEE operations: scale = f_new / f, rw = trunc(w * scale_x) (Python's int()),
// x0 = rint(cx * scale_x - cx_new) (Python 3's round(): half to even), BILINEAR if scale_x > 1 else LANCZOS on both axes.
// Invalid (all fill, status 2): a focal length not finite and positive, a principal point not finite, rw or rh outside
// 1..8192 or an offset beyond +-2^24.  rw = rh = 0 then, so that no tap reads the source.
__device__ Window window_of(const IntrinsicsWindow& win, int z, int h, int w, int oh, int ow) {
  const double* k = win.K + 4L * z;
  const double fx = k[0], fy = k[1], cx = k[2], cy = k[3];
  const double scale_x = fdiv(win.fx, fx), scale_y = fdiv(win.fy, fy);
  const double rw = fmul((double)w, scale_x), rh = fmul((double)h, scale_y);
  const double x0 = rint(fsub(fmul(cx, scale_x), win.cx)), y0 = rint(fsub(fmul(cy, scale_y), win.cy));
  const double kMaxOffset = 16777216.0;
  Window d = {0, 0, 0, 0, kAxisCopy, kAxisCopy, 2};
  if (!(isfinite(fx) && fx > 0.0 && isfinite(fy) && fy > 0.0 && isfinite(cx) && isfinite(cy) && rw >= 1.0 && rw < kMaxSide + 1.0 &&
        rh >= 1.0 && rh < kMaxSide + 1.0 && fabs(x0) <= kMaxOffset && fabs(y0) <= kMaxOffset))
    return d;
  d.rw = (int)rw; d.rh = (int)rh; d.x0 = (int)x0; d.y0 = (int)y0;
  const int f = scale_x > 1.0 ? kAxisTriangle : kAxisLanczos;
  d.fx = d.rw == w ? kAxisCopy : f;
  d.fy = d.rh == h ? kAxisCopy : f;
  d.status = (d.x0 < 0 || d.y0 < 0 || d.x0 + ow > d.rw || d.y0 + oh > d.rh) ? 1 : 0;
  return d;
}

constexpr unsigned char kFill = 127;

// grid (ceil(ow / kTX), ceil(oh / kTY), n); fx / fy: AxisFilter of the first (horizontal) / second (vertical) pass.
// sy / sx: source bytes between rows / pixels; dn / dy / dx: output bytes between images / rows / pixels.
// Win = IntrinsicsWindow: oh x ow is the window, and fx / fy are replaced by each image's own (window_of).
template <class Win>
__global__ void __launch_bounds__(kThreads) resize_u8_kernel(const unsigned char* __restrict__ src, long s_outer, long s_inner, int per,
                                                             long sy, long sx, int h, int w, unsigned char* __restrict__ dst, long dn,
                                                             long dy, long dx, int oh, int ow, int fx, int fy, Win win) {
  constexpr bool kWin = Win::kWindowed;
  __shared__ int x_lo[kTX], x_cnt[kTX], y_lo[kTY], y_cnt[kTY];
  __shared__ double x_center[kTX], x_ww[kTX], y_center[kTY], y_ww[kTY];
  __shared__ int hk[kTX][kTaps + 1];                   // horizontal weights of one tap chunk (+1: lanes read one column each)
  __shared__ int vk[kTY][kRows];                       // vertical weights of the current row chunk
  __shared__ unsigned char rows[kRows][kTX * 3];       // horizontal pass of the current row chunk
  __shared__ unsigned char row_used[kRows];

  pdl_launch_dependents();   // common.cuh: programmatic dependent launch
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int z = blockIdx.z;
  const unsigned char* img = src + (long)(z / per) * s_outer + (long)(z % per) * s_inner;
  int rw = ow, rh = oh, wx = 0, wy = 0;   // size of the resized image and offset of the output in it
  if constexpr (kWin) {
    pdl_wait();   // K may have been written by the kernel before
    const Window d = window_of(win, z, h, w, oh, ow);
    rw = d.rw; rh = d.rh; wx = d.x0; wy = d.y0; fx = d.fx; fy = d.fy;
    if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) win.status[z] = (unsigned char)d.status;
  }
  const int x0 = blockIdx.x * kTX + wx, y0 = blockIdx.y * kTY + wy;
  if (warp == 0) axis_setup<kWin>(fx, w, rw, x0, kTX, lane, x_lo, x_cnt, x_center, x_ww);
  if (warp == 1) axis_setup<kWin>(fy, h, rh, y0, kTY, lane, y_lo, y_cnt, y_center, y_ww);
  if constexpr (!kWin) pdl_wait();
  __syncthreads();

  const double ssx = (fx >= kAxisTriangle) ? axis_scale<kWin>(fx, w, rw).ss : 0.0;
  const double ssy = (fy >= kAxisTriangle) ? axis_scale<kWin>(fy, h, rh).ss : 0.0;
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
      hk[c][j] = (j0 + j < x_cnt[c]) ? tap_weight<kWin>(fx, x_lo[c] + j0 + j, x_center[c], x_ww[c], ssx) : 0;
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
      vk[y][i] = in_support ? tap_weight<kWin>(fy, r, y_center[y], y_ww[y], ssy) : 0;
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
  if constexpr (kWin) {
    const int u = x - wx, v = y - wy;   // output pixel
    if (u < ow && v < oh) {
      const bool inside = x >= 0 && x < rw && y >= 0 && y < rh;
      unsigned char* o = dst + z * dn + v * dy + u * dx;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = inside ? clip8(acc[c]) : kFill;
    }
  } else {
    if (x < ow && y < oh) {
      unsigned char* o = dst + z * dn + y * dy + x * dx;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = clip8(acc[c]);
    }
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
    (void)launch_pdl(resize_u8_kernel<FullImage>, dim3(ceil_div(oh, kTX), ceil_div(ow, kTY), n), dim3(kThreads), 0, stream, src, (long)s_outer,
                     (long)s_inner, per, 3L, (long)sy, w, h, dst, dn, 3L, (long)ow * 3, ow, oh, axis(h, oh), axis(w, ow), FullImage{});
  else
    (void)launch_pdl(resize_u8_kernel<FullImage>, dim3(ceil_div(ow, kTX), ceil_div(oh, kTY), n), dim3(kThreads), 0, stream, src, (long)s_outer,
                     (long)s_inner, per, (long)sy, 3L, h, w, dst, dn, (long)ow * 3, 3L, oh, ow, axis(w, ow), axis(h, oh), FullImage{});
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int adjust_intrinsics_check(int h, int w, const double* knew, int oh, int ow, const char* who) {
  DEMON_REQUIRE(h >= 1 && w >= 1 && h <= kMaxSide && w <= kMaxSide, "%s: source size %dx%d (width x height) outside 1..%d", who, w, h,
                kMaxSide);
  // Pillow runs the vertical pass first for such sources (see resize_u8_launch); the window has no transposed form
  DEMON_REQUIRE(h <= 100L * w, "%s: source %dx%d (width x height) is more than 100 times taller than wide", who, w, h);
  DEMON_REQUIRE(oh >= 1 && ow >= 1 && oh <= kMaxSide && ow <= kMaxSide, "%s: output size %dx%d (width x height) outside 1..%d", who, ow,
                oh, kMaxSide);
  DEMON_REQUIRE(std::isfinite(knew[0]) && knew[0] > 0.0 && std::isfinite(knew[1]) && knew[1] > 0.0,
                "%s: target focal lengths %g, %g must be finite and positive", who, knew[0], knew[1]);
  DEMON_REQUIRE(std::isfinite(knew[2]) && std::isfinite(knew[3]), "%s: target principal point %g, %g must be finite", who, knew[2],
                knew[3]);
  return DEMON_OK;
}

int adjust_intrinsics_launch(const uint8_t* src, int64_t s_outer, int64_t s_inner, int per, int64_t sy, int n, int h, int w, const double* K,
                             const double* knew, uint8_t* dst, int oh, int ow, uint8_t* status, cudaStream_t stream) {
  if (n == 0) return DEMON_OK;
  const IntrinsicsWindow win = {K, knew[0], knew[1], knew[2], knew[3], status};
  (void)launch_pdl(resize_u8_kernel<IntrinsicsWindow>, dim3(ceil_div(ow, kTX), ceil_div(oh, kTY), n), dim3(kThreads), 0, stream, src,
                   (long)s_outer, (long)s_inner, per, (long)sy, 3L, h, w, dst, (long)oh * ow * 3, (long)ow * 3, 3L, oh, ow, 0, 0, win);
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

int demon_adjust_intrinsics_u8(const uint8_t* src, int64_t src_sn, int64_t src_sy, int n, int h, int w, const double* K, double fx_new,
                               double fy_new, double cx_new, double cy_new, uint8_t* dst, int oh, int ow, uint8_t* status, void* stream) {
  DEMON_REQUIRE(src && K && dst && status, "adjust_intrinsics_u8: null pointer");
  DEMON_REQUIRE(n >= 0 && n <= 65535, "adjust_intrinsics_u8: n %d outside 0..65535", n);
  DEMON_REQUIRE(src_sn >= 0 && src_sy >= 0, "adjust_intrinsics_u8: negative stride");
  const double knew[4] = {fx_new, fy_new, cx_new, cy_new};
  int rc = adjust_intrinsics_check(h, w, knew, oh, ow, "adjust_intrinsics_u8");
  if (rc) return rc;
  return adjust_intrinsics_launch(src, src_sn, 0, 1, src_sy, n, h, w, K, knew, dst, oh, ow, status, (cudaStream_t)stream);
}

}  // extern "C"
