// The per-pixel compute of the reference's multi-view training reader (multivih5datareaderop/multivih5datareader.cpp) on
// the device; demon_b200/datareader.py drives it and does the per-item pose math on the host.
//
// * prepare_kernel: prepareScene (:1384-1520) for a table of views of any source size: INTER_AREA downscaling of the uint8
//   image by the path OpenCV's cv::resize takes for the view (the 2x2 vector path, the other integer factors, or the
//   general float-weighted path), half -> float depth, INTER_NEAREST scaling of the depth and ray length -> camera z with
//   the scaled float K.  One thread per output pixel, blockIdx.y = view.  Both resizes are bit for bit OpenCV 4.13.0's
//   (tests/golden/datareader_resize_digests.json).
// * batch_kernel: the batch loop (:1585-1950) for every item of a batch in one launch.  Each output pixel is remapped
//   through the item's rot180 / mirror_x to the pixel of the prepared pool it comes from; IMAGE_PAIR (:344-363 and
//   augmentImage :641-714), DEPTH (:1857-1908), FLOW (computeFlow :370-424 on the unrotated cameras, then negated) and
//   DEPTHMASKS (computeDepthmask :431-498) are all written from there.  There is no separate flip pass.
//
// The reference is x86 code built without FMA; arithmetic goes through common.cuh's round-to-nearest helpers, and the few
// places where x86 and CUDA differ on NaN or on out-of-range conversions are restated explicitly (DESIGN.md section 3.8).
#include "common.cuh"
#include "geometry.cuh"
#include <cfloat>
#include <cstdint>

namespace demon {
namespace {

constexpr int kThreads = 256;
constexpr uint32_t kNaN = 0x7fc00000u;          // the C macro NAN
constexpr uint32_t kDefaultNaN = 0xffc00000u;   // what an x86 SSE operation returns for an invalid operation (0/0, inf-inf)

// a NaN operand of an x86 SSE arithmetic operation comes out of it quieted, sign and payload kept
__device__ __forceinline__ float quiet(float x) { return __int_as_float(__float_as_int(x) | 0x00400000); }
__device__ __forceinline__ float neg_bits(float x) { return __int_as_float(__float_as_int(x) ^ 0x80000000); }

// ---- prepareScene ----------------------------------------------------------------------------------------------------
// IEEE half -> float, exact; a NaN keeps its sign and payload (shifted into the float's mantissa)
__device__ __forceinline__ float half_bits_to_float(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
  if (e == 0x1fu) return __uint_as_float(sign | 0x7f800000u | (m << 13));
  if (e == 0) {
    if (m == 0) return __uint_as_float(sign);
    e = 1;
    while (!(m & 0x400u)) { m <<= 1; --e; }
    m &= 0x3ffu;
  }
  return __uint_as_float(sign | ((e + 112u) << 23) | (m << 13));
}

// cv::resize(INTER_AREA) of uint8 images, downscaling only (imgproc/src/resize.cpp).  An axis of n -> m cells has the scale
// 1 / (m / (double)n); it is integral when |scale - cvRound(scale)| < DBL_EPSILON, and for sides up to 8192 that implies
// n = scale * m (the converse fails: 98 -> 2 has the scale 49.00000000000001).  Returns the integer factor, or 0.
__device__ __forceinline__ int area_factor(double scale) {
  const int k = __double2int_rn(scale);
  return fabs(fsub(scale, (double)k)) < DBL_EPSILON ? k : 0;
}

// computeResizeAreaTab's entries of output index d: source cells lo..hi, consecutive, with the weight `lead` on cell lo if
// `has_lead` (the leading partial cell), `trail` on cell hi if `has_trail` (the trailing one) and `full` on the others.
// Each weight is computed in double and cast to float, as the table stores it.
struct AreaCells {
  int lo, hi;
  bool has_lead, has_trail;
  float lead, full, trail;
  __device__ __forceinline__ float weight(int i) const { return (has_lead && i == lo) ? lead : (has_trail && i == hi) ? trail : full; }
};

__device__ __forceinline__ AreaCells area_cells(int d, int n, double scale) {
  const double fs1 = fmul((double)d, scale), fs2 = fadd(fs1, scale);
  const double cell = fmin(scale, fsub((double)n, fs1));
  const int s2 = min((int)floor(fs2), n - 1);
  const int s1 = min((int)ceil(fs1), s2);
  AreaCells c;
  c.has_lead = fsub((double)s1, fs1) > 1e-3;   // a sliver of at most 1e-3 of a cell gets no entry
  c.has_trail = fsub(fs2, (double)s2) > 1e-3;
  c.lo = c.has_lead ? s1 - 1 : s1;
  c.hi = c.has_trail ? s2 : s2 - 1;
  c.lead = __double2float_rn(fdiv(fsub((double)s1, fs1), cell));
  c.full = __double2float_rn(fdiv(1.0, cell));
  c.trail = __double2float_rn(fdiv(fmin(fmin(fsub(fs2, (double)s2), 1.0), cell), cell));
  return c;
}

// Output pixel (x, y) of INTER_AREA, per channel, by the path OpenCV takes for the view (both axes integral or not):
//   2x2          (a + b + c + d + 2) >> 2, ties up (ResizeAreaFastVec);
//   other k x l  float(int block sum) * (1.f / (k * l)), cvRound: ties to even (resizeAreaFast_);
//   otherwise    ResizeArea_Invoker: per source row, buf = buf + S * alpha over the x cells in order, in float; then
//                sum = beta * buf for the first row, sum = sum + beta * buf for the rest; cvRound.
__device__ __forceinline__ void area_pixel(const uint8_t* __restrict__ img, int sh, int sw, int x, int y, double scale_x,
                                           double scale_y, uint8_t out[3]) {
  const int kx = area_factor(scale_x), ky = area_factor(scale_y);
  if (kx && ky) {
    unsigned acc[3] = {0, 0, 0};   // OpenCV's block sum is an int, which wraps (two's complement) above 2^31 - 1
    for (int sy = y * ky; sy < (y + 1) * ky; ++sy) {
      const uint8_t* q = img + ((long)sy * sw + (long)x * kx) * 3;
      for (int i = 0; i < kx * 3; i += 3)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += __ldg(q + i + c);
    }
    const float inv_area = fdiv(1.0f, (float)(kx * ky));   // 1.f / area: an area above 2^24 is rounded to float first
#pragma unroll
    for (int c = 0; c < 3; ++c)
      out[c] = (kx == 2 && ky == 2) ? (uint8_t)((acc[c] + 2) >> 2) : (uint8_t)min(max(__float2int_rn(fmul((float)(int)acc[c], inv_area)), 0), 255);
    return;
  }
  const AreaCells cx = area_cells(x, sw, scale_x), cy = area_cells(y, sh, scale_y);
  float sum[3] = {0.0f, 0.0f, 0.0f};
  for (int sy = cy.lo; sy <= cy.hi; ++sy) {
    const uint8_t* row = img + (long)sy * sw * 3;
    float buf[3] = {0.0f, 0.0f, 0.0f};
    for (int sx = cx.lo; sx <= cx.hi; ++sx) {
      const float alpha = cx.weight(sx);
#pragma unroll
      for (int c = 0; c < 3; ++c) buf[c] = fadd(buf[c], fmul((float)__ldg(row + sx * 3 + c), alpha));
    }
    const float beta = cy.weight(sy);
#pragma unroll
    for (int c = 0; c < 3; ++c) sum[c] = sy == cy.lo ? fmul(beta, buf[c]) : fadd(sum[c], fmul(beta, buf[c]));
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = (uint8_t)min(max(__float2int_rn(sum[c]), 0), 255);
}

__global__ void __launch_bounds__(kThreads) prepare_kernel(const uint8_t* __restrict__ staging, const demon_datareader_view* __restrict__ views,
                                                           int h, int w, uint8_t* __restrict__ pool_image, float* __restrict__ pool_depth) {
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= h * w) return;
  const demon_datareader_view v = views[blockIdx.y];
  const int x = p % w, y = p / w;
  const int sw = v.width, sh = v.height;
  // cv::resize's scale of each axis, 1 / inv_scale with inv_scale = dsize / (double)ssize: both calls use it
  const double ifx = fdiv(1.0, fdiv((double)w, (double)sw)), ify = fdiv(1.0, fdiv((double)h, (double)sh));

  uint8_t rgb[3];
  area_pixel(staging + v.image_offset, sh, sw, x, y, ifx, ify, rgb);
  uint8_t* out = pool_image + ((long)v.pool_index * h * w + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = rgb[c];

  // cv::resize(INTER_NEAREST): sx = cvFloor(x * ifx), clamped
  const int sx = min((int)floor(fmul((double)x, ifx)), sw - 1), sy = min((int)floor(fmul((double)y, ify)), sh - 1);
  const long si = (long)sy * sw + sx;
  float d = v.depth_f16 ? half_bits_to_float(__ldg(reinterpret_cast<const uint16_t*>(staging + v.depth_offset) + si))
                        : __ldg(reinterpret_cast<const float*>(staging + v.depth_offset) + si);
  if (v.ray_length) {   // :1489-1511, K of the normalised intrinsics cast to float and scaled by the scaled size
    const D2NCamera<float> ik = eigen_inverse_k(fmul(v.k[0], (float)w), v.k[1], fmul(v.k[3], (float)h), fmul(v.k[2], (float)w),
                                                fmul(v.k[4], (float)h));
    const float px = fadd(fmul(ik.i00, fadd((float)x, 0.5f)), ik.i02);
    const float py = fadd(fmul(ik.i11, fadd((float)y, 0.5f)), ik.i12);
    const float norm = sqrtf(fadd(fadd(fmul(px, px), fmul(py, py)), fmul(1.0f, 1.0f)));
    d = isnan(d) ? quiet(d) : fdiv(d, norm);
  }
  pool_depth[(long)v.pool_index * h * w + p] = d;
}

// ---- augmentImage ----------------------------------------------------------------------------------------------------
// std::min / std::max as the reference calls them: min(a, b) = b < a ? b : a, max(a, b) = a < b ? b : a
__device__ __forceinline__ float saturate(float v) {
  const float m = (v < 1.0f) ? v : 1.0f;
  return (0.0f < m) ? m : 0.0f;
}

// fast_powf (:633-638): u.x = (int)(b * (float)(u.x - 1064866805) + (float)1064866805).  The subtraction overflows int for
// negative a (undefined behaviour in C++); x86 wraps it, and cvttss2si turns an out-of-range float into INT_MIN.
__device__ __forceinline__ float fast_powf(float a, float b) {
  const int d = (int)((unsigned)__float_as_int(a) - 1064866805u);
  const float f = fadd(fmul(b, __int2float_rn(d)), __int2float_rn(1064866805));
  return __int_as_float(cvtt_x86(f));
}

__device__ __forceinline__ void augment(float layer[3], const float aug[6]) {
  // rgb[0] is layer 2 (:684-686); the +-0.5 offsets are fixed whatever the image range
  float r = fadd(layer[2], 0.5f), g = fadd(layer[1], 0.5f), b = fadd(layer[0], 0.5f);
  // rgb2hsv (:547-559)
  const float gb_min = (b < g) ? b : g, gb_max = (g < b) ? b : g;
  const float mn = (gb_min < r) ? gb_min : r;
  const float v0 = (r < gb_max) ? gb_max : r;
  const float den = fadd(fsub(v0, mn), 1e-6f);
  float h;
  if (r == v0) h = fdiv(fmul(60.0f, fsub(g, b)), den);
  else if (g == v0) h = fadd(120.0f, fdiv(fmul(60.0f, fsub(r, g)), den));
  else h = fadd(240.0f, fdiv(fmul(60.0f, fsub(r, g)), den));
  float s = fdiv(fsub(v0, mn), fadd(v0, 1e-6f));
  float v = v0;
  h = fadd(h, aug[0]);
  while (h < 0) h = fadd(h, 360.f);
  while (h >= 360) h = fsub(h, 360.f);
  s = saturate(fadd(s, aug[1]));
  v = saturate(fadd(v, aug[2]));
  // hsv2rgb (:561-612)
  if (s == 0) {
    r = g = b = v;
  } else {
    const float hh = fdiv(h, 60.0f);
    const int i = (int)floorf(hh);
    const float f = fsub(hh, (float)i);
    const float p = fmul(v, fsub(1.0f, s));
    const float q = fmul(v, fsub(1.0f, fmul(s, f)));
    const float t = fmul(v, fsub(1.0f, fmul(s, fsub(1.0f, f))));
    switch (i) {
      case 0: r = v; g = t; b = p; break;
      case 1: r = q; g = v; b = p; break;
      case 2: r = p; g = v; b = t; break;
      case 3: r = p; g = q; b = v; break;
      case 4: r = t; g = p; b = v; break;
      default: r = v; g = p; b = q; break;
    }
  }
  float rgb[3] = {r, g, b};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float value = fadd(fadd(fmul(fsub(rgb[c], 0.5f), aug[3]), aug[4]), 0.5f);
    value = fast_powf(value, aug[5]);
    rgb[c] = saturate(value);
  }
  layer[2] = fsub(rgb[0], 0.5f);
  layer[1] = fsub(rgb[1], 0.5f);
  layer[0] = fsub(rgb[2], 0.5f);
}

// ---- computeFlow / computeDepthmask ------------------------------------------------------------------------------------
// cam = [fx, skew, cx, fy, cy] (normalised, the skew in pixels), R row-major [9], t [3], as float casts of the doubles
struct Projection {
  D2NCamera<float> ik;   // inverse of cam1's scaled K
  float inv_r[9];        // cam1.R^T
  float t[3];            // cam1.t
  float P[12];           // cam2's K2 * [R2 | t2], row-major
};

__device__ __forceinline__ Projection make_projection(const float* c1, const float* c2, int h, int w) {
  Projection pr;
  pr.ik = eigen_inverse_k(fmul(c1[0], (float)w), c1[1], fmul(c1[3], (float)h), fmul(c1[2], (float)w), fmul(c1[4], (float)h));
  const float* r1 = c1 + 5;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) pr.inv_r[i * 3 + k] = r1[k * 3 + i];
  pr.t[0] = c1[14]; pr.t[1] = c1[15]; pr.t[2] = c1[16];
  const float K[9] = {fmul(c2[0], (float)w), c2[1], fmul(c2[2], (float)w), 0.0f, fmul(c2[3], (float)h), fmul(c2[4], (float)h), 0.0f, 0.0f, 1.0f};
  const float* r2 = c2 + 5;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float m0 = j < 3 ? r2[0 * 3 + j] : c2[14], m1 = j < 3 ? r2[1 * 3 + j] : c2[15], m2 = j < 3 ? r2[2 * 3 + j] : c2[16];
      pr.P[i * 4 + j] = fadd(fadd(fmul(K[i * 3 + 0], m0), fmul(K[i * 3 + 1], m1)), fmul(K[i * 3 + 2], m2));
    }
  return pr;
}

// p2 of pixel (x, y) at camera-z depth d > 0 (:394-418; the prepared depth is camera z, so depth/norm is depth/1)
__device__ __forceinline__ void project(const Projection& pr, int x, int y, float d, float& p1x, float& p1y, float& p2x, float& p2y) {
  p1x = fadd((float)x, 0.5f);
  p1y = fadd((float)y, 0.5f);
  const float s = fdiv(d, 1.0f);
  float pos[3] = {fmul(fadd(fmul(pr.ik.i00, p1x), pr.ik.i02), s), fmul(fadd(fmul(pr.ik.i11, p1y), pr.ik.i12), s), fmul(1.0f, s)};
#pragma unroll
  for (int i = 0; i < 3; ++i) pos[i] = fsub(pos[i], pr.t[i]);
  float q[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) q[i] = fadd(fadd(fmul(pr.inv_r[i * 3], pos[0]), fmul(pr.inv_r[i * 3 + 1], pos[1])), fmul(pr.inv_r[i * 3 + 2], pos[2]));
  float p2[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    p2[i] = fadd(fadd(fadd(fmul(pr.P[i * 4], q[0]), fmul(pr.P[i * 4 + 1], q[1])), fmul(pr.P[i * 4 + 2], q[2])), fmul(pr.P[i * 4 + 3], 1.0f));
  p2x = fdiv(p2[0], p2[2]);
  p2y = fdiv(p2[1], p2[2]);
}

__device__ __forceinline__ bool bad_depth(float d) { return d <= 0 || !isfinite(d); }

__device__ __forceinline__ float depthmask(const Projection& pr, int x, int y, float d, int h, int w, int border1, int border2) {
  if (x < border1 || y < border1 || x >= w - border1 || y >= h - border1) return 0.0f;
  if (bad_depth(d)) return 0.0f;
  float p1x, p1y, p2x, p2y;
  project(pr, x, y, d, p1x, p1y, p2x, p2y);
  return (p2x < (float)border2 || p2y < (float)border2 || p2x >= (float)(w - border2) || p2y >= (float)(h - border2)) ? 0.0f : 1.0f;
}

struct BatchArgs {
  const uint8_t* pool_image;
  const float* pool_depth;
  const demon_datareader_item* items;
  int h, w;
  int colour, inverse_depth, depth_pair, border1, border2;
  float range_min, range_max, min_depth, max_depth;
  float *image_pair, *flow, *depth, *depthmasks;
};

__global__ void __launch_bounds__(kThreads) batch_kernel(const BatchArgs a) {
  const int hw = a.h * a.w;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (p >= hw) return;
  const int b = blockIdx.y;
  const demon_datareader_item& it = a.items[b];
  const bool rot = it.flags & 1, mir = it.flags & 2;
  const int x = p % a.w, y = p / a.w;
  const int mx = mir ? a.w - 1 - x : x;          // mirrorImageX after rotateImageBy180 (:1636-1639)
  const int rx = rot ? a.w - 1 - mx : mx, ry = rot ? a.h - 1 - y : y;
  const long src = (long)ry * a.w + rx;
  const int views[2] = {it.view1, it.view2};

  if (a.image_pair) {
    const float scale = fdiv(fsub(a.range_max, a.range_min), 255.0f);
    for (int i = 0; i < 2; ++i) {
      const uint8_t* q = a.pool_image + ((long)views[i] * hw + src) * 3;
      float layer[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) layer[c] = fadd(fmul(scale, (float)__ldg(q + c)), a.range_min);
      if (a.colour) augment(layer, it.aug);
#pragma unroll
      for (int c = 0; c < 3; ++c) a.image_pair[((long)b * 6 + 3 * i + c) * hw + p] = layer[c];
    }
  }
  const int nd = a.depth_pair ? 2 : 1;
  if (a.depth) {
    for (int i = 0; i < nd; ++i) {
      float d = __ldg(a.pool_depth + (long)views[i] * hw + src);
      if (d == 0 || (a.max_depth > 0 && d > a.max_depth) || (a.min_depth > 0 && d < a.min_depth)) {
        d = __uint_as_float(kNaN);
      } else if (isnan(d)) {
        d = quiet(d);   // d *= depth_scale_factor and 1/d pass the NaN through
      } else {
        d = __double2float_rn(fmul((double)d, it.depth_scale_factor));
        if (a.inverse_depth) d = fdiv(1.0f, d);
      }
      a.depth[((long)b * nd + i) * hw + p] = d;
    }
  }
  if (a.flow || a.depthmasks) {
    const float d1 = __ldg(a.pool_depth + (long)views[0] * hw + src);
    const Projection pr = make_projection(it.cam[0], it.cam[1], a.h, a.w);
    if (a.flow) {
      float fx = __uint_as_float(kNaN), fy = fx;
      if (!bad_depth(d1)) {
        float p1x, p1y, p2x, p2y;
        project(pr, rx, ry, d1, p1x, p1y, p2x, p2y);
        fx = fsub(p2x, p1x);
        fy = fsub(p2y, p1y);
        if (isnan(fx)) fx = __uint_as_float(kDefaultNaN);
        if (isnan(fy)) fy = __uint_as_float(kDefaultNaN);
      }
      if (rot) { fx = neg_bits(fx); fy = neg_bits(fy); }   // :1826-1843
      if (mir) fx = neg_bits(fx);
      a.flow[((long)b * 2 + 0) * hw + p] = fx;
      a.flow[((long)b * 2 + 1) * hw + p] = fy;
    }
    if (a.depthmasks) {
      a.depthmasks[((long)b * nd) * hw + p] = depthmask(pr, rx, ry, d1, a.h, a.w, a.border1, a.border2);
      if (a.depth_pair) {
        const float d2 = __ldg(a.pool_depth + (long)views[1] * hw + src);
        const Projection pr2 = make_projection(it.cam[1], it.cam[0], a.h, a.w);
        a.depthmasks[((long)b * nd + 1) * hw + p] = depthmask(pr2, rx, ry, d2, a.h, a.w, a.border1, a.border2);
      }
    }
  }
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int demon_datareader_prepare(const uint8_t* staging, const demon_datareader_view* views, int n_views, int h, int w, uint8_t* pool_image,
                             float* pool_depth, void* stream) {
  DEMON_REQUIRE(n_views >= 0 && n_views <= 65535, "datareader_prepare: %d views (up to 65535 per call)", n_views);
  DEMON_REQUIRE(h >= 1 && w >= 1 && h <= 8192 && w <= 8192, "datareader_prepare: bad scaled size %dx%d", w, h);
  if (n_views == 0) return DEMON_OK;
  DEMON_REQUIRE(staging && views && pool_image && pool_depth, "datareader_prepare: null pointer");
  prepare_kernel<<<dim3((unsigned)ceil_div(h * w, kThreads), (unsigned)n_views), kThreads, 0, (cudaStream_t)stream>>>(
      staging, views, h, w, pool_image, pool_depth);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_datareader_batch(const uint8_t* pool_image, const float* pool_depth, int h, int w, const demon_datareader_item* items, int batch,
                           int colour, float range_min, float range_max, float min_depth, float max_depth, int inverse_depth, int depth_pair,
                           int border1, int border2, float* image_pair, float* flow, float* depth, float* depthmasks, void* stream) {
  DEMON_REQUIRE(batch >= 0 && batch <= 65535, "datareader_batch: batch %d (up to 65535)", batch);
  DEMON_REQUIRE(h >= 1 && w >= 1 && h <= 8192 && w <= 8192, "datareader_batch: bad size %dx%d", w, h);
  if (batch == 0 || !(image_pair || flow || depth || depthmasks)) return DEMON_OK;
  DEMON_REQUIRE(pool_image && pool_depth && items, "datareader_batch: null pointer");
  BatchArgs a;
  a.pool_image = pool_image; a.pool_depth = pool_depth; a.items = items; a.h = h; a.w = w;
  a.colour = colour; a.inverse_depth = inverse_depth; a.depth_pair = depth_pair; a.border1 = border1; a.border2 = border2;
  a.range_min = range_min; a.range_max = range_max; a.min_depth = min_depth; a.max_depth = max_depth;
  a.image_pair = image_pair; a.flow = flow; a.depth = depth; a.depthmasks = depthmasks;
  batch_kernel<<<dim3((unsigned)ceil_div(h * w, kThreads), (unsigned)batch), kThreads, 0, (cudaStream_t)stream>>>(a);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // extern "C"
