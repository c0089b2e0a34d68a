// FlowNet warping and resampling on the device: lmbspecialops' FlowWarp / FlowWarpGrad (flowwarp.cc, flowwarp_cuda.cu),
// FlowOutOfFrame (flow_out_of_frame.cc) and Resample (resample.cc, resample_cuda.cu), NCHW.
//
// Every element keeps the reference's operation order, written with explicit _rn intrinsics so that the bits do not
// depend on nvcc's contraction:
//   flow_warp        x2 = x + fx, y2 = y + fy; in frame (x2 >= 0, y2 >= 0, x2 < w, y2 < h): L = (int)x2, T = (int)y2,
//                    R = min(L + 1, w - 1), B = min(T + 1, h - 1), a = x2 - L, b = y2 - T and
//                    out = fma(cBR, BR, fma(cBL, BL, fma(cTL, TL, cTR TR))) with cTL = (1-a)(1-b), cTR = a(1-b),
//                    cBL = (1-a)b, cBR = ab: the contraction nvcc applies to flow_warp_kernel_smem.  Out of frame (a NaN
//                    flow included): the fill, 0 or the reference GPU kernel's NaN 0xFFE00000.  One pass: the flow is read
//                    once per pixel and the corners are gathered straight from NCHW, with no transposed copy.
//   flow_grad        the reference GPU kernel's sums over channels: temp = fma(g, TR - TL, 0), temp = fma(1 - g, BR - BL,
//                    temp), sum = fma(dout, temp, sum) with g = B - y2 for the x component, and the same over BL - TL,
//                    BR - TR with g = R - x2 for the y component; 0 out of frame.  At the clamped last row (column) g is
//                    not the derivative of the forward op (B = T there), and it is kept as the reference has it.
//   image_grad       deterministic, no float atomics: the reference CPU kernel's sum.  It starts from +0 and adds the
//                    rounded products (dout (1-a))(1-b), (dout a)(1-b), (dout (1-a))b, (dout a)b in its loop order: image,
//                    then target x, then target y, then corners TL, TR, BL, BR.  Its GPU kernel forms the same products
//                    (an atomicAdd operand is not contracted) and adds them in scheduling order.
//   flow_out_of_frame  the CPU kernel's ROUND_2_INT in double; a NaN, infinite or out-of-int-range position is out of
//                    frame, as x86's conversion to INT_MIN makes it there.
//   resample         NearestNeighborKernel / InterpolationKernel, swapped half offsets and antialias rule included; the
//                    NEAREST source pixel is clamped to the image (the reference reads outside it when fy / 2 >~ fx).
//
// image_grad: the targets (x-major, as the reference's loop visits them) are stably sorted by their source cell (T, L);
// the image element at (py, px) then merges the buckets of the cells (py, px), (py, px-1), (py-1, px), (py-1, px-1) in
// target order and adds each target's corners that land on it in corner order (the clamped edge cells give one target
// several corners on one pixel).  A flow that sends every pixel into one cell costs that cell's four pixels a pass over
// all targets each: linear, never quadratic.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cmath>

namespace demon {
namespace {

constexpr int kWarpThreads = 128;
constexpr int kWarpCh = 8;          // channels per thread of flow_warp and of the image_grad gather
constexpr int kResampleThreads = 256;

struct Cell {
  bool in;
  int L, T, R, B;
  float x2, y2, a, b;
};

__device__ __forceinline__ Cell cell_of(const float* __restrict__ flow, int n, int h, int w, int y, int x) {
  const size_t plane = (size_t)h * w;
  const float fx = __ldg(flow + (size_t)2 * n * plane + (size_t)y * w + x);
  const float fy = __ldg(flow + ((size_t)2 * n + 1) * plane + (size_t)y * w + x);
  Cell c;
  c.x2 = __fadd_rn((float)x, fx);
  c.y2 = __fadd_rn((float)y, fy);
  c.in = c.x2 >= 0.f && c.y2 >= 0.f && c.x2 < (float)w && c.y2 < (float)h;   // false for NaN
  c.L = c.in ? (int)c.x2 : 0;
  c.T = c.in ? (int)c.y2 : 0;
  c.R = min(c.L + 1, w - 1);
  c.B = min(c.T + 1, h - 1);
  c.a = __fsub_rn(c.x2, (float)c.L);
  c.b = __fsub_rn(c.y2, (float)c.T);
  return c;
}

// one thread = one pixel and kWarpCh channels
__global__ void __launch_bounds__(kWarpThreads) flow_warp_kernel(const float* __restrict__ image, const float* __restrict__ flow,
                                                                  float* __restrict__ out, int n_img, int c, int h, int w, int ncg,
                                                                  float fill) {
  const int64_t plane = (int64_t)h * w;
  const int64_t pblocks = (plane + kWarpThreads - 1) / kWarpThreads;
  int64_t b = blockIdx.x;
  const int64_t pb = b % pblocks; b /= pblocks;
  const int cg = (int)(b % ncg);
  const int n = (int)(b / ncg);
  const int64_t p = pb * kWarpThreads + threadIdx.x;
  if (p >= plane || n >= n_img) return;
  const int y = (int)(p / w), x = (int)(p % w);
  const Cell q = cell_of(flow, n, h, w, y, x);
  const float a1 = __fsub_rn(1.f, q.a), b1 = __fsub_rn(1.f, q.b);
  const float cTL = __fmul_rn(a1, b1), cTR = __fmul_rn(q.a, b1), cBL = __fmul_rn(a1, q.b), cBR = __fmul_rn(q.a, q.b);
  const int64_t oTL = (int64_t)q.T * w + q.L, oTR = (int64_t)q.T * w + q.R, oBL = (int64_t)q.B * w + q.L, oBR = (int64_t)q.B * w + q.R;
  const int c0 = cg * kWarpCh, c1 = min(c, c0 + kWarpCh);
  for (int ch = c0; ch < c1; ++ch) {
    const float* src = image + ((int64_t)n * c + ch) * plane;
    float v = fill;
    if (q.in) {
      v = __fmul_rn(cTR, __ldg(src + oTR));
      v = __fmaf_rn(cTL, __ldg(src + oTL), v);
      v = __fmaf_rn(cBL, __ldg(src + oBL), v);
      v = __fmaf_rn(cBR, __ldg(src + oBR), v);
    }
    out[((int64_t)n * c + ch) * plane + p] = v;
  }
}

// one thread = one pixel, both flow components, all channels in order
__global__ void __launch_bounds__(kWarpThreads) flow_warp_flow_grad_kernel(const float* __restrict__ image, const float* __restrict__ flow,
                                                                            const float* __restrict__ dout, float* __restrict__ flow_grad,
                                                                            int n_img, int c, int h, int w) {
  const int64_t plane = (int64_t)h * w;
  const int64_t i = (int64_t)blockIdx.x * kWarpThreads + threadIdx.x;
  if (i >= (int64_t)n_img * plane) return;
  const int n = (int)(i / plane);
  const int64_t p = i % plane;
  const int y = (int)(p / w), x = (int)(p % w);
  const Cell q = cell_of(flow, n, h, w, y, x);
  float sx = 0.f, sy = 0.f;
  if (q.in) {
    const float gy = __fsub_rn((float)q.B, q.y2), gy1 = __fsub_rn(1.f, gy);
    const float gx = __fsub_rn((float)q.R, q.x2), gx1 = __fsub_rn(1.f, gx);
    const int64_t oTL = (int64_t)q.T * w + q.L, oTR = (int64_t)q.T * w + q.R, oBL = (int64_t)q.B * w + q.L, oBR = (int64_t)q.B * w + q.R;
#pragma unroll 4
    for (int ch = 0; ch < c; ++ch) {
      const float* src = image + ((int64_t)n * c + ch) * plane;
      const float TL = __ldg(src + oTL), TR = __ldg(src + oTR), BL = __ldg(src + oBL), BR = __ldg(src + oBR);
      const float g = __ldg(dout + ((int64_t)n * c + ch) * plane + p);
      float t = __fmaf_rn(gy, __fsub_rn(TR, TL), 0.f);
      t = __fmaf_rn(gy1, __fsub_rn(BR, BL), t);
      sx = __fmaf_rn(g, t, sx);
      t = __fmaf_rn(gx, __fsub_rn(BL, TL), 0.f);
      t = __fmaf_rn(gx1, __fsub_rn(BR, TR), t);
      sy = __fmaf_rn(g, t, sy);
    }
  }
  flow_grad[(int64_t)2 * n * plane + p] = sx;
  flow_grad[((int64_t)2 * n + 1) * plane + p] = sy;
}

// targets in x-major order i = (n w + x) h + y -> (source cell key, i); clears the bucket bounds
__global__ void __launch_bounds__(kWarpThreads) flow_warp_cells_kernel(const float* __restrict__ flow, uint32_t* __restrict__ keys,
                                                                        uint32_t* __restrict__ vals, uint32_t* __restrict__ start,
                                                                        uint32_t* __restrict__ end, int n_img, int h, int w) {
  const uint32_t total = (uint32_t)n_img * h * w;
  const uint32_t i = blockIdx.x * kWarpThreads + threadIdx.x;
  if (i >= total) return;
  const int y = (int)(i % h);
  const uint32_t nx = i / h;
  const int x = (int)(nx % w), n = (int)(nx / w);
  const Cell q = cell_of(flow, n, h, w, y, x);
  keys[i] = q.in ? ((uint32_t)n * h + q.T) * w + q.L : total;   // out of frame: past every cell
  vals[i] = i;
  start[i] = 0;
  end[i] = 0;
}

__global__ void __launch_bounds__(kWarpThreads) flow_warp_bounds_kernel(const uint32_t* __restrict__ keys, uint32_t* __restrict__ start,
                                                                         uint32_t* __restrict__ end, uint32_t total) {
  const uint32_t i = blockIdx.x * kWarpThreads + threadIdx.x;
  if (i >= total) return;
  const uint32_t k = keys[i];
  if (k == total) return;
  if (i == 0 || keys[i - 1] != k) start[k] = i;
  if (i + 1 == total || keys[i + 1] != k) end[k] = i + 1;
}

// one thread = one image pixel and kWarpCh channels: merges the four neighbouring buckets in target order
__global__ void __launch_bounds__(kWarpThreads) flow_warp_image_grad_kernel(const float* __restrict__ flow, const float* __restrict__ dout,
                                                                             const uint32_t* __restrict__ order,
                                                                             const uint32_t* __restrict__ start, const uint32_t* __restrict__ end,
                                                                             float* __restrict__ image_grad, int n_img, int c, int h, int w, int ncg) {
  const int64_t plane = (int64_t)h * w;
  const int64_t pblocks = (plane + kWarpThreads - 1) / kWarpThreads;
  int64_t bb = blockIdx.x;
  const int64_t pb = bb % pblocks; bb /= pblocks;
  const int cg = (int)(bb % ncg);
  const int n = (int)(bb / ncg);
  const int64_t p = pb * kWarpThreads + threadIdx.x;
  if (p >= plane || n >= n_img) return;
  const int py = (int)(p / w), px = (int)(p % w);
  const int c0 = cg * kWarpCh, nc = min(c - c0, kWarpCh);

  // the cells whose corners can land on (py, px): TL of (py, px), TR of (py, px-1), BL of (py-1, px), BR of (py-1, px-1),
  // and at the clamped last row / column the other corners of the same cells
  uint32_t pos[4], lim[4];
  const int cy[4] = {py, py, py - 1, py - 1}, cx[4] = {px, px - 1, px, px - 1};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const bool ok = cy[k] >= 0 && cx[k] >= 0;
    const uint32_t cell = ok ? ((uint32_t)n * h + cy[k]) * w + cx[k] : 0;
    pos[k] = ok ? __ldg(start + cell) : 0;
    lim[k] = ok ? __ldg(end + cell) : 0;
  }
  float sum[kWarpCh];
#pragma unroll
  for (int k = 0; k < kWarpCh; ++k) sum[k] = 0.f;
  for (;;) {
    // the next target in x-major order among the four buckets (a target lies in one cell only)
    uint32_t best = 0xffffffffu;
    int kb = -1;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (pos[k] < lim[k]) {
        const uint32_t t = __ldg(order + pos[k]);
        if (t < best) { best = t; kb = k; }
      }
    }
    if (kb < 0) break;
#pragma unroll
    for (int k = 0; k < 4; ++k) pos[k] += (k == kb);
    const int ty = (int)(best % h);
    const int tx = (int)((best / h) % w);
    const Cell q = cell_of(flow, n, h, w, ty, tx);
    const bool hTL = q.T == py && q.L == px, hTR = q.T == py && q.R == px;
    const bool hBL = q.B == py && q.L == px, hBR = q.B == py && q.R == px;
    const float a1 = __fsub_rn(1.f, q.a), b1 = __fsub_rn(1.f, q.b);
    const int64_t tp = (int64_t)ty * w + tx;
#pragma unroll
    for (int k = 0; k < kWarpCh; ++k) {
      if (k >= nc) break;
      const float g = __ldg(dout + ((int64_t)n * c + c0 + k) * plane + tp);
      const float ga1 = __fmul_rn(g, a1), ga = __fmul_rn(g, q.a);
      float s = sum[k];
      if (hTL) s = __fadd_rn(s, __fmul_rn(ga1, b1));
      if (hTR) s = __fadd_rn(s, __fmul_rn(ga, b1));
      if (hBL) s = __fadd_rn(s, __fmul_rn(ga1, q.b));
      if (hBR) s = __fadd_rn(s, __fmul_rn(ga, q.b));
      sum[k] = s;
    }
  }
  for (int k = 0; k < nc; ++k) image_grad[((int64_t)n * c + c0 + k) * plane + p] = sum[k];
}

__global__ void __launch_bounds__(kWarpThreads) flow_out_of_frame_kernel(const float* __restrict__ flow, const float* __restrict__ occ,
                                                                          float* __restrict__ out, int n_img, int h, int w) {
  const int64_t plane = (int64_t)h * w;
  const int64_t i = (int64_t)blockIdx.x * kWarpThreads + threadIdx.x;
  if (i >= (int64_t)n_img * plane) return;
  const int64_t n = i / plane, p = i % plane;
  const int y = (int)(p / w), x = (int)(p % w);
  const float fx = __ldg(flow + 2 * n * plane + p), fy = __ldg(flow + (2 * n + 1) * plane + p);
  // ROUND_2_INT(f) = (int)(f >= 0.0 ? f + 0.5 : f - 0.5) in double: its truncation lies in [0, size) exactly when
  // -1 < d < size; a NaN or infinite d fails both tests, as x86's INT_MIN does, and so does any d past the int range
  const float xf = __fadd_rn((float)x, fx), yf = __fadd_rn((float)y, fy);
  const double dx = xf >= 0.0 ? __dadd_rn((double)xf, 0.5) : __dsub_rn((double)xf, 0.5);
  const double dy = yf >= 0.0 ? __dadd_rn((double)yf, 0.5) : __dsub_rn((double)yf, 0.5);
  const bool in = dx > -1.0 && dy > -1.0 && dx < (double)w && dy < (double)h;
  const float o = __ldg(occ + i);
  out[i] = (in || isnan(o)) ? o : 1.0f;
}

struct ResampleGeom {
  int64_t nc;                 // n * c planes
  int ih, iw, oh, ow;
  float fx, fy, ax, ay;
  int rx, ry;
  int type;                   // DEMON_LMB_RESAMPLE_*
};

__device__ __forceinline__ float bicubic_coeff(float v) {
  const float x = fabsf(v);
  if (x <= 1.0f) return __fmaf_rn(__fmul_rn(x, x), __fmaf_rn(1.5f, x, -2.5f), 1.0f);
  if (x < 2.0f) return __fmaf_rn(x, __fmaf_rn(x, __fmaf_rn(-0.5f, x, 2.5f), -4.0f), 2.0f);
  return 0.0f;
}

__device__ __forceinline__ float triangle_coeff(float x) {
  if (-1.f <= x && x < 0.f) return __fadd_rn(x, 1.f);
  if (0.f <= x && x <= 1.f) return __fsub_rn(1.f, x);
  return 0.f;
}

__device__ __forceinline__ float dmix(float w, float v, float s) { return __fmaf_rn(w, v, s); }
__device__ __forceinline__ double dmix(float w, double v, double s) { return __fma_rn((double)w, v, s); }
__device__ __forceinline__ float dacc(float s, float w) { return __fadd_rn(s, w); }
__device__ __forceinline__ double dacc(double s, float w) { return __dadd_rn(s, (double)w); }

template <typename T>
__global__ void __launch_bounds__(kResampleThreads) resample_kernel(const T* __restrict__ in, T* __restrict__ out, const ResampleGeom g) {
  const int64_t oplane = (int64_t)g.oh * g.ow;
  const int64_t idx = (int64_t)blockIdx.x * kResampleThreads + threadIdx.x;
  if (idx >= g.nc * oplane) return;
  const int64_t pl = idx / oplane, r = idx % oplane;
  const int xo = (int)(r % g.ow), yo = (int)(r / g.ow);
  // the reference's half offsets are swapped: fy / 2 along x, fx / 2 along y
  const float x_in = __fadd_rn(__fmaf_rn((float)xo, g.fx, __fmul_rn(g.fy, 0.5f)), -0.5f);
  const float y_in = __fadd_rn(__fmaf_rn((float)yo, g.fy, __fmul_rn(g.fx, 0.5f)), -0.5f);
  const int xr = (int)roundf(x_in), yr = (int)roundf(y_in);
  const T* src = in + pl * (int64_t)g.ih * g.iw;
  if (g.type == DEMON_LMB_RESAMPLE_NEAREST) {
    const int xc = min(max(xr, 0), g.iw - 1), yc = min(max(yr, 0), g.ih - 1);
    out[idx] = src[(int64_t)yc * g.iw + xc];
    return;
  }
  T sum = 0, wsum = 0;
  // the reference's window minus the positions it skips (outside the image), in its order
  const int y0 = max(yr - g.ry, 0), y1 = min(yr + g.ry, g.ih - 1);
  const int x0 = max(xr - g.rx, 0), x1 = min(xr + g.rx, g.iw - 1);
  for (int y = y0; y <= y1; ++y) {
    const float dy = __fmul_rn(g.ay, __fsub_rn(y_in, (float)y));
    const float ky = g.type == DEMON_LMB_RESAMPLE_CUBIC ? bicubic_coeff(dy) : triangle_coeff(dy);
    const T* row = src + (int64_t)y * g.iw;
    for (int x = x0; x <= x1; ++x) {
      const float dx = __fmul_rn(g.ax, __fsub_rn(x_in, (float)x));
      const float kx = g.type == DEMON_LMB_RESAMPLE_CUBIC ? bicubic_coeff(dx) : triangle_coeff(dx);
      const float wt = __fmul_rn(__fmul_rn(__fmul_rn(g.ax, kx), g.ay), ky);
      sum = dmix(wt, __ldg(row + x), sum);
      wsum = dacc(wsum, wt);
    }
  }
  out[idx] = (wsum == (T)0) ? (T)0 : sum / wsum;
}

int flow_warp_run(const float* image, const float* flow, float* out, int n, int c, int h, int w, int fill, void* stream) {
  DEMON_REQUIRE(fill == DEMON_FLOW_WARP_ZERO || fill == DEMON_FLOW_WARP_NAN,
                "flow_warp: fill must be DEMON_FLOW_WARP_ZERO or DEMON_FLOW_WARP_NAN (got %d)", fill);
  DEMON_REQUIRE(n >= 0 && c >= 0 && h >= 0 && w >= 0, "flow_warp: negative size");
  if ((int64_t)n * c * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(image && flow && out, "flow_warp: null pointer");
  const int ncg = ceil_div(c, kWarpCh);
  const int64_t blocks = ceil_div64((int64_t)h * w, kWarpThreads) * ncg * n;
  DEMON_REQUIRE(blocks < (1ll << 31), "flow_warp: input too large");
  uint32_t nan_bits = 0xFFE00000u;   // the reference GPU kernel's fill (flowwarp_cuda.cu: int nan = 0xFFE00000)
  float fv = 0.f;
  if (fill == DEMON_FLOW_WARP_NAN) memcpy(&fv, &nan_bits, sizeof fv);
  flow_warp_kernel<<<(unsigned)blocks, kWarpThreads, 0, (cudaStream_t)stream>>>(image, flow, out, n, c, h, w, ncg, fv);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// workspace: keys, sorted keys, order, sorted order, start, end (uint32 per target each), then CUB's temporary storage
int64_t grad_arrays_bytes(int64_t total) { return (6 * total * (int64_t)sizeof(uint32_t) + 255) / 256 * 256; }

int sort_bits(int64_t total) {
  int bits = 1;
  while (bits < 32 && ((uint64_t)1 << bits) <= (uint64_t)total) ++bits;
  return bits;
}

int grad_workspace(int n, int h, int w, int64_t* bytes, size_t* cub_bytes) {
  DEMON_REQUIRE(n >= 0 && h >= 0 && w >= 0, "flow_warp_grad: negative size");
  const int64_t total = (int64_t)n * h * w;
  DEMON_REQUIRE(total < (1ll << 31) - 1, "flow_warp_grad: n*h*w must be below 2^31 - 1 (got %lld)", (long long)total);
  *bytes = 0;
  *cub_bytes = 0;
  if (total == 0) return DEMON_OK;
  DEMON_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, *cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                   (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)total, 0, sort_bits(total)));
  *bytes = grad_arrays_bytes(total) + (int64_t)*cub_bytes;
  return DEMON_OK;
}

int flow_warp_grad_run(const float* image, const float* flow, const float* dout, float* image_grad, float* flow_grad, int n, int c, int h,
                       int w, void* workspace, int64_t workspace_bytes, void* stream) {
  DEMON_REQUIRE(c >= 0, "flow_warp_grad: negative size");
  size_t cub_bytes = 0;
  int64_t need = 0;
  const int rc = grad_workspace(n, h, w, &need, &cub_bytes);
  if (rc != DEMON_OK) return rc;
  const int64_t total = (int64_t)n * h * w;
  if (total == 0) return DEMON_OK;
  DEMON_REQUIRE(image && flow && dout && image_grad && flow_grad, "flow_warp_grad: null pointer");
  DEMON_REQUIRE(workspace && workspace_bytes >= need, "flow_warp_grad: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                (long long)need);
  DEMON_REQUIRE(((uintptr_t)workspace & 255) == 0, "flow_warp_grad: workspace must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  uint32_t* keys = (uint32_t*)workspace;
  uint32_t* keys_sorted = keys + total;
  uint32_t* vals = keys_sorted + total;
  uint32_t* order = vals + total;
  uint32_t* start = order + total;
  uint32_t* end = start + total;
  void* cub_tmp = (char*)workspace + grad_arrays_bytes(total);
  const unsigned tblocks = (unsigned)ceil_div64(total, kWarpThreads);

  flow_warp_flow_grad_kernel<<<tblocks, kWarpThreads, 0, st>>>(image, flow, dout, flow_grad, n, c, h, w);
  DEMON_LAUNCH_CHECK();
  if (c == 0) return DEMON_OK;
  flow_warp_cells_kernel<<<tblocks, kWarpThreads, 0, st>>>(flow, keys, vals, start, end, n, h, w);
  DEMON_LAUNCH_CHECK();
  // stable: each cell's bucket keeps the targets in x-major order
  size_t tmp = cub_bytes;
  DEMON_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, tmp, keys, keys_sorted, vals, order, (int)total, 0, sort_bits(total), st));
  flow_warp_bounds_kernel<<<tblocks, kWarpThreads, 0, st>>>(keys_sorted, start, end, (uint32_t)total);
  DEMON_LAUNCH_CHECK();
  const int ncg = ceil_div(c, kWarpCh);
  const int64_t blocks = ceil_div64((int64_t)h * w, kWarpThreads) * ncg * n;
  DEMON_REQUIRE(blocks < (1ll << 31), "flow_warp_grad: input too large");
  flow_warp_image_grad_kernel<<<(unsigned)blocks, kWarpThreads, 0, st>>>(flow, dout, order, start, end, image_grad, n, c, h, w, ncg);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

template <typename T>
int resample_run(const T* in, T* out, int n, int c, int ih, int iw, int oh, int ow, int antialias, int type, void* stream) {
  DEMON_REQUIRE(type == DEMON_LMB_RESAMPLE_NEAREST || type == DEMON_LMB_RESAMPLE_CUBIC || type == DEMON_LMB_RESAMPLE_LINEAR,
                "resample: type must be DEMON_LMB_RESAMPLE_NEAREST, _CUBIC or _LINEAR (got %d)", type);
  DEMON_REQUIRE(oh >= 1 && ow >= 1, "resample: width and height must be >= 1 (got %d, %d)", ow, oh);
  DEMON_REQUIRE(n >= 0 && c >= 0 && ih >= 0 && iw >= 0, "resample: negative size");
  const int64_t total = (int64_t)n * c * oh * ow;
  if (total == 0) return DEMON_OK;
  DEMON_REQUIRE(ih >= 1 && iw >= 1, "resample: empty input image");
  DEMON_REQUIRE(in && out, "resample: null pointer");
  ResampleGeom g;
  g.nc = (int64_t)n * c;
  g.ih = ih; g.iw = iw; g.oh = oh; g.ow = ow;
  g.type = type;
  // ResampleOp_GPU::Compute: the scale factors in float, antialias only when either axis downsamples
  g.fx = (float)iw / (float)ow;
  g.fy = (float)ih / (float)oh;
  const bool aa = antialias && (g.fx > 1.f || g.fy > 1.f);
  g.ax = 1.0f / (aa ? g.fx : 1.0f);
  g.ay = 1.0f / (aa ? g.fy : 1.0f);
  const float kw = type == DEMON_LMB_RESAMPLE_CUBIC ? 4.f : 2.f;
  g.rx = g.fx < 1.0f ? 2 : (int)std::ceil(kw / g.ax);
  g.ry = g.fy < 1.0f ? 2 : (int)std::ceil(kw / g.ay);
  const int64_t blocks = ceil_div64(total, kResampleThreads);
  DEMON_REQUIRE(blocks < (1ll << 31), "resample: output too large");
  resample_kernel<T><<<(unsigned)blocks, kResampleThreads, 0, (cudaStream_t)stream>>>(in, out, g);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

extern "C" {

int demon_flow_warp_f32(const float* image, const float* flow, float* warped, int n, int c, int h, int w, int fill, void* stream) {
  return demon::flow_warp_run(image, flow, warped, n, c, h, w, fill, stream);
}

int64_t demon_flow_warp_grad_workspace_bytes(int n, int h, int w) {
  size_t cub_bytes = 0;
  int64_t bytes = 0;
  return demon::grad_workspace(n, h, w, &bytes, &cub_bytes) == DEMON_OK ? bytes : -1;
}

int demon_flow_warp_grad_f32(const float* image, const float* flow, const float* gradient, float* image_grad, float* flow_grad, int n, int c,
                             int h, int w, void* workspace, int64_t workspace_bytes, void* stream) {
  return demon::flow_warp_grad_run(image, flow, gradient, image_grad, flow_grad, n, c, h, w, workspace, workspace_bytes, stream);
}

int demon_flow_out_of_frame_f32(const float* flow, const float* occ, float* output, int n, int h, int w, void* stream) {
  DEMON_REQUIRE(n >= 0 && h >= 0 && w >= 0, "flow_out_of_frame: negative size");
  const int64_t total = (int64_t)n * h * w;
  if (total == 0) return DEMON_OK;
  DEMON_REQUIRE(flow && occ && output, "flow_out_of_frame: null pointer");
  const int64_t blocks = demon::ceil_div64(total, demon::kWarpThreads);
  DEMON_REQUIRE(blocks < (1ll << 31), "flow_out_of_frame: input too large");
  demon::flow_out_of_frame_kernel<<<(unsigned)blocks, demon::kWarpThreads, 0, (cudaStream_t)stream>>>(flow, occ, output, n, h, w);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_resample_f32(const float* input, float* output, int n, int c, int in_h, int in_w, int out_h, int out_w, int antialias, int type,
                       void* stream) {
  return demon::resample_run<float>(input, output, n, c, in_h, in_w, out_h, out_w, antialias, type, stream);
}

int demon_resample_f64(const double* input, double* output, int n, int c, int in_h, int in_w, int out_h, int out_w, int antialias, int type,
                       void* stream) {
  return demon::resample_run<double>(input, output, n, c, in_h, in_w, out_h, out_w, antialias, type, stream);
}

}  // extern "C"
