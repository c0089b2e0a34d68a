// Evaluation metrics of the DeMoN path on the device (SURVEY.md section 8 f3): the masked per-sample sums behind
// depthmotionnet.evaluation.metrics.compute_errors / evaluate_depth / compute_flow_epe
// (python/depthmotionnet/evaluation/metrics.py:25-38,62-237,240-372,377-387), so that a dataset-level accuracy run never
// copies a depth map to the host: one pass over prediction and ground truth produces every sum the eleven distances and
// the least-squares scale factor need.  HBM-bound streaming reductions: 8 bytes in per pixel, nothing out but
// [n][16] doubles.
//
// Element-wise arithmetic is float32 with IEEE operations like numpy's (reciprocal, division, subtraction; log / log10 are
// CUDA's logf / log10f, within 1-2 ulp of numpy's), accumulation is double in a FIXED order (per-thread strided partial
// sums -> warp shuffle tree -> per-CTA slots -> one warp folds the slots in index order), so results are deterministic
// run to run; the reference accumulates pairwise in float32, which is where the documented 1e-5 tolerance comes from.
// Promotion is NumPy 1.x's: the gt divide and the prediction's scale are float32, and the ratio thresholds compare the
// float32 |ld| with float32(log t), which is what logf(t) gives here (DESIGN.md §3.4, tests/test_gpu_metrics_oracle.py).
#include "common.cuh"
#include <cmath>

namespace demon {
namespace {

constexpr int kSums = 16;
constexpr int kMetricThreads = 256;
constexpr int kMaxSlots = 64;   // CTAs per sample

__device__ __forceinline__ bool valid_pair(float a, float b) { return isfinite(a) && isfinite(b) && a > 0.f && b > 0.f; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Where pixel i of sample n lives.  Dense: pred and gt are [n, hw].  Resampled: i enumerates the output window
// [oh, ow] of a [gh, gw] ground truth; the prediction [ph, pw] is read through the nearest-neighbour tables (-1 reads 0,
// skimage's cval) and a gt pixel whose gt_valid byte is 0 reads NaN.  Both kernels below take the mapping as a template
// argument, so the per-pixel arithmetic and the reduction order are one piece of code for both.
struct DensePixels {
  const float* pred;
  const float* gt;
  long hw;
  __device__ __forceinline__ long count() const { return hw; }
  __device__ __forceinline__ void load(int n, long i, float& p, float& g) const {
    p = __ldg(pred + (long)n * hw + i);
    g = __ldg(gt + (long)n * hw + i);
  }
  // the two channels of a flow field [n, 2, hw]
  __device__ __forceinline__ void load2(int n, long i, float& px, float& py, float& gx, float& gy) const {
    const long b = (long)n * 2 * hw + i;
    px = __ldg(pred + b); py = __ldg(pred + b + hw);
    gx = __ldg(gt + b); gy = __ldg(gt + b + hw);
  }
};

struct ResampledPixels {
  const float* pred;
  const float* gt;
  const unsigned char* gt_valid;
  const int* row_idx;
  const int* col_idx;
  int ph, pw, gh, gw, y0, x0, oh, ow;
  __device__ __forceinline__ long count() const { return (long)oh * ow; }
  // offsets of window pixel i in the prediction (-1: outside) and in the ground truth
  __device__ __forceinline__ void offsets(long i, long& po, long& go) const {
    const int r = (int)(i / ow), c = (int)(i - (long)r * ow);
    const int pr = __ldg(row_idx + r), pc = __ldg(col_idx + c);
    po = (pr < 0 || pc < 0) ? -1 : (long)pr * pw + pc;
    go = (long)(y0 + r) * gw + (x0 + c);
  }
  __device__ __forceinline__ void load(int n, long i, float& p, float& g) const {
    long po, go;
    offsets(i, po, go);
    const long gn = (long)n * gh * gw;
    p = po < 0 ? 0.f : __ldg(pred + (long)n * ph * pw + po);
    g = (gt_valid && __ldg(gt_valid + gn + go) == 0) ? __int_as_float(0x7fc00000) : __ldg(gt + gn + go);
  }
  __device__ __forceinline__ void load2(int n, long i, float& px, float& py, float& gx, float& gy) const {
    long po, go;
    offsets(i, po, go);
    const long pp = (long)ph * pw, gp = (long)gh * gw;
    const float* a = pred + (long)n * 2 * pp;
    const float* b = gt + (long)n * 2 * gp;
    px = po < 0 ? 0.f : __ldg(a + po);
    py = po < 0 ? 0.f : __ldg(a + pp + po);
    gx = __ldg(b + go); gy = __ldg(b + gp + go);
  }
};

// partial[n][slot][kSums]
template <class Pixels>
__global__ void __launch_bounds__(kMetricThreads) depth_sums_kernel(const Pixels px, bool inverse_pred, bool inverse_gt,
                                                                   const float* __restrict__ gt_div, const float* __restrict__ pred_scale,
                                                                   double* __restrict__ partial) {
  const int n = blockIdx.y, slot = blockIdx.x, nslots = gridDim.x;
  const long hw = px.count();
  const float gdiv = gt_div ? __ldg(gt_div + n) : 1.0f;
  const float pscale = pred_scale ? __ldg(pred_scale + n) : 1.0f;
  const float l125 = logf(1.25f), l156 = logf(1.5625f), l195 = logf(1.953125f);
  double acc[kSums];
#pragma unroll
  for (int k = 0; k < kSums; ++k) acc[k] = 0.0;
  for (long i = (long)slot * kMetricThreads + threadIdx.x; i < hw; i += (long)nslots * kMetricThreads) {
    float pi, gi;
    px.load(n, i, pi, gi);
    if (!valid_pair(pi, gi)) continue;                       // compute_valid_depth_mask on the inputs (metrics.py:337)
    float dp = inverse_pred ? fdiv(1.0f, pi) : pi;           // metrics.py:339-342
    float dg = inverse_gt ? fdiv(1.0f, gi) : gi;
    if (gt_div) dg = fdiv(dg, gdiv);                         // metrics.py:349-355
    // least-squares scale factor sums on the UNSCALED prediction (metrics.py:283-318)
    const float pp = fmul(dp, dp), pg = fmul(dp, dg);
    if (isfinite(pg) && pg > 0.f) { acc[12] += (double)pp; acc[13] += (double)pg; }
    const float ip = fdiv(1.0f, dp), ig = fdiv(1.0f, dg);
    const float ipp = fmul(ip, ip), ipg = fmul(ip, ig);
    if (isfinite(ipg) && ipg > 0.f) { acc[14] += (double)ipp; acc[15] += (double)ipg; }
    if (pred_scale) dp = fmul(dp, pscale);                   // metrics.py:362
    if (!valid_pair(dp, dg)) continue;                       // compute_errors masks again (metrics.py:252)
    const float d = fsub(dp, dg);
    const float ld = fsub(logf(dp), logf(dg));
    acc[0] += 1.0;
    acc[1] += (double)fabsf(d);
    acc[2] += (double)fabsf(fsub(fdiv(1.0f, dp), fdiv(1.0f, dg)));
    acc[3] += (double)ld;
    acc[4] += (double)fmul(ld, ld);
    acc[5] += (double)fdiv(fabsf(d), dg);
    acc[6] += (double)fdiv(fmul(d, d), dg);
    acc[7] += (double)fabsf(fsub(log10f(dp), log10f(dg)));
    acc[8] += (double)fmul(d, d);
    const float ald = fabsf(ld);
    acc[9] += (ald < l125) ? 1.0 : 0.0;
    acc[10] += (ald < l156) ? 1.0 : 0.0;
    acc[11] += (ald < l195) ? 1.0 : 0.0;
  }
  __shared__ double red[kMetricThreads / 32][kSums];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < kSums; ++k) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < kSums) {
    double v = 0.0;
    for (int w = 0; w < kMetricThreads / 32; ++w) v += red[w][threadIdx.x];
    partial[((long)n * nslots + slot) * kSums + threadIdx.x] = v;
  }
}

__global__ void fold_kernel(const double* __restrict__ partial, int nslots, int width, double* __restrict__ sums) {
  const int n = blockIdx.x, k = threadIdx.x;
  if (k >= width) return;
  double v = 0.0;
  for (int s = 0; s < nslots; ++s) v += partial[((long)n * nslots + s) * width + k];
  sums[(long)n * width + k] = v;
}

// scale[n] from the folded sums: mode 0 'abs', 1 'log', 2 'inv' (metrics.py:283-318)
__global__ void scale_kernel(const double* __restrict__ sums, int n, int mode, float* __restrict__ scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* s = sums + (long)i * kSums;
  double r = 1.0;
  if (mode == 0) { if (s[12] > 0.0) r = s[13] / s[12]; }
  else if (mode == 1) { if (s[0] > 0.0) r = exp(-s[3] / s[0]); }
  else { if (s[14] > 0.0) r = 1.0 / (s[15] / s[14]); }
  scale[i] = (float)r;
}

template <class Pixels>
__global__ void __launch_bounds__(kMetricThreads) epe_sums_kernel(const Pixels px, double* __restrict__ partial) {
  const int n = blockIdx.y, slot = blockIdx.x, nslots = gridDim.x;
  const long hw = px.count();
  double sum = 0.0, cnt = 0.0;
  for (long i = (long)slot * kMetricThreads + threadIdx.x; i < hw; i += (long)nslots * kMetricThreads) {
    float ax, ay, bx, by;
    px.load2(n, i, ax, ay, bx, by);
    const float dx = fsub(ax, bx), dy = fsub(ay, by);
    const float epe = sqrtf(fadd(fmul(dx, dx), fmul(dy, dy)));     // metrics.py:379-380
    if (isfinite(epe) && epe > 0.f) { sum += (double)epe; cnt += 1.0; }   // compute_valid_depth_mask(epe), metrics.py:382
  }
  __shared__ double red[kMetricThreads / 32][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  sum = warp_sum(sum); cnt = warp_sum(cnt);
  if (lane == 0) { red[warp][0] = sum; red[warp][1] = cnt; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double v = 0.0;
    for (int w = 0; w < kMetricThreads / 32; ++w) v += red[w][threadIdx.x];
    partial[((long)n * nslots + slot) * 2 + threadIdx.x] = v;
  }
}

// compute_motion_errors (metrics.py:390-445) with normalize_translations, as demon_b200.evaluation restates it: minieigen's
// Quaternion(angle, axis) with the 1e-6 angle rule, angularDistance = 2 acos(|q1 . q2|) unless |q1 . q2| >= 1; NaN in,
// NaN out (no comparison below is true for a NaN, and the clip keeps NaN like numpy.clip)
__device__ void motion_quat(const double aa[3], double q[4]) {
  double angle = sqrt(aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]);
  double ax[3] = {1.0, 0.0, 0.0};
  if (angle < 1e-6) {
    angle = 0.0;
  } else {
    for (int k = 0; k < 3; ++k) ax[k] = aa[k] / angle;
    const double m = sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
    for (int k = 0; k < 3; ++k) ax[k] = ax[k] / m;
  }
  const double s = sin(angle / 2);
  q[0] = cos(angle / 2);
  for (int k = 0; k < 3; ++k) q[k + 1] = s * ax[k];
}

__global__ void motion_errors_kernel(const float* __restrict__ prot, const float* __restrict__ ptrans, const float* __restrict__ gt, int n,
                                     double* __restrict__ out, float* __restrict__ gt_div) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double rad2deg = 180.0 / 3.14159265358979323846;
  double gr[3], pr[3], gtr[3], pt[3];
  bool gt_nan = false;
  for (int k = 0; k < 3; ++k) {
    gr[k] = gt[6 * i + k]; gtr[k] = gt[6 * i + 3 + k];
    pr[k] = prot[3 * i + k]; pt[k] = ptrans[3 * i + k];
    gt_nan = gt_nan || isnan(gr[k]) || isnan(gtr[k]);
  }
  double qg[4], qp[4];
  motion_quat(gr, qg);
  motion_quat(pr, qp);
  const double d = fabs(qg[0] * qp[0] + qg[1] * qp[1] + qg[2] * qp[2] + qg[3] * qp[3]);
  const double rot = d >= 1.0 ? 0.0 : 2.0 * acos(d);
  const double gn = sqrt(gtr[0] * gtr[0] + gtr[1] * gtr[1] + gtr[2] * gtr[2]);
  const double pn = sqrt(pt[0] * pt[0] + pt[1] * pt[1] + pt[2] * pt[2]);
  double g[3], p[3];
  for (int k = 0; k < 3; ++k) { g[k] = gtr[k] / gn; p[k] = pn > 1e-6 ? pt[k] / pn : pt[k]; }
  const double dx = g[0] - p[0], dy = g[1] - p[1], dz = g[2] - p[2];
  double c = g[0] * p[0] + g[1] * p[1] + g[2] * p[2];
  if (c < -1.0) c = -1.0;
  if (c > 1.0) c = 1.0;
  double* o = out + 4L * i;
  o[0] = rot * rad2deg;
  o[1] = sqrt(dx * dx + dy * dy + dz * dz);
  o[2] = acos(c) * rad2deg;
  o[3] = gt_nan ? nan("") : gn;
  if (gt_div) {
    // evaluate_to_xarray.py:290-294: t_gt = (1, 0, 0) for a motion with a NaN; then evaluate_depth_batch's isclose rule
    const double norm = gt_nan ? 1.0 : gn;
    gt_div[i] = (float)(fabs(1.0 - norm) <= 1e-8 + 1e-5 * fabs(norm) ? 1.0 : norm);
  }
}

int slots_for(int64_t hw) {
  int64_t s = (hw + 4 * kMetricThreads - 1) / (4 * kMetricThreads);
  return (int)(s < 1 ? 1 : (s > kMaxSlots ? kMaxSlots : s));
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int64_t demon_metric_workspace_bytes(int n, int64_t hw) {
  // hw == 0 still launches one slot per sample, which writes its (zero) partial sums
  if (n <= 0 || hw < 0) return 0;
  return (int64_t)n * slots_for(hw) * kSums * (int64_t)sizeof(double);
}

int demon_depth_error_sums_f32(const float* pred, const float* gt, int n, int64_t hw, int inverse_pred, int inverse_gt, const float* gt_div,
                               const float* pred_scale, double* sums, void* workspace, void* stream) {
  DEMON_REQUIRE(n >= 0 && hw >= 0 && n <= 65535, "depth_error_sums: bad size");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(sums && workspace && (hw == 0 || (pred && gt)), "depth_error_sums: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int nslots = slots_for(hw);
  depth_sums_kernel<<<dim3(nslots, n), kMetricThreads, 0, s>>>(DensePixels{pred, gt, (long)hw}, inverse_pred != 0, inverse_gt != 0, gt_div,
                                                               pred_scale, static_cast<double*>(workspace));
  DEMON_LAUNCH_CHECK();
  fold_kernel<<<n, 32, 0, s>>>(static_cast<const double*>(workspace), nslots, kSums, sums);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_depth_scale_factor(const double* sums, int n, int mode, float* scale, void* stream) {
  DEMON_REQUIRE(n >= 0 && mode >= 0 && mode <= 2, "depth_scale_factor: bad argument");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(sums && scale, "depth_scale_factor: null pointer");
  scale_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(sums, n, mode, scale);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_flow_epe_sums_f32(const float* flow1, const float* flow2, int n, int64_t hw, double* sums, void* workspace, void* stream) {
  DEMON_REQUIRE(n >= 0 && hw >= 0 && n <= 65535, "flow_epe_sums: bad size");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(sums && workspace && (hw == 0 || (flow1 && flow2)), "flow_epe_sums: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int nslots = slots_for(hw);
  epe_sums_kernel<<<dim3(nslots, n), kMetricThreads, 0, s>>>(DensePixels{flow1, flow2, (long)hw}, static_cast<double*>(workspace));
  DEMON_LAUNCH_CHECK();
  fold_kernel<<<n, 32, 0, s>>>(static_cast<const double*>(workspace), nslots, 2, sums);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_depth_error_sums_resampled_f32(const float* pred, int ph, int pw, const float* gt, const uint8_t* gt_valid, int gh, int gw,
                                         int n, int y0, int x0, int oh, int ow, const int* row_idx, const int* col_idx,
                                         int inverse_pred, int inverse_gt, const float* gt_div, const float* pred_scale,
                                         double* sums, void* workspace, void* stream) {
  DEMON_REQUIRE(n >= 0 && n <= 65535 && ph > 0 && pw > 0 && gh > 0 && gw > 0 && oh >= 0 && ow >= 0, "depth_error_sums_resampled: bad size");
  DEMON_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + oh <= gh && x0 + ow <= gw, "depth_error_sums_resampled: window outside the ground truth");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(sums && workspace && pred && gt && row_idx && col_idx, "depth_error_sums_resampled: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int nslots = slots_for((int64_t)oh * ow);
  const ResampledPixels px{pred, gt, gt_valid, row_idx, col_idx, ph, pw, gh, gw, y0, x0, oh, ow};
  depth_sums_kernel<<<dim3(nslots, n), kMetricThreads, 0, s>>>(px, inverse_pred != 0, inverse_gt != 0, gt_div, pred_scale,
                                                               static_cast<double*>(workspace));
  DEMON_LAUNCH_CHECK();
  fold_kernel<<<n, 32, 0, s>>>(static_cast<const double*>(workspace), nslots, kSums, sums);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_flow_epe_sums_resampled_f32(const float* pred, int ph, int pw, const float* gt, int gh, int gw, int n, int y0, int x0,
                                      int oh, int ow, const int* row_idx, const int* col_idx, double* sums, void* workspace,
                                      void* stream) {
  DEMON_REQUIRE(n >= 0 && n <= 65535 && ph > 0 && pw > 0 && gh > 0 && gw > 0 && oh >= 0 && ow >= 0, "flow_epe_sums_resampled: bad size");
  DEMON_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + oh <= gh && x0 + ow <= gw, "flow_epe_sums_resampled: window outside the ground truth");
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(sums && workspace && pred && gt && row_idx && col_idx, "flow_epe_sums_resampled: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int nslots = slots_for((int64_t)oh * ow);
  const ResampledPixels px{pred, gt, nullptr, row_idx, col_idx, ph, pw, gh, gw, y0, x0, oh, ow};
  epe_sums_kernel<<<dim3(nslots, n), kMetricThreads, 0, s>>>(px, static_cast<double*>(workspace));
  DEMON_LAUNCH_CHECK();
  fold_kernel<<<n, 32, 0, s>>>(static_cast<const double*>(workspace), nslots, 2, sums);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_motion_errors(const float* pred_rotation, const float* pred_translation, const float* gt_motion, int n, double* out,
                        float* gt_div, void* stream) {
  DEMON_REQUIRE(n >= 0, "motion_errors: n %d", n);
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(pred_rotation && pred_translation && gt_motion && out, "motion_errors: null pointer");
  motion_errors_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(pred_rotation, pred_translation, gt_motion, n, out, gt_div);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // extern "C"
