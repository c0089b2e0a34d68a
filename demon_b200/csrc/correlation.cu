// FlowNet cost volumes on the device: lmbspecialops' Correlation / CorrelationGrad (correlation.cc, correlation_cuda.cu) and
// Correlation1D / Correlation1DGrad (correlation_1d.cc, correlation_1d_cuda.cu), float32 NCHW, bit for bit the reference's
// own CUDA kernels.
//
// Geometry, in coordinates of the zero-padded input (pad_size columns left and right, and for the 2D op pad_size rows above
// and below): top pixel (x, y) correlates the ks x ks patch of input1 whose top-left corner is (X1, Y1) = (x s1 + md,
// y s1 + mdy) with the patch of input2 displaced by (dx, dy) = ((dxi + xshift) s2, (dyi - ry) s2); top channel
// tc = dyi * gw + dxi.  2D: gw = gh = 2R + 1 with R = md / s2, xshift = -R, ry = R, mdy = md; 1D: gh = 1, ry = mdy = 0,
// gw = 2R + 1 (single_dir 0, xshift -R) or R + 1 (single_dir 1: xshift 0; single_dir -1: xshift -(R + 1), the reference's
// displacement set).  A read outside the padded input is 0: that is the padding, and for single_dir -1 it defines the
// reads the reference makes before the start of a padded row.
//
// What fixes each element's bits is the reference's operation order, kept here exactly:
//   mult forward  p_l = fma(a, b, p_l) over kernel row j, column i, then channels ch = l, l + 32, ... (l = 0..31), then
//                 total = ((0 + p_0) + p_1) + ... + p_31 and total / (ks ks C).  Lanes l >= C hold +0 and adding +0 to a
//                 total that cannot be -0 changes nothing, so they are skipped.
//   subt forward  sum += |a - b| over j, i, then every channel in order, / (ks ks C).
//   gradients     for every input element a gather over displacement row, displacement column, then the clamped top window
//                 (y, x): sum = fma(topdiff, v, sum), / (ks ks C); v is the other input at the displaced position (mult) or
//                 the sign of input1 >= input2 at one position (subt: +-1 for input1_grad, -+1 for input2_grad), exactly as
//                 the reference defines it.  No atomics: every element is written by one thread.
//
// Forward tiling: a CTA owns one top row of one image, 32 P consecutive top pixels (lane = pixel) and a block of NDY x NDX
// displacements (warp w takes displacements w, w + W, ...; D = 8 per thread), so a thread keeps 2 P D accumulators.  The
// inputs are staged through shared memory by channel class: for mult, stage l holds channels l, l + 32, ... of the patch
// rows and of the displaced windows, so the stride-32 channel walk of one lane partial reads consecutive shared rows and
// every global load is a coalesced row segment.
#include "common.cuh"
#include <cmath>

namespace demon {
namespace {

struct CorrGeom {
  int n, c, h, w;
  int ks, md, s1, s2, pad;
  int pady, mdy;              // 2D: pad, md; 1D: 0, 0
  int gw, gh, xshift, ry;     // displacement grid
  int tw, th, tc;             // top
  float sumelems;
};

// forward block plan (host-chosen)
struct FwdPlan {
  int nseg, ndxg, ndyg;       // top-pixel segments, displacement-column groups, displacement-row groups
  int ndx, ndy;               // displacements per group
  int rows;                   // kernel rows per stage: ks (all rows staged at once) or 1
  int ch;                     // channels per stage
  int colsA, colsB;           // staged columns of input1 / of each displaced input2 window
};

constexpr int kFwdD = 8;           // displacements per thread
constexpr int kFwdMaxWarps = 8;
constexpr int kSmemBudget = 48 * 1024;
constexpr int kGradThreads = 64;   // consecutive input pixels of one row
constexpr int kGradCh = 8;         // channels per thread

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
__device__ __forceinline__ int ceil_div_signed(int a, int b) { return floor_div(a + b - 1, b); }

__device__ __forceinline__ float padded(const float* plane, int py, int px, const CorrGeom& g) {
  const int y = py - g.pady, x = px - g.pad;
  return (y >= 0 && y < g.h && x >= 0 && x < g.w) ? __ldg(plane + (size_t)y * g.w + x) : 0.f;
}

template <bool SUBT, int P>
__global__ void __launch_bounds__(kFwdMaxWarps * 32, 2) correlation_fwd_kernel(const float* __restrict__ in1, const float* __restrict__ in2,
                                                                            float* __restrict__ out, const CorrGeom g, const FwdPlan f) {
  extern __shared__ float smem[];
  int b = blockIdx.x;
  const int seg = b % f.nseg; b /= f.nseg;
  const int dxg = b % f.ndxg; b /= f.ndxg;
  const int dyg = b % f.ndyg; b /= f.ndyg;
  const int y = b % g.th;
  const int img = b / g.th;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

  const int x0 = seg * 32 * P;                      // first top pixel of the CTA
  const int X10 = x0 * g.s1 + g.md;                 // its patch's first padded column
  const int Y1 = y * g.s1 + g.mdy;
  const int dxi0 = dxg * f.ndx, dyi0 = dyg * f.ndy;
  const int dxmin = (dxi0 + g.xshift) * g.s2;       // the group's first displacement column
  float* sA = smem;                                               // [rows][ch][colsA]
  float* sB = smem + (size_t)f.rows * f.ch * f.colsA;             // [ndy][rows][ch][colsB]

  // this thread's displacements
  int dxl[kFwdD], dyl[kFwdD];
  bool dvalid[kFwdD];
#pragma unroll
  for (int d = 0; d < kFwdD; ++d) {
    const int e = warp + nwarps * d;
    const bool in_group = e < f.ndx * f.ndy;
    const int yl = in_group ? e / f.ndx : 0, xl = in_group ? e % f.ndx : 0;
    dvalid[d] = in_group && dxi0 + xl < g.gw && dyi0 + yl < g.gh;
    dxl[d] = dvalid[d] ? xl : 0;
    dyl[d] = dvalid[d] ? yl : 0;
  }
  // shared-memory offset of each displacement's window (sB is [ndy][rows][ch][colsB])
  int boff[kFwdD];
#pragma unroll
  for (int d = 0; d < kFwdD; ++d) boff[d] = dyl[d] * f.rows * f.ch * f.colsB + dxl[d] * g.s2;

  const size_t plane = (size_t)g.h * g.w;
  const float* img1 = in1 + (size_t)img * g.c * plane;
  const float* img2 = in2 + (size_t)img * g.c * plane;

  float total[P][kFwdD], acc[P][kFwdD];
#pragma unroll
  for (int p = 0; p < P; ++p)
#pragma unroll
    for (int d = 0; d < kFwdD; ++d) total[p][d] = 0.f;

  const int nl = SUBT ? 1 : min(32, g.c);
  for (int l = 0; l < nl; ++l) {
    const int nch = SUBT ? g.c : (g.c - l + 31) / 32;    // channels of this class
    const int nchunks = (nch + f.ch - 1) / f.ch;
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
      for (int d = 0; d < kFwdD; ++d) acc[p][d] = 0.f;
    for (int j = 0; j < g.ks; ++j) {
      for (int i = 0; i < g.ks; ++i) {
        for (int k = 0; k < nchunks; ++k) {
          const int k0 = k * f.ch;
          const int nt = min(f.ch, nch - k0);
          // several chunks: every chunk is staged where it is used; one chunk: once per class (all rows) or per row
          const bool restage = nchunks > 1 || ((f.rows == g.ks) ? (j == 0 && i == 0) : i == 0);
          if (restage) {
            const int jlo = (f.rows == g.ks) ? 0 : j;
            __syncthreads();
            // one warp per staged row, lanes along its columns: coalesced global reads, no per-element division
            const int na = f.rows * f.ch;
            for (int r = warp; r < na + f.ndy * na; r += nwarps) {
              const bool is_a = r < na;
              const int rr = is_a ? r : r - na;
              const int t = rr % f.ch, jr = (rr / f.ch) % f.rows, yl = is_a ? 0 : rr / na;
              const int ch = SUBT ? k0 + t : l + 32 * (k0 + t);
              const int py = Y1 + jlo + jr + (is_a ? 0 : (dyi0 + yl - g.ry) * g.s2) - g.pady;
              const int px0 = X10 + (is_a ? 0 : dxmin) - g.pad;
              const int ncols = is_a ? f.colsA : f.colsB;
              float* dst = is_a ? sA + (size_t)rr * f.colsA : sB + (size_t)rr * f.colsB;
              const bool row_ok = t < nt && py >= 0 && py < g.h && (is_a || dyi0 + yl < g.gh);
              const float* src = (is_a ? img1 : img2) + (size_t)(row_ok ? ch : 0) * plane + (size_t)(row_ok ? py : 0) * g.w;
              for (int col = lane; col < ncols; col += 32) {
                const int x = px0 + col;
                dst[col] = (row_ok && x >= 0 && x < g.w) ? __ldg(src + x) : 0.f;
              }
            }
            __syncthreads();
          }
          const int jr = (f.rows == g.ks) ? j : 0;
          const float* a_row = sA + jr * f.ch * f.colsA + lane * g.s1 + i;
          const float* b_row = sB + jr * f.ch * f.colsB + lane * g.s1 + i;
          for (int t = 0; t < nt; ++t) {
            float a[P];
#pragma unroll
            for (int p = 0; p < P; ++p) a[p] = a_row[t * f.colsA + 32 * p * g.s1];
#pragma unroll
            for (int d = 0; d < kFwdD; ++d) {
              const float* bd = b_row + boff[d] + t * f.colsB;
#pragma unroll
              for (int p = 0; p < P; ++p) {
                const float bv = bd[32 * p * g.s1];
                if (SUBT) acc[p][d] = __fadd_rn(acc[p][d], fabsf(__fsub_rn(a[p], bv)));
                else acc[p][d] = __fmaf_rn(a[p], bv, acc[p][d]);
              }
            }
          }
        }
      }
    }
    if (!SUBT) {
#pragma unroll
      for (int p = 0; p < P; ++p)
#pragma unroll
        for (int d = 0; d < kFwdD; ++d) total[p][d] = __fadd_rn(total[p][d], acc[p][d]);
    }
  }

#pragma unroll
  for (int d = 0; d < kFwdD; ++d) {
    if (!dvalid[d]) continue;
    const int tc = (dyi0 + dyl[d]) * g.gw + dxi0 + dxl[d];
    float* o = out + (((size_t)img * g.tc + tc) * g.th + y) * g.tw;
#pragma unroll
    for (int p = 0; p < P; ++p) {
      const int x = x0 + lane + 32 * p;
      if (x < g.tw) o[x] = __fdiv_rn(SUBT ? acc[p][d] : total[p][d], g.sumelems);
    }
  }
}

// One thread = one input pixel of one row and kGradCh channels.  SECOND: input2_grad, else input1_grad.
template <bool SUBT, bool SECOND>
__global__ void __launch_bounds__(kGradThreads) correlation_grad_kernel(const float* __restrict__ in1, const float* __restrict__ in2,
                                                                        const float* __restrict__ gtop, float* __restrict__ grad,
                                                                        const CorrGeom g, int nxseg, int ncg) {
  int b = blockIdx.x;
  const int xs = b % nxseg; b /= nxseg;
  const int cg = b % ncg; b /= ncg;
  const int yy = b % g.h;
  const int img = b / g.h;
  const int xx = xs * kGradThreads + threadIdx.x;
  if (xx >= g.w) return;
  const int l = xx + g.pad, m = yy + g.pady;
  const int kr2 = g.ks - 1;                        // 2 * kernel radius
  const size_t plane = (size_t)g.h * g.w;
  const float* p1[kGradCh];
  const float* p2[kGradCh];
#pragma unroll
  for (int cc = 0; cc < kGradCh; ++cc) {
    const int ch = min(cg * kGradCh + cc, g.c - 1);
    p1[cc] = in1 + ((size_t)img * g.c + ch) * plane;
    p2[cc] = in2 + ((size_t)img * g.c + ch) * plane;
  }
  const float* gt = gtop + (size_t)img * g.tc * g.th * g.tw;
  float sum[kGradCh];
#pragma unroll
  for (int cc = 0; cc < kGradCh; ++cc) sum[cc] = 0.f;

  int xmin = 0, xmax = -1, ymin = 0, ymax = -1;
  bool any = true;
  if (!SECOND) {   // the top window whose patches cover (m, l) does not depend on the displacement
    xmin = ceil_div_signed(l - kr2 - g.md, g.s1);
    xmax = floor_div(l - g.md, g.s1);
    ymin = ceil_div_signed(m - kr2 - g.mdy, g.s1);
    ymax = floor_div(m - g.mdy, g.s1);
    any = xmax >= 0 && ymax >= 0 && xmin <= g.tw - 1 && ymin <= g.th - 1;
    xmin = max(0, xmin); xmax = min(g.tw - 1, xmax);
    ymin = max(0, ymin); ymax = min(g.th - 1, ymax);
  }
  if (any) {
    for (int dyi = 0; dyi < g.gh; ++dyi) {
      const int s2p = (dyi - g.ry) * g.s2;
      for (int dxi = 0; dxi < g.gw; ++dxi) {
        const int s2o = (dxi + g.xshift) * g.s2;
        if (SECOND) {
          xmin = ceil_div_signed(l - kr2 - g.md - s2o, g.s1);
          xmax = floor_div(l - g.md - s2o, g.s1);
          ymin = ceil_div_signed(m - kr2 - g.mdy - s2p, g.s1);
          ymax = floor_div(m - g.mdy - s2p, g.s1);
          if (!(xmax >= 0 && ymax >= 0 && xmin <= g.tw - 1 && ymin <= g.th - 1)) continue;
          xmin = max(0, xmin); xmax = min(g.tw - 1, xmax);
          ymin = max(0, ymin); ymax = min(g.th - 1, ymax);
        }
        const int py = SECOND ? m - s2p : m + s2p, px = SECOND ? l - s2o : l + s2o;
        float v[kGradCh];
#pragma unroll
        for (int cc = 0; cc < kGradCh; ++cc) {
          if (SUBT) {
            const bool ge = padded(p1[cc], py, px, g) >= padded(p2[cc], py, px, g);   // false with a NaN
            v[cc] = (ge != SECOND) ? 1.f : -1.f;
          } else {
            v[cc] = padded(SECOND ? p1[cc] : p2[cc], py, px, g);
          }
        }
        const float* gop = gt + (size_t)(dyi * g.gw + dxi) * g.th * g.tw;
        for (int y = ymin; y <= ymax; ++y)
          for (int x = xmin; x <= xmax; ++x) {
            const float t = __ldg(gop + (size_t)y * g.tw + x);
#pragma unroll
            for (int cc = 0; cc < kGradCh; ++cc) sum[cc] = __fmaf_rn(t, v[cc], sum[cc]);
          }
      }
    }
  }
#pragma unroll
  for (int cc = 0; cc < kGradCh; ++cc) {
    const int ch = cg * kGradCh + cc;
    if (ch < g.c) grad[((size_t)img * g.c + ch) * plane + (size_t)yy * g.w + xx] = __fdiv_rn(sum[cc], g.sumelems);
  }
}

// Validates the attributes and fills the geometry (DEMON_E_INVALID before any launch).
int make_geom(CorrGeom& g, bool one_d, int n, int c, int h, int w, int corr_type, int ks, int md, int s1, int s2, int pad, int single_dir) {
  DEMON_REQUIRE(corr_type == DEMON_CORR_MULT || corr_type == DEMON_CORR_SUBT, "correlation: corr_type must be DEMON_CORR_MULT or DEMON_CORR_SUBT (got %d)", corr_type);
  DEMON_REQUIRE(ks >= 1 && ks % 2 == 1, "Correlation cannot be done with even kernel_size (got %d)", ks);
  DEMON_REQUIRE(s1 >= 1 && s2 >= 1, "correlation: stride1 and stride2 must be >= 1 (got %d, %d)", s1, s2);
  DEMON_REQUIRE(md >= 0 && pad >= 0, "correlation: max_displacement and pad_size must be >= 0 (got %d, %d)", md, pad);
  DEMON_REQUIRE(single_dir >= -1 && single_dir <= 1, "correlation_1d: single_dir must be -1, 0 or 1 (got %d)", single_dir);
  DEMON_REQUIRE(n >= 0 && c >= 0 && h >= 0 && w >= 0, "correlation: negative size");
  const int kr = (ks - 1) / 2;
  g.n = n; g.c = c; g.h = h; g.w = w;
  g.ks = ks; g.md = md; g.s1 = s1; g.s2 = s2; g.pad = pad;
  g.pady = one_d ? 0 : pad;
  g.mdy = one_d ? 0 : md;
  // top size as the reference computes it: ceil in float (correlation.cc:62-77, correlation_1d_cuda.cu:485-505)
  g.tw = (int)std::ceil((float)(w + 2 * pad - 2 * (md + kr)) / (float)s1);
  g.th = one_d ? (int)std::ceil((float)(h - 2 * kr) / (float)s1) : (int)std::ceil((float)(h + 2 * pad - 2 * (md + kr)) / (float)s1);
  DEMON_REQUIRE(g.tw >= 1 && g.th >= 1, "Correlation cannot be done with current settings. Neighborhood and kernel don't fit in blob");
  const int R = md / s2;
  if (one_d) {
    g.gw = single_dir != 0 ? R + 1 : 2 * R + 1;
    g.gh = 1;
    g.xshift = single_dir == -1 ? -g.gw : (single_dir == 1 ? 0 : -R);
    g.ry = 0;
  } else {
    g.gw = g.gh = 2 * R + 1;
    g.xshift = -R;
    g.ry = R;
  }
  g.tc = g.gw * g.gh;
  g.sumelems = (float)(ks * ks * c);
  return DEMON_OK;
}

template <bool SUBT, int P>
int fwd_launch(const float* in1, const float* in2, float* out, const CorrGeom& g, cudaStream_t stream) {
  FwdPlan f;
  const int tile = 32 * P;
  f.nseg = ceil_div(g.tw, tile);
  f.colsA = (tile - 1) * g.s1 + g.ks;
  const int maxnch = SUBT ? g.c : ceil_div(g.c, 32);
  // displacement block: up to kFwdMaxWarps * kFwdD displacements, shrunk until one channel of one row fits the budget
  int ndx_cap = kFwdMaxWarps * kFwdD;
  for (;;) {
    f.ndxg = ceil_div(g.gw, ndx_cap);
    f.ndx = ceil_div(g.gw, f.ndxg);
    f.ndy = std::min(g.gh, std::max(1, kFwdMaxWarps * kFwdD / f.ndx));
    f.ndyg = ceil_div(g.gh, f.ndy);
    f.ndy = ceil_div(g.gh, f.ndyg);
    f.colsB = f.colsA + (f.ndx - 1) * g.s2;
    if ((size_t)(f.colsA + f.ndy * f.colsB) * sizeof(float) <= (size_t)kSmemBudget || ndx_cap == 1) break;
    ndx_cap = std::max(1, ndx_cap / 2);
  }
  const size_t per_ch_row = (size_t)(f.colsA + f.ndy * f.colsB) * sizeof(float);
  DEMON_REQUIRE(per_ch_row <= (size_t)kSmemBudget, "correlation: displacement window too wide for shared memory");
  const int chmax = std::max(1, maxnch);
  if ((size_t)g.ks * chmax * per_ch_row <= (size_t)kSmemBudget) { f.rows = g.ks; f.ch = chmax; }
  else { f.rows = 1; f.ch = std::max(1, std::min(chmax, (int)(kSmemBudget / per_ch_row))); }
  const int warps = ceil_div(f.ndx * f.ndy, kFwdD);
  const int64_t blocks = (int64_t)f.nseg * f.ndxg * f.ndyg * g.th * g.n;
  DEMON_REQUIRE(blocks < (1ll << 31), "correlation: output too large");
  const size_t smem = (size_t)f.rows * f.ch * per_ch_row;
  correlation_fwd_kernel<SUBT, P><<<(unsigned)blocks, warps * 32, smem, stream>>>(in1, in2, out, g, f);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

template <bool SUBT, bool SECOND>
int grad_launch(const float* in1, const float* in2, const float* gtop, float* grad, const CorrGeom& g, cudaStream_t stream) {
  const int nxseg = ceil_div(g.w, kGradThreads), ncg = ceil_div(g.c, kGradCh);
  const int64_t blocks = (int64_t)nxseg * ncg * g.h * g.n;
  DEMON_REQUIRE(blocks < (1ll << 31), "correlation_grad: input too large");
  correlation_grad_kernel<SUBT, SECOND><<<(unsigned)blocks, kGradThreads, 0, stream>>>(in1, in2, gtop, grad, g, nxseg, ncg);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int correlation_run(bool one_d, const float* in1, const float* in2, float* out, int n, int c, int h, int w, int corr_type, int ks, int md,
                    int s1, int s2, int pad, int single_dir, void* stream) {
  CorrGeom g;
  const int rc = make_geom(g, one_d, n, c, h, w, corr_type, ks, md, s1, s2, pad, single_dir);
  if (rc != DEMON_OK) return rc;
  if (n == 0) return DEMON_OK;
  DEMON_REQUIRE(in1 && in2 && out, "correlation: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const bool subt = corr_type == DEMON_CORR_SUBT;
  if (g.tw > 32) return subt ? fwd_launch<true, 2>(in1, in2, out, g, st) : fwd_launch<false, 2>(in1, in2, out, g, st);
  return subt ? fwd_launch<true, 1>(in1, in2, out, g, st) : fwd_launch<false, 1>(in1, in2, out, g, st);
}

int correlation_grad_run(bool one_d, const float* in1, const float* in2, const float* gradient, float* grad1, float* grad2, int n, int c, int h,
                         int w, int corr_type, int ks, int md, int s1, int s2, int pad, int single_dir, void* stream) {
  CorrGeom g;
  const int rc = make_geom(g, one_d, n, c, h, w, corr_type, ks, md, s1, s2, pad, single_dir);
  if (rc != DEMON_OK) return rc;
  if ((int64_t)n * c * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(in1 && in2 && gradient && grad1 && grad2, "correlation_grad: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int r;
  if (corr_type == DEMON_CORR_SUBT) {
    if ((r = grad_launch<true, false>(in1, in2, gradient, grad1, g, st)) != DEMON_OK) return r;
    return grad_launch<true, true>(in1, in2, gradient, grad2, g, st);
  }
  if ((r = grad_launch<false, false>(in1, in2, gradient, grad1, g, st)) != DEMON_OK) return r;
  return grad_launch<false, true>(in1, in2, gradient, grad2, g, st);
}

}  // namespace
}  // namespace demon

extern "C" {

int demon_correlation_f32(const float* input1, const float* input2, float* output, int n, int c, int h, int w, int corr_type,
                          int kernel_size, int max_displacement, int stride1, int stride2, int pad_size, int do_abs, void* stream) {
  (void)do_abs;   // the reference reads the attribute and never uses it
  return demon::correlation_run(false, input1, input2, output, n, c, h, w, corr_type, kernel_size, max_displacement, stride1, stride2,
                                pad_size, 0, stream);
}

int demon_correlation_grad_f32(const float* input1, const float* input2, const float* gradient, float* input1_grad, float* input2_grad,
                               int n, int c, int h, int w, int corr_type, int kernel_size, int max_displacement, int stride1,
                               int stride2, int pad_size, int do_abs, void* stream) {
  (void)do_abs;
  return demon::correlation_grad_run(false, input1, input2, gradient, input1_grad, input2_grad, n, c, h, w, corr_type, kernel_size,
                                     max_displacement, stride1, stride2, pad_size, 0, stream);
}

int demon_correlation_1d_f32(const float* input1, const float* input2, float* output, int n, int c, int h, int w, int corr_type,
                             int kernel_size, int max_displacement, int stride1, int stride2, int pad_size, int do_abs, int single_dir,
                             void* stream) {
  (void)do_abs;
  return demon::correlation_run(true, input1, input2, output, n, c, h, w, corr_type, kernel_size, max_displacement, stride1, stride2,
                                pad_size, single_dir, stream);
}

int demon_correlation_1d_grad_f32(const float* input1, const float* input2, const float* gradient, float* input1_grad,
                                  float* input2_grad, int n, int c, int h, int w, int corr_type, int kernel_size, int max_displacement,
                                  int stride1, int stride2, int pad_size, int do_abs, int single_dir, void* stream) {
  (void)do_abs;
  return demon::correlation_grad_run(true, input1, input2, gradient, input1_grad, input2_grad, n, c, h, w, corr_type, kernel_size,
                                     max_displacement, stride1, stride2, pad_size, single_dir, stream);
}

}  // extern "C"
