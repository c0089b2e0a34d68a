// The training losses of DeMoN v2 (python/depthmotionnet/v2/losses.py) and their gradients on the device.
//
// Three pieces:
//   * ground truth (prepare_ground_truth_tensors, losses.py:312-356): the 5-level median chain through the standalone
//     median op, then ONE kernel for every derived field -- depth_to_flow at levels 0, 2 and 5, depth_to_normals at levels
//     0 and 2, and the three 5-delta SIG stacks.  Each pixel runs the same device functions as the standalone ops
//     (d2f_camera / d2f_pixel, d2n_pixel, sig_term of geometry.cuh), so every output is bit for bit their composition.  The
//     flow SIG recomputes the flow of its neighbours instead of reading the flow back.
//   * losses: a table of terms (demon_loss_term) evaluated by one partial-sum launch and one fold launch.
//       L2   pointwise_l2_loss (losses.py:32-53): t = sqrt_rn(sum_c d_c^2 + eps), d_c = replace_nonfinite(pr_c - gt_c),
//            channels summed in ascending order, mean over n*h*w pixels;
//       SIG  pointwise_l2_loss of the prediction's 10-channel SIG stack (deltas 1, 2, 4, 8, 16, computed on the fly from a
//            shared-memory tile with a 16-pixel halo, never stored) against a ground-truth stack, or against the SIG of a
//            ground-truth plane taken on the fly as well (the confidence SIG, losses.py:182-188);
//       L1   l1_loss (losses.py:23-29): sum of sqrt_rn(x^2 + eps), x = pr - gt.
//     Every term also yields its epsilon-0 mean (the *_unscaled summaries).  Sums are double: per-thread partials in a
//     fixed stride order, a fixed shuffle tree, one slot per CTA, slots folded by one warp in a fixed order.  The slot
//     count depends on the shape only, so the bits do too.  The mean is rounded once to T, then multiplied by the weight.
//   * gradients of each term's weighted output: L2 w*g*d_c/(M*t) (0 where d_c is not finite), L1 w*g*x/sqrt(x^2+eps), SIG
//     the same per SIG channel (a scratch plane stack U), gathered through each delta's SIG derivative like
//     ScaleInvariantGradientGrad.  Terms on one prediction write, then add, in table order: deterministic.
//
// Nothing here allocates or synchronises; scratch comes from the caller (demon_loss_workspace_bytes,
// demon_loss_ground_truth_workspace_bytes).
#include "geometry.cuh"

namespace demon {
namespace {

constexpr int kLossThreads = 256;
constexpr int kMaxLossSlots = 264;   // two CTAs per SM
constexpr int kMaxTerms = 8;
constexpr int kSigDeltas = 5;        // deltas 1, 2, 4, 8, 16 (losses.py:173,234,291,339)
constexpr int kSigChannels = 2 * kSigDeltas;
constexpr int kHalo = 16;
constexpr int kTileW = 64, kTileH = 16;

__device__ __forceinline__ float sqrt_rn(float x) { return __fsqrt_rn(x); }
__device__ __forceinline__ double sqrt_rn(double x) { return __dsqrt_rn(x); }
template <class T>
__device__ __forceinline__ T nonfinite_to_zero(T x) { return isfinite(x) ? x : (T)0; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <class T>
struct Term {
  int kind, c, h, w, gt_plane, accumulate;
  int64_t n;
  const T* pr;
  const T* gt;
  T eps, sig_eps, gt_sig_eps, weight;
  const T* weight_dev;
  T* out;
  T* out0;
  T* terms;
  const T* grad_out;
  T* grad;
  int slot0, nslots;   // this term's partial slots [slot0, slot0 + nslots)
  int64_t count;       // the mean's divisor (L1: 1, a sum)
};

template <class T>
struct Terms {
  Term<T> t[kMaxTerms];
  int num;
};

template <class T>
__device__ __forceinline__ T term_weight(const Term<T>& t) { return t.weight_dev ? __ldg(t.weight_dev) : t.weight; }

int64_t sig_tiles(int64_t n, int h, int w) { return n * ceil_div(w, kTileW) * ceil_div(h, kTileH); }

int slots_of(const demon_loss_term& t) {
  int64_t s = 1;
  if (t.kind == DEMON_LOSS_L2) s = ceil_div64(t.n * t.h * t.w, 4 * kLossThreads);
  else if (t.kind == DEMON_LOSS_SIG) s = sig_tiles(t.n, t.h, t.w);
  return (int)(s < 1 ? 1 : (s > kMaxLossSlots ? kMaxLossSlots : s));
}

// The SIG stack of one pixel of a tile: channels (2i, 2i+1) = (x, y) of delta 2^i with weight 1, one delta per call
// (losses.py:76-79: gx = 0 + term, as the single-delta op computes it).
template <class T>
__device__ __forceinline__ void sig_stack_tile(T s[kSigChannels], const T (*tile)[kTileW + kHalo], int lx, int ly, int x, int y, int H, int W, T eps) {
  const T v0 = tile[ly][lx];
#pragma unroll
  for (int i = 0; i < kSigDeltas; ++i) {
    const int d = 1 << i;
    const T vx = (x + d < W) ? tile[ly][lx + d] : v0;
    const T vy = (y + d < H) ? tile[ly + d][lx] : v0;
    s[2 * i] = fadd((T)0, sig_term(v0, vx, (T)1, eps));
    s[2 * i + 1] = fadd((T)0, sig_term(v0, vy, (T)1, eps));
  }
}

// The SIG term's tiles [kTileH][kTileW] of plane p, tile index ti = (p * tiles_y + ty) * tiles_x + tx, strided by `stride`.
// WRITE_U false: accumulate t (eps) and t (eps 0) into ae / a0.  WRITE_U true: write U = gs * d_c / (M * t) (0 where d_c
// is not finite) as the [n][10][h][w] stack.
template <class T, bool WRITE_U>
__device__ void sig_tiles_run(const Term<T>& t, int64_t first, int64_t stride, T (*tile)[kTileH + kHalo][kTileW + kHalo], double& ae,
                              double& a0, T* __restrict__ U, T gs) {
  const int H = t.h, W = t.w;
  const int tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
  const int64_t ntiles = t.n * tiles_x * tiles_y;
  const int64_t hw = (int64_t)H * W;
  const T count = (T)t.count;
  const int lx = threadIdx.x % kTileW, ly0 = threadIdx.x / kTileW;
  for (int64_t ti = first; ti < ntiles; ti += stride) {
    const int64_t plane = ti / (tiles_x * tiles_y);
    const int r = (int)(ti - plane * tiles_x * tiles_y);
    const int y0 = (r / tiles_x) * kTileH, x0 = (r % tiles_x) * kTileW;
    const T* pp = t.pr + plane * hw;
    const T* gp = t.gt_plane ? t.gt + plane * hw : nullptr;
    __syncthreads();   // the previous tile is consumed
    for (int j = threadIdx.x; j < (kTileH + kHalo) * (kTileW + kHalo); j += kLossThreads) {
      const int jy = j / (kTileW + kHalo), jx = j - jy * (kTileW + kHalo);
      const int gy = y0 + jy, gx = x0 + jx;
      const bool in = gy < H && gx < W;
      tile[0][jy][jx] = in ? __ldg(pp + (int64_t)gy * W + gx) : (T)0;
      if (gp) tile[1][jy][jx] = in ? __ldg(gp + (int64_t)gy * W + gx) : (T)0;
    }
    __syncthreads();
#pragma unroll 1
    for (int k = 0; k < kTileH / (kLossThreads / kTileW); ++k) {
      const int ly = ly0 + k * (kLossThreads / kTileW);
      const int x = x0 + lx, y = y0 + ly;
      if (x >= W || y >= H) continue;
      const int64_t pix = (int64_t)y * W + x;
      T ps[kSigChannels], gs_[kSigChannels];
      sig_stack_tile(ps, tile[0], lx, ly, x, y, H, W, t.sig_eps);
      if (gp) {
        sig_stack_tile(gs_, tile[1], lx, ly, x, y, H, W, t.gt_sig_eps);
      } else {
        const T* g = t.gt + plane * kSigChannels * hw + pix;
#pragma unroll
        for (int c = 0; c < kSigChannels; ++c) gs_[c] = __ldg(g + c * hw);
      }
      T d[kSigChannels];
      T s = 0;
#pragma unroll
      for (int c = 0; c < kSigChannels; ++c) {
        d[c] = fsub(ps[c], gs_[c]);
        const T e = nonfinite_to_zero(d[c]);
        s = fadd(s, fmul(e, e));
      }
      const T te = sqrt_rn(fadd(s, t.eps));
      if (!WRITE_U) {
        ae += (double)te;
        a0 += (double)sqrt_rn(s);
      } else {
        const T den = fmul(count, te);
        T* u = U + plane * kSigChannels * hw + pix;
#pragma unroll
        for (int c = 0; c < kSigChannels; ++c) u[c * hw] = isfinite(d[c]) ? fdiv(fmul(gs, d[c]), den) : (T)0;
      }
    }
  }
}

// one CTA per partial slot; partial[slot][2] = (sum of t, sum of t with eps 0)
template <class T>
__global__ void __launch_bounds__(kLossThreads) loss_partial_kernel(const Terms<T> tt, double* __restrict__ partial) {
  __shared__ T tile[2][kTileH + kHalo][kTileW + kHalo];
  __shared__ double red[kLossThreads / 32][2];
  const int slot = blockIdx.x;
  int k = 0;
  while (k + 1 < tt.num && slot >= tt.t[k + 1].slot0) ++k;
  const Term<T>& t = tt.t[k];
  const int local = slot - t.slot0;
  double ae = 0.0, a0 = 0.0;
  if (t.kind == DEMON_LOSS_SIG) {
    sig_tiles_run<T, false>(t, local, t.nslots, tile, ae, a0, nullptr, (T)0);
  } else if (t.kind == DEMON_LOSS_L2) {
    const int64_t hw = (int64_t)t.h * t.w, m = t.n * hw;
    for (int64_t i = (int64_t)local * kLossThreads + threadIdx.x; i < m; i += (int64_t)t.nslots * kLossThreads) {
      const int64_t sample = i / hw, p = i - sample * hw;
      const T* a = t.pr + sample * t.c * hw + p;
      const T* b = t.gt + sample * t.c * hw + p;
      T s = 0;
      for (int c = 0; c < t.c; ++c) {
        const T d = nonfinite_to_zero(fsub(__ldg(a + c * hw), __ldg(b + c * hw)));
        s = fadd(s, fmul(d, d));
      }
      const T te = sqrt_rn(fadd(s, t.eps));
      if (t.terms) t.terms[i] = te;
      ae += (double)te;
      a0 += (double)sqrt_rn(s);
    }
  } else {   // L1: x = pr - gt, no replace_nonfinite (losses.py:29)
    const int64_t m = t.n * t.c;
    for (int64_t i = threadIdx.x; i < m; i += kLossThreads) {
      const T x = t.gt ? fsub(__ldg(t.pr + i), __ldg(t.gt + i)) : __ldg(t.pr + i);
      const T x2 = fmul(x, x);
      ae += (double)sqrt_rn(fadd(x2, t.eps));
      a0 += (double)sqrt_rn(x2);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ae = warp_sum(ae);
  a0 = warp_sum(a0);
  if (lane == 0) { red[warp][0] = ae; red[warp][1] = a0; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double v = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) v += red[w][threadIdx.x];
    partial[2 * slot + threadIdx.x] = v;
  }
}

// one warp per term: the slots in a fixed order, rounded once to T, then weighted
template <class T>
__global__ void loss_fold_kernel(const Terms<T> tt, const double* __restrict__ partial) {
  const Term<T>& t = tt.t[blockIdx.x];
  const int lane = threadIdx.x;
  double se = 0.0, s0 = 0.0;
  for (int s = lane; s < t.nslots; s += 32) {
    se += partial[2 * (t.slot0 + s)];
    s0 += partial[2 * (t.slot0 + s) + 1];
  }
  se = warp_sum(se);
  s0 = warp_sum(s0);
  if (lane == 0) {
    const T mean = (T)(se / (double)t.count);
    if (t.out) *t.out = fmul(term_weight(t), mean);
    if (t.out0) *t.out0 = (T)(s0 / (double)t.count);
  }
}

// the upstream scale g * w of a term's gradient
template <class T>
__device__ __forceinline__ T grad_scale(const Term<T>& t) {
  const T g = t.grad_out ? __ldg(t.grad_out) : (T)0;
  return fmul(g, term_weight(t));
}

template <class T>
__device__ __forceinline__ void store_grad(T* p, T v, bool accumulate) { *p = accumulate ? fadd(*p, v) : v; }

// L2 and L1 gradients: thread = one pixel (L2) or one element (L1)
template <class T>
__global__ void __launch_bounds__(kLossThreads) pointwise_grad_kernel(const Term<T> t) {
  const T gs = grad_scale(t);
  const bool acc = t.accumulate != 0;
  if (t.kind == DEMON_LOSS_L1) {
    const int64_t m = t.n * t.c;
    for (int64_t i = (int64_t)blockIdx.x * kLossThreads + threadIdx.x; i < m; i += (int64_t)gridDim.x * kLossThreads) {
      const T x = t.gt ? fsub(__ldg(t.pr + i), __ldg(t.gt + i)) : __ldg(t.pr + i);
      store_grad(t.grad + i, fdiv(fmul(gs, x), sqrt_rn(fadd(fmul(x, x), t.eps))), acc);
    }
    return;
  }
  const int64_t hw = (int64_t)t.h * t.w, m = t.n * hw;
  const T count = (T)t.count;
  for (int64_t i = (int64_t)blockIdx.x * kLossThreads + threadIdx.x; i < m; i += (int64_t)gridDim.x * kLossThreads) {
    const int64_t sample = i / hw, p = i - sample * hw;
    const int64_t base = sample * t.c * hw + p;
    T s = 0;
    for (int c = 0; c < t.c; ++c) {
      const T d = nonfinite_to_zero(fsub(__ldg(t.pr + base + c * hw), __ldg(t.gt + base + c * hw)));
      s = fadd(s, fmul(d, d));
    }
    const T den = fmul(count, sqrt_rn(fadd(s, t.eps)));
    for (int c = 0; c < t.c; ++c) {
      const T d = fsub(__ldg(t.pr + base + c * hw), __ldg(t.gt + base + c * hw));
      store_grad(t.grad + base + c * hw, isfinite(d) ? fdiv(fmul(gs, d), den) : (T)0, acc);
    }
  }
}

template <class T>
__global__ void __launch_bounds__(kLossThreads) sig_u_kernel(const Term<T> t, T* __restrict__ U) {
  __shared__ T tile[2][kTileH + kHalo][kTileW + kHalo];
  double unused0 = 0.0, unused1 = 0.0;
  sig_tiles_run<T, true>(t, blockIdx.x, gridDim.x, tile, unused0, unused1, U, grad_scale(t));
}

// U [z][10][h][w] pushed through each delta's SIG derivative, summed over the deltas (gather form of
// ScaleInvariantGradientGrad, training_ops.cu sig_grad_kernel, with one gradient pair per delta); thread = one input pixel
template <class T>
__global__ void __launch_bounds__(128) sig_gather_kernel(const T* __restrict__ in, const T* __restrict__ U, T* __restrict__ out, int H, int W,
                                                        T eps, bool accumulate) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int64_t z = blockIdx.z;
  if (x >= W) return;
  const size_t hw = (size_t)H * W;
  const T* p = in + z * hw;
  const size_t i0 = (size_t)y * W + x;
  const T v0 = __ldg(p + i0);
  T diff = 0;
  if (isfinite(v0)) {
#pragma unroll
    for (int c = 0; c < kSigDeltas; ++c) {
      const int d = 1 << c;
      const T* gx = U + (z * kSigChannels + 2 * c) * hw;
      const T* gy = gx + hw;
      T tmp = 0;
      if (x + d < W) {
        const T vx = __ldg(p + i0 + d);
        if (isfinite(vx)) tmp = fadd(tmp, fmul(sig_dcenter(v0, vx, eps), __ldg(gx + i0)));
      }
      if (x - d >= 0) {
        const T vx = __ldg(p + i0 - d);
        if (isfinite(vx)) tmp = fadd(tmp, fmul(sig_dneighbour(vx, v0, eps), __ldg(gx + i0 - d)));
      }
      if (y + d < H) {
        const T vy = __ldg(p + i0 + (size_t)d * W);
        if (isfinite(vy)) tmp = fadd(tmp, fmul(sig_dcenter(v0, vy, eps), __ldg(gy + i0)));
      }
      if (y - d >= 0) {
        const T vy = __ldg(p + i0 - (size_t)d * W);
        if (isfinite(vy)) tmp = fadd(tmp, fmul(sig_dneighbour(vy, v0, eps), __ldg(gy + i0 - (size_t)d * W)));
      }
      diff = fadd(diff, tmp);
    }
  }
  if (!isfinite(diff)) diff = 0;
  store_grad(out + z * hw + i0, diff, accumulate);
}

// exp(-scale * |pr - gt|): the product in T, exp in double, rounded once (losses.py:360-373)
template <class T>
__global__ void __launch_bounds__(256) confidence_kernel(const T* __restrict__ pr, const T* __restrict__ gt, T* __restrict__ out, int64_t size,
                                                        T neg_scale) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < size; i += (int64_t)gridDim.x * 256)
    out[i] = (T)exp((double)fmul(neg_scale, tabs(fsub(__ldg(pr + i), __ldg(gt + i)))));
}

// ---- ground truth ---------------------------------------------------------------------------------------------------------
template <class T>
struct GtLevel {
  const T* depth;    // [n][h][w]
  T* flow;           // [n][2][h][w]
  T* normal;         // [n][3][h][w] or null
  T* depth_sig;      // [n][10][h][w] or null
  T* flow_sig;       // [2n][10][h][w] or null
  int h, w, ctas;    // ctas per sample
};

template <class T>
struct GtArgs {
  GtLevel<T> lv[3];
  const T* intrinsics;
  const T* rotation;
  const T* translation;
  int n;
  T sig_eps;
};

template <class T>
__device__ __forceinline__ void gt_sig_plane(T* __restrict__ out, const T* __restrict__ plane, int x, int y, int H, int W, size_t hw, T eps) {
  const size_t i0 = (size_t)y * W + x;
  const T v0 = __ldg(plane + i0);
#pragma unroll
  for (int i = 0; i < kSigDeltas; ++i) {
    const int d = 1 << i;
    const T vx = (x + d < W) ? __ldg(plane + i0 + d) : v0;
    const T vy = (y + d < H) ? __ldg(plane + i0 + (size_t)d * W) : v0;
    out[(2 * i) * hw + i0] = fadd((T)0, sig_term(v0, vx, (T)1, eps));
    out[(2 * i + 1) * hw + i0] = fadd((T)0, sig_term(v0, vy, (T)1, eps));
  }
}

// blockIdx.x enumerates (level, sample, chunk of 256 pixels); thread 0 sets up the sample's camera at that level's size
template <class T>
__global__ void __launch_bounds__(256) gt_fields_kernel(const GtArgs<T> a) {
  __shared__ D2FCamera<T> cam;
  int b = blockIdx.x, l = 0;
  while (l < 2 && b >= a.n * a.lv[l].ctas) { b -= a.n * a.lv[l].ctas; ++l; }
  const GtLevel<T>& L = a.lv[l];
  const int n = b / L.ctas, chunk = b - n * L.ctas;
  if (threadIdx.x == 0)
    d2f_camera(cam, a.intrinsics + 4 * n, a.rotation + 3 * n, a.translation + 3 * n, DEMON_ROT_ANGLEAXIS3, L.w, L.h);
  __syncthreads();
  const int H = L.h, W = L.w;
  const size_t hw = (size_t)H * W;
  const int i = chunk * 256 + threadIdx.x;
  if (i >= (int)hw) return;
  const int y = i / W, x = i - y * W;
  const T* dm = L.depth + (size_t)n * hw;
  T fx, fy;
  d2f_pixel(fx, fy, __ldg(dm + i), x, y, cam, true, true);   // losses.py:332-334: inverse_depth, normalize_flow
  L.flow[(size_t)n * 2 * hw + i] = fx;
  L.flow[(size_t)n * 2 * hw + hw + i] = fy;
  if (L.normal) {
    T nrm[3];
    d2n_pixel(nrm, dm, a.intrinsics + 4 * n, x, y, H, W, true);
    T* o = L.normal + (size_t)n * 3 * hw + i;
    o[0] = nrm[0]; o[hw] = nrm[1]; o[2 * hw] = nrm[2];
  }
  if (L.depth_sig) gt_sig_plane(L.depth_sig + (size_t)n * kSigChannels * hw, dm, x, y, H, W, hw, a.sig_eps);
  if (L.flow_sig) {
    // the flow of the neighbours at +delta, recomputed from their depth by the same d2f_pixel
    T* su = L.flow_sig + (size_t)(2 * n) * kSigChannels * hw + i;
    T* sv = su + kSigChannels * hw;
#pragma unroll 1
    for (int k = 0; k < kSigDeltas; ++k) {
      const int d = 1 << k;
      T ux = fx, vx = fy, uy = fx, vy = fy;
      if (x + d < W) d2f_pixel(ux, vx, __ldg(dm + i + d), x + d, y, cam, true, true);
      if (y + d < H) d2f_pixel(uy, vy, __ldg(dm + i + (size_t)d * W), x, y + d, cam, true, true);
      su[(2 * k) * hw] = fadd((T)0, sig_term(fx, ux, (T)1, a.sig_eps));
      su[(2 * k + 1) * hw] = fadd((T)0, sig_term(fx, uy, (T)1, a.sig_eps));
      sv[(2 * k) * hw] = fadd((T)0, sig_term(fy, vx, (T)1, a.sig_eps));
      sv[(2 * k + 1) * hw] = fadd((T)0, sig_term(fy, vy, (T)1, a.sig_eps));
    }
  }
}

// ---- launchers ------------------------------------------------------------------------------------------------------------
int check_term(const demon_loss_term& t, int i) {
  DEMON_REQUIRE(t.kind == DEMON_LOSS_L2 || t.kind == DEMON_LOSS_SIG || t.kind == DEMON_LOSS_L1, "loss term %d: unknown kind %d", i, t.kind);
  DEMON_REQUIRE(t.n >= 1 && t.c >= 1, "loss term %d: n and c must be >= 1 (got %lld, %d)", i, (long long)t.n, t.c);
  DEMON_REQUIRE(t.kind == DEMON_LOSS_L1 || (t.h >= 1 && t.w >= 1), "loss term %d: empty plane %dx%d", i, t.h, t.w);
  DEMON_REQUIRE(t.pr && (t.gt || t.kind == DEMON_LOSS_L1), "loss term %d: null pointer", i);
  DEMON_REQUIRE(t.kind != DEMON_LOSS_SIG || t.n <= 65535, "loss term %d: a SIG term takes at most 65535 planes (got %lld)", i, (long long)t.n);
  DEMON_REQUIRE(t.kind != DEMON_LOSS_SIG || t.h <= 65535, "loss term %d: h must be <= 65535 (got %d)", i, t.h);
  return DEMON_OK;
}

template <class T>
int make_terms(Terms<T>& tt, const demon_loss_term* terms, int num, int* total_slots) {
  DEMON_REQUIRE(num >= 1 && num <= kMaxTerms, "loss: 1 to %d terms (got %d)", kMaxTerms, num);
  DEMON_REQUIRE(terms, "loss: null term table");
  int slot = 0;
  tt.num = num;
  for (int i = 0; i < num; ++i) {
    const demon_loss_term& s = terms[i];
    const int rc = check_term(s, i);
    if (rc != DEMON_OK) return rc;
    Term<T>& t = tt.t[i];
    t.kind = s.kind; t.c = s.c; t.h = s.h; t.w = s.w; t.gt_plane = s.gt_plane; t.accumulate = s.accumulate; t.n = s.n;
    t.pr = static_cast<const T*>(s.pr); t.gt = static_cast<const T*>(s.gt);
    t.eps = (T)s.eps; t.sig_eps = (T)s.sig_eps; t.gt_sig_eps = (T)s.gt_sig_eps; t.weight = (T)s.weight;
    t.weight_dev = static_cast<const T*>(s.weight_dev);
    t.out = static_cast<T*>(s.out); t.out0 = static_cast<T*>(s.out0); t.terms = static_cast<T*>(s.terms);
    t.grad_out = static_cast<const T*>(s.grad_out); t.grad = static_cast<T*>(s.grad);
    t.slot0 = slot;
    t.nslots = slots_of(s);
    t.count = s.kind == DEMON_LOSS_L1 ? 1 : s.n * s.h * s.w;
    slot += t.nslots;
  }
  for (int i = num; i < kMaxTerms; ++i) tt.t[i] = tt.t[0];
  *total_slots = slot;
  return DEMON_OK;
}

int64_t partial_bytes(int slots) { return ((int64_t)slots * 2 * (int64_t)sizeof(double) + 255) / 256 * 256; }

template <class T>
int loss_forward(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  Terms<T> tt;
  int slots = 0;
  const int rc = make_terms(tt, terms, num, &slots);
  if (rc != DEMON_OK) return rc;
  DEMON_REQUIRE(ws && ws_bytes >= partial_bytes(slots), "loss_forward: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
                (long long)partial_bytes(slots));
  cudaStream_t s = (cudaStream_t)stream;
  double* partial = static_cast<double*>(ws);
  loss_partial_kernel<T><<<slots, kLossThreads, 0, s>>>(tt, partial);
  DEMON_LAUNCH_CHECK();
  loss_fold_kernel<T><<<num, 32, 0, s>>>(tt, partial);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

template <class T>
int loss_backward(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  Terms<T> tt;
  int slots = 0;
  const int rc = make_terms(tt, terms, num, &slots);
  if (rc != DEMON_OK) return rc;
  // every SIG term's scratch is checked before the first launch, so a refused call writes no gradient
  for (int i = 0; i < num; ++i) {
    const Term<T>& t = tt.t[i];
    if (!t.grad || t.kind != DEMON_LOSS_SIG) continue;
    const int64_t need = t.n * kSigChannels * t.h * t.w * (int64_t)sizeof(T);
    DEMON_REQUIRE(ws && ws_bytes >= need, "loss_backward: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
  }
  cudaStream_t s = (cudaStream_t)stream;
  for (int i = 0; i < num; ++i) {
    const Term<T>& t = tt.t[i];
    if (!t.grad) continue;
    if (t.kind == DEMON_LOSS_SIG) {
      T* U = static_cast<T*>(ws);
      const int64_t tiles = sig_tiles(t.n, t.h, t.w);
      sig_u_kernel<T><<<(int)(tiles < 132 * 8 ? tiles : 132 * 8), kLossThreads, 0, s>>>(t, U);
      DEMON_LAUNCH_CHECK();
      sig_gather_kernel<T><<<dim3(ceil_div(t.w, 128), t.h, (unsigned)t.n), 128, 0, s>>>(t.pr, U, t.grad, t.h, t.w, t.sig_eps, t.accumulate != 0);
      DEMON_LAUNCH_CHECK();
    } else {
      const int64_t m = t.kind == DEMON_LOSS_L1 ? t.n * t.c : t.n * t.h * t.w;
      int64_t blocks = ceil_div64(m, kLossThreads);
      if (blocks > 132 * 8) blocks = 132 * 8;
      pointwise_grad_kernel<T><<<(int)blocks, kLossThreads, 0, s>>>(t);
      DEMON_LAUNCH_CHECK();
    }
  }
  return DEMON_OK;
}

template <class T>
int confidence_launch(const T* pr, const T* gt, T* out, int64_t size, double scale, void* stream) {
  DEMON_REQUIRE(size >= 0, "confidence_map: negative size");
  if (size == 0) return DEMON_OK;
  DEMON_REQUIRE(pr && gt && out, "confidence_map: null pointer");
  int64_t blocks = ceil_div64(size, 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  confidence_kernel<T><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(pr, gt, out, size, (T)(-scale));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

inline int half_up(int v) { return (v + 1) / 2; }

int64_t gt_workspace_elems(int n, int h, int w) {   // median levels 1, 3, 4 and 5 (level 2 is an output)
  int64_t e = 0;
  int hh = h, ww = w;
  for (int l = 1; l <= 5; ++l) {
    hh = half_up(hh); ww = half_up(ww);
    if (l != 2) e += (int64_t)n * hh * ww;
  }
  return e;
}

template <class T>
int median_level(const T* in, T* out, int64_t z, int h, int w, void* stream);
template <>
int median_level<float>(const float* in, float* out, int64_t z, int h, int w, void* stream) { return demon_median3x3_downsample_f32(in, out, z, h, w, stream); }
template <>
int median_level<double>(const double* in, double* out, int64_t z, int h, int w, void* stream) { return demon_median3x3_downsample_f64(in, out, z, h, w, stream); }

template <class T>
int ground_truth(const T* depth, const T* intrinsics, const T* rotation, const T* translation, int n, int h, int w, T* depth2, T* flow0, T* flow2,
                 T* flow5, T* normal0, T* normal2, T* depth0_sig, T* depth2_sig, T* flow2_sig, void* ws, int64_t ws_bytes, void* stream) {
  DEMON_REQUIRE(n >= 1 && n <= 32767 && h >= 1 && w >= 1, "loss_ground_truth: bad size n=%d h=%d w=%d", n, h, w);
  DEMON_REQUIRE(h <= 65535, "loss_ground_truth: h must be <= 65535 (got %d)", h);
  DEMON_REQUIRE((int64_t)h * w < (1ll << 31), "loss_ground_truth: h*w must be < 2^31");
  DEMON_REQUIRE(depth && intrinsics && rotation && translation && depth2 && flow0 && flow2 && flow5 && normal0 && normal2 && depth0_sig &&
                depth2_sig && flow2_sig, "loss_ground_truth: null pointer");
  const int64_t need = gt_workspace_elems(n, h, w) * (int64_t)sizeof(T);
  DEMON_REQUIRE(ws && ws_bytes >= need, "loss_ground_truth: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
  int hs[6], wss[6];
  hs[0] = h; wss[0] = w;
  for (int l = 1; l <= 5; ++l) { hs[l] = half_up(hs[l - 1]); wss[l] = half_up(wss[l - 1]); }
  // recursive_median_downsample (v2/helpers.py:94-103) through the standalone op
  T* scratch = static_cast<T*>(ws);
  T* lv[6];
  lv[0] = const_cast<T*>(depth);
  for (int l = 1; l <= 5; ++l) {
    if (l == 2) { lv[l] = depth2; continue; }
    lv[l] = scratch;
    scratch += (int64_t)n * hs[l] * wss[l];
  }
  for (int l = 1; l <= 5; ++l) {
    const int rc = median_level<T>(lv[l - 1], lv[l], n, hs[l - 1], wss[l - 1], stream);
    if (rc != DEMON_OK) return rc;
  }
  GtArgs<T> a;
  const int lvl[3] = {0, 2, 5};
  for (int j = 0; j < 3; ++j) {
    GtLevel<T>& L = a.lv[j];
    const int l = lvl[j];
    L.depth = lv[l];
    L.h = hs[l]; L.w = wss[l];
    L.ctas = ceil_div(hs[l] * wss[l], 256);
    L.flow = j == 0 ? flow0 : (j == 1 ? flow2 : flow5);
    L.normal = j == 0 ? normal0 : (j == 1 ? normal2 : nullptr);
    L.depth_sig = j == 0 ? depth0_sig : (j == 1 ? depth2_sig : nullptr);
    L.flow_sig = j == 1 ? flow2_sig : nullptr;
  }
  a.intrinsics = intrinsics; a.rotation = rotation; a.translation = translation; a.n = n;
  a.sig_eps = (T)0.001f;   // a float attribute converted to T (scaleinvariantgradient.cc:109-113), losses.py:339
  const int64_t ctas = (int64_t)n * (a.lv[0].ctas + a.lv[1].ctas + a.lv[2].ctas);
  DEMON_REQUIRE(ctas < (1ll << 31), "loss_ground_truth: too large");
  gt_fields_kernel<T><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(a);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int64_t demon_loss_workspace_bytes(const demon_loss_term* terms, int num, int elem_size, int backward) {
  if (!terms || num < 1 || num > kMaxTerms || (elem_size != 4 && elem_size != 8)) return -1;
  int slots = 0;
  int64_t u = 0;
  for (int i = 0; i < num; ++i) {
    if (check_term(terms[i], i) != DEMON_OK) return -1;
    slots += slots_of(terms[i]);
    if (terms[i].kind == DEMON_LOSS_SIG) {
      const int64_t b = terms[i].n * kSigChannels * terms[i].h * terms[i].w * elem_size;
      if (b > u) u = b;
    }
  }
  return backward ? u : partial_bytes(slots);
}

int demon_loss_forward_f32(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  return loss_forward<float>(terms, num, ws, ws_bytes, stream);
}
int demon_loss_forward_f64(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  return loss_forward<double>(terms, num, ws, ws_bytes, stream);
}
int demon_loss_backward_f32(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  return loss_backward<float>(terms, num, ws, ws_bytes, stream);
}
int demon_loss_backward_f64(const demon_loss_term* terms, int num, void* ws, int64_t ws_bytes, void* stream) {
  return loss_backward<double>(terms, num, ws, ws_bytes, stream);
}
int demon_confidence_map_f32(const float* pr, const float* gt, float* out, int64_t size, double scale, void* stream) {
  return confidence_launch<float>(pr, gt, out, size, scale, stream);
}
int demon_confidence_map_f64(const double* pr, const double* gt, double* out, int64_t size, double scale, void* stream) {
  return confidence_launch<double>(pr, gt, out, size, scale, stream);
}

int64_t demon_loss_ground_truth_workspace_bytes(int n, int h, int w, int elem_size) {
  if (n < 1 || h < 1 || w < 1 || (elem_size != 4 && elem_size != 8)) return -1;
  return gt_workspace_elems(n, h, w) * elem_size;
}

int demon_loss_ground_truth_f32(const float* depth, const float* intrinsics, const float* rotation, const float* translation, int n, int h, int w,
                                float* depth2, float* flow0, float* flow2, float* flow5, float* normal0, float* normal2, float* depth0_sig,
                                float* depth2_sig, float* flow2_sig, void* ws, int64_t ws_bytes, void* stream) {
  return ground_truth<float>(depth, intrinsics, rotation, translation, n, h, w, depth2, flow0, flow2, flow5, normal0, normal2, depth0_sig,
                             depth2_sig, flow2_sig, ws, ws_bytes, stream);
}
int demon_loss_ground_truth_f64(const double* depth, const double* intrinsics, const double* rotation, const double* translation, int n, int h,
                                int w, double* depth2, double* flow0, double* flow2, double* flow5, double* normal0, double* normal2,
                                double* depth0_sig, double* depth2_sig, double* flow2_sig, void* ws, int64_t ws_bytes, void* stream) {
  return ground_truth<double>(depth, intrinsics, rotation, translation, n, h, w, depth2, flow0, flow2, flow5, normal0, normal2, depth0_sig,
                              depth2_sig, flow2_sig, ws, ws_bytes, stream);
}

}  // extern "C"
