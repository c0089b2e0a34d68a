// fp32 CUDA-core implicit-GEMM convolution (NHWC) for sm_90a.
//
// Role in the design: (1) the exact-fp32 path for the layers whose shapes do not suit tensor-core tiles
// (Cin in {4,6,7,8,9,24}, Cout in {1,2,4,7}, the dense layers) and (2) the on-device fp32 reference
// the tensor-core path is validated against in tests/.  Classic register-blocked SGEMM structure:
// 256 threads, a BM x BN output tile (BM*BN = 4096), 4x4 outputs per thread, BK = 16, the A tile
// gathered on the fly from the NHWC input (zero for padding taps), global loads of tile k+1 in flight
// while tile k is multiplied out of shared memory.
#include <cstdlib>

#include "conv.cuh"

namespace demon {

namespace {

constexpr int BK = 16;

template <int BM, int BN>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvProblem p) {
  static_assert(BM * BN == 4096, "256 threads x 16 outputs");
  pdl_launch_dependents();   // (common.cuh: the next kernel may start its prologue)
  pdl_wait();                // inputs come from the previous kernel; the output buffer may still be in use by it
  constexpr int ROWS_PER_THREAD_LD = BM / 64;   // A-tile float4 loads per thread
  constexpr int TXN = BN / 4;                   // thread columns
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];

  const int tid = threadIdx.x;
  const int M = p.B * p.Ho * p.Wo;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A-load bookkeeping: this thread always loads channel quad `kv` of rows tid/4 + 64*i ------
  const int kv = tid & 3;
  int row_n[ROWS_PER_THREAD_LD], row_y[ROWS_PER_THREAD_LD], row_x[ROWS_PER_THREAD_LD];
#pragma unroll
  for (int i = 0; i < ROWS_PER_THREAD_LD; ++i) {
    const int m = m0 + (tid >> 2) + 64 * i;
    if (m < M) {
      const int n = m / (p.Ho * p.Wo);
      const int r = m - n * (p.Ho * p.Wo);
      const int oy = r / p.Wo;
      row_n[i] = n; row_y[i] = oy * p.sy; row_x[i] = (r - oy * p.Wo) * p.sx;
    } else {
      row_n[i] = -1; row_y[i] = 0; row_x[i] = 0;
    }
  }
  // ---- B-load bookkeeping ---------------------------------------------------------------------
  const bool b_active = tid < 4 * BN;
  const int bk = tid / TXN;            // 0..15 when active
  const int bn = (tid % TXN) * 4;

  // The GEMM K axis is the flattened (tap, channel) index: k = tap * Cin + ci.  Cin is a multiple of 4, so every
  // float4 of a K chunk lies inside one tap -- layers with 4, 8 or 12 input channels fill their 16-wide chunks with
  // several taps instead of padding.  blockIdx.z selects a contiguous range of K chunks (split-K, dense layers).
  const int Ktot = p.ntaps * p.Cin;
  const int nk_all = (Ktot + BK - 1) / BK;
  const int per_split = (nk_all + gridDim.z - 1) / gridDim.z;
  const int it_begin = blockIdx.z * per_split;
  const int it_end = min(nk_all, it_begin + per_split);
  const int nk = max(0, it_end - it_begin);

  float4 a_reg[ROWS_PER_THREAD_LD];
  float4 b_reg;

  auto load_global = [&](int it) {
    const int k0 = (it_begin + it) * BK;
    const int ka = k0 + kv * 4;
    const int tap = ka / p.Cin;
    const int ci = ka - tap * p.Cin;
    const bool kvalid = ka < Ktot;
    const int dy = kvalid ? p.dy[tap] : 0, dx = kvalid ? p.dx[tap] : 0;
#pragma unroll
    for (int i = 0; i < ROWS_PER_THREAD_LD; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int iy = row_y[i] + dy, ix = row_x[i] + dx;
      if (row_n[i] >= 0 && kvalid && iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi)
        v = __ldg(reinterpret_cast<const float4*>(p.in + ((size_t)(row_n[i] * p.Hi + iy) * p.Wi + ix) * p.in_pitch + ci));
      a_reg[i] = v;
    }
    b_reg = make_float4(0.f, 0.f, 0.f, 0.f);
    if (b_active && k0 + bk < Ktot && n0 + bn < p.Cout_pad)
      b_reg = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)(k0 + bk) * p.Cout_pad + n0 + bn));
  };
  auto store_smem = [&]() {
#pragma unroll
    for (int i = 0; i < ROWS_PER_THREAD_LD; ++i) {
      const int r = (tid >> 2) + 64 * i;
      As[kv * 4 + 0][r] = a_reg[i].x;
      As[kv * 4 + 1][r] = a_reg[i].y;
      As[kv * 4 + 2][r] = a_reg[i].z;
      As[kv * 4 + 3][r] = a_reg[i].w;
    }
    if (b_active) *reinterpret_cast<float4*>(&Bs[bk][bn]) = b_reg;
  };

  const int tx = tid % TXN, ty = tid / TXN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  if (nk > 0) {
    load_global(0);
    store_smem();
  }
  __syncthreads();
  for (int it = 0; it < nk; ++it) {
    if (it + 1 < nk) load_global(it + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (it + 1 < nk) {
      store_smem();
      __syncthreads();
    }
  }

  // ---- epilogue: bias, leaky ReLU, per-sample scale on channel 0, write into the concat slice ----
  const int col = n0 + tx * 4;
  if (col >= p.Cout) return;
  if (p.partial != nullptr) {   // split-K: raw partial sums [z][M][Cout_pad], reduced by splitk_reduce_kernel
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + ty * 4 + i;
      if (m < M && col < p.Cout_pad)
        *reinterpret_cast<float4*>(p.partial + ((size_t)blockIdx.z * M + m) * p.Cout_pad + col) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
    return;
  }
  float bias[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) bias[j] = (col + j < p.Cout_pad) ? __ldg(p.bias + col + j) : 0.f;
  const bool vec = (col + 3 < p.Cout) && ((p.out_pitch & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int n = m / (p.Ho * p.Wo);
    const int r = m - n * (p.Ho * p.Wo);
    const int oy = r / p.Wo, ox = r - oy * p.Wo;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float x = acc[i][j] + bias[j];
      if (p.leaky) x = fmaxf(0.1f * x, x);
      v[j] = x;
    }
    if (p.scale != nullptr && col == 0) v[0] *= __ldg(p.scale + (size_t)n * p.scale_stride);
    float* o = p.out + ((size_t)(n * p.Hfull + oy * p.osy + p.ooy) * p.Wfull + ox * p.osx + p.oox) * p.out_pitch + col;
    if (vec) {
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (col + j < p.Cout) o[j] = v[j];
    }
  }
}

// Direct convolution for the prediction heads' last layers (Cout <= 4, Cin <= 32, e.g. 24 -> 4 and 16 -> 1, 3x3).  These
// layers have ~150 MACs per pixel and are bound by reading their input (64-128 B per pixel): LPP lanes share one output
// pixel, each owning a float4 of its channels, so that a warp load covers 32 / LPP adjacent pixels = 512 contiguous bytes
// (one thread per pixel touched 16 B of every 64-B pixel per instruction and ran at a tenth of the HBM rate); the taps'
// re-reads hit L1; the LPP partial sums are combined by shuffles in a fixed order.  Weights sit in shared memory.
// grid (ceil(Wo / (8 * 128 / LPP)), Ho, B).
constexpr int kSmallCoutGroups = 4;
template <int COUT, int LPP, int NT>   // NT: compile-time tap count (9 = 3x3) or 0 = run-time loop
__global__ void __launch_bounds__(128) conv_small_cout_kernel(const ConvProblem p) {
  pdl_launch_dependents();
  __shared__ __align__(16) float ws[kMaxTaps * 32 * COUT];
  const int nw = p.ntaps * p.Cin;
  for (int i = threadIdx.x; i < nw * COUT; i += 128) {
    const int k = i / COUT, co = i - k * COUT;
    ws[i] = (co < p.Cout) ? __ldg(p.w + (size_t)k * p.Cout_pad + co) : 0.f;
  }
  __syncthreads();
  pdl_wait();   // the weights above are constants; activations come from the previous kernel
  constexpr int PPB = 128 / LPP;
  const int pix = threadIdx.x / LPP, chunk = threadIdx.x % LPP;
  const int oy = blockIdx.y, n = blockIdx.z;
  for (int g = 0; g < kSmallCoutGroups; ++g) {   // the CTA's weights serve kSmallCoutGroups x PPB pixels of the row
    const int ox = (blockIdx.x * kSmallCoutGroups + g) * PPB + pix;
    const bool active = ox < p.Wo && chunk * 4 < p.Cin;
    float acc[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
    if (active && NT > 0) {
      // all taps' loads in flight before the first FMA (a tap outside the image contributes 0 * w)
      float4 v[NT > 0 ? NT : 1];
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int iy = oy * p.sy + p.dy[t], ix = ox * p.sx + p.dx[t];
        v[t] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi)
          v[t] = __ldg(reinterpret_cast<const float4*>(p.in + ((size_t)(n * p.Hi + iy) * p.Wi + ix) * p.in_pitch) + chunk);
      }
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const float* wt = ws + (size_t)(t * p.Cin + chunk * 4) * COUT;
        const float vv[4] = {v[t].x, v[t].y, v[t].z, v[t].w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int c = 0; c < COUT; ++c) acc[c] = fmaf(vv[j], wt[j * COUT + c], acc[c]);
      }
    } else if (active) {
      for (int t = 0; t < p.ntaps; ++t) {
        const int iy = oy * p.sy + p.dy[t], ix = ox * p.sx + p.dx[t];
        if (iy < 0 || iy >= p.Hi || ix < 0 || ix >= p.Wi) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(p.in + ((size_t)(n * p.Hi + iy) * p.Wi + ix) * p.in_pitch) + chunk);
        const float* wt = ws + (size_t)(t * p.Cin + chunk * 4) * COUT;
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int c = 0; c < COUT; ++c) acc[c] = fmaf(vv[j], wt[j * COUT + c], acc[c]);
      }
    }
#pragma unroll
    for (int off = LPP / 2; off >= 1; off >>= 1)
#pragma unroll
      for (int c = 0; c < COUT; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], off);
    if (chunk != 0 || ox >= p.Wo) continue;
    float* o = p.out + ((size_t)(n * p.Hfull + oy * p.osy + p.ooy) * p.Wfull + ox * p.osx + p.oox) * p.out_pitch;
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
      if (c < p.Cout) {
        float x = acc[c] + __ldg(p.bias + c);
        if (p.leaky) x = fmaxf(0.1f * x, x);
        if (c == 0 && p.scale != nullptr) x *= __ldg(p.scale + (size_t)n * p.scale_stride);
        o[c] = x;
      }
    }
  }
}

// One thread per output pixel: faster than lane sharing for the 24 -> 4 heads at 48x64 (0.036 vs 0.10 ms at batch 64, the
// shuffles and the 6-of-8 active lanes cost more than the uncoalesced loads), slower for 16 -> 1 at 192x256 (0.27 vs 0.16 ms)
template <int COUT>
__global__ void __launch_bounds__(128) conv_small_cout_pixel_kernel(const ConvProblem p) {
  pdl_launch_dependents();
  __shared__ float ws[kMaxTaps * 32 * COUT];
  const int nw = p.ntaps * p.Cin;
  for (int i = threadIdx.x; i < nw * COUT; i += 128) {
    const int k = i / COUT, co = i - k * COUT;
    ws[i] = (co < p.Cout) ? __ldg(p.w + (size_t)k * p.Cout_pad + co) : 0.f;
  }
  __syncthreads();
  pdl_wait();   // the weights above are constants; activations come from the previous kernel
  const int ox = blockIdx.x * 128 + threadIdx.x, oy = blockIdx.y, n = blockIdx.z;
  if (ox >= p.Wo) return;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  for (int t = 0; t < p.ntaps; ++t) {
    const int iy = oy * p.sy + p.dy[t], ix = ox * p.sx + p.dx[t];
    if (iy < 0 || iy >= p.Hi || ix < 0 || ix >= p.Wi) continue;
    const float4* src = reinterpret_cast<const float4*>(p.in + ((size_t)(n * p.Hi + iy) * p.Wi + ix) * p.in_pitch);
    const float* wt = ws + (size_t)t * p.Cin * COUT;
    for (int c4 = 0; c4 < p.Cin / 4; ++c4) {
      const float4 v = __ldg(src + c4);
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < COUT; ++c) acc[c] = fmaf(vv[j], wt[(c4 * 4 + j) * COUT + c], acc[c]);
    }
  }
  float* o = p.out + ((size_t)(n * p.Hfull + oy * p.osy + p.ooy) * p.Wfull + ox * p.osx + p.oox) * p.out_pitch;
#pragma unroll
  for (int c = 0; c < COUT; ++c) {
    if (c < p.Cout) {
      float x = acc[c] + __ldg(p.bias + c);
      if (p.leaky) x = fmaxf(0.1f * x, x);
      if (c == 0 && p.scale != nullptr) x *= __ldg(p.scale + (size_t)n * p.scale_stride);
      o[c] = x;
    }
  }
}

// out[m][c] = act(bias[c] + sum_z partial[z][m][c]); only used for 1x1 problems on 1x1 images (dense layers)
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const ConvProblem p, int ksplit, int M) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= M * p.Cout) return;
  const int m = i / p.Cout, c = i - m * p.Cout;
  float s = 0.f;
  for (int z = 0; z < ksplit; ++z) s += p.partial[((size_t)z * M + m) * p.Cout_pad + c];
  s += __ldg(p.bias + c);
  if (p.leaky) s = fmaxf(0.1f * s, s);
  if (p.scale != nullptr && c == 0) s *= __ldg(p.scale + (size_t)m * p.scale_stride);
  p.out[(size_t)m * p.out_pitch + c] = s;
}

}  // namespace

// every launch may start while its predecessor drains (common.cuh: launch_pdl); a failed launch is picked up by
// DEMON_LAUNCH_CHECK through cudaPeekAtLastError
#define SIMT_LAUNCH(kernel, grid, block, ...) (void)launch_pdl(kernel, dim3(grid), dim3(block), 0, stream, __VA_ARGS__)

int conv_simt_launch(const ConvProblem& p, cudaStream_t stream) {
  DEMON_REQUIRE(p.in && p.out && p.w && p.bias, "conv: null pointer");
  DEMON_REQUIRE((p.Cin & 3) == 0 && (p.in_pitch & 3) == 0 && (p.Cout_pad & 3) == 0, "conv: Cin (%d), in_pitch (%d), Cout_pad (%d) must be multiples of 4", p.Cin, p.in_pitch, p.Cout_pad);
  DEMON_REQUIRE((reinterpret_cast<uintptr_t>(p.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.w) & 15) == 0, "conv: in/w must be 16-byte aligned");
  DEMON_REQUIRE(p.ntaps >= 1 && p.ntaps <= kMaxTaps, "conv: ntaps %d", p.ntaps);
  const int64_t M = (int64_t)p.B * p.Ho * p.Wo;
  DEMON_REQUIRE(M < (1ll << 31), "conv: too many output pixels");
  if (M == 0 || p.Cout == 0) return DEMON_OK;
  if (p.Cout <= 4 && p.Cin <= 32 && p.ntaps > 1 && p.partial == nullptr && p.Ho <= 65535 && p.B <= 65535) {
    static const int pixel_mode = []() { const char* e = getenv("DEMON_SMALL_COUT_PIXEL"); return e ? atoi(e) : 2; }();   // 0: lane sharing everywhere, 1: pixel kernel everywhere, 2 (default, measured): lane sharing for Cout == 1 only
    if (pixel_mode == 1 || (pixel_mode == 2 && p.Cout > 1)) {
      dim3 g1(ceil_div(p.Wo, 128), p.Ho, p.B);
      if (p.Cout == 1) SIMT_LAUNCH((conv_small_cout_pixel_kernel<1>), g1, 128, p);
      else SIMT_LAUNCH((conv_small_cout_pixel_kernel<4>), g1, 128, p);
      DEMON_LAUNCH_CHECK();
      return DEMON_OK;
    }
    const int lpp = (p.Cin <= 16) ? 4 : 8;   // lanes per output pixel, one float4 of channels each
    dim3 grid(ceil_div(p.Wo, (128 / lpp) * kSmallCoutGroups), p.Ho, p.B);
    const bool nine = p.ntaps == 9;
    if (p.Cout == 1 && lpp == 4) { if (nine) SIMT_LAUNCH((conv_small_cout_kernel<1, 4, 9>), grid, 128, p); else SIMT_LAUNCH((conv_small_cout_kernel<1, 4, 0>), grid, 128, p); }
    else if (p.Cout == 1) { if (nine) SIMT_LAUNCH((conv_small_cout_kernel<1, 8, 9>), grid, 128, p); else SIMT_LAUNCH((conv_small_cout_kernel<1, 8, 0>), grid, 128, p); }
    else if (lpp == 4) { if (nine) SIMT_LAUNCH((conv_small_cout_kernel<4, 4, 9>), grid, 128, p); else SIMT_LAUNCH((conv_small_cout_kernel<4, 4, 0>), grid, 128, p); }
    else { if (nine) SIMT_LAUNCH((conv_small_cout_kernel<4, 8, 9>), grid, 128, p); else SIMT_LAUNCH((conv_small_cout_kernel<4, 8, 0>), grid, 128, p); }
    DEMON_LAUNCH_CHECK();
    return DEMON_OK;
  }
  const int ks = (p.partial != nullptr && p.ksplit > 1) ? p.ksplit : 1;
  if (ks > 1) DEMON_REQUIRE(p.Hi == 1 && p.Wi == 1 && p.Ho == 1 && p.Wo == 1, "conv: split-K is for dense layers only");
  ConvProblem q = p;
  if (ks == 1) q.partial = nullptr;
  // tile choice: widest N tile that the layer fills
  if (p.Cout > 32) {
    dim3 grid(ceil_div((int)M, 64), ceil_div(p.Cout, 64), ks);
    SIMT_LAUNCH((conv_simt_kernel<64, 64>), grid, 256, q);
  } else if (p.Cout > 16) {
    dim3 grid(ceil_div((int)M, 128), ceil_div(p.Cout, 32), ks);
    SIMT_LAUNCH((conv_simt_kernel<128, 32>), grid, 256, q);
  } else if (p.Cout > 8) {
    dim3 grid(ceil_div((int)M, 256), ceil_div(p.Cout, 16), ks);
    SIMT_LAUNCH((conv_simt_kernel<256, 16>), grid, 256, q);
  } else {
    dim3 grid(ceil_div((int)M, 512), ceil_div(p.Cout, 8), ks);
    SIMT_LAUNCH((conv_simt_kernel<512, 8>), grid, 256, q);
  }
  DEMON_LAUNCH_CHECK();
  if (ks > 1) {
    SIMT_LAUNCH(splitk_reduce_kernel, ceil_div((int)M * p.Cout, 256), 256, q, ks, (int)M);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

}  // namespace demon
