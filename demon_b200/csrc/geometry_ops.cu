// Standalone geometry ops of the DeMoN hot path (the lmbspecialops ops the network threads between
// its blocks) as HBM-roofline kernels for sm_90a.  All of them move a few bytes per pixel and do
// almost no arithmetic, so the design rules are: one thread per (vector of) output pixel(s), the W
// dimension on threadIdx.x so every warp reads and writes whole 128-byte lines, grids sized from the
// tensor (they are far larger than 132 SMs at the benchmark sizes), no shared memory except the
// per-sample camera.
#include <cstdlib>
#include "geometry.cuh"

namespace demon {

std::string& last_error_ref() {
  static thread_local std::string s;
  return s;
}
std::atomic<int64_t> g_launch_count{0};

bool pdl_enabled() {
  static const bool on = []() {
    const char* e = getenv("DEMON_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error_ref() = buf;
  return code;
}

// ---------------------------------------------------------------------------------------------
// warp2d  (replaces warp2d.cc:171-256 / warp2d_cuda.cu:31-115)
// grid (ceil(W/128), H, N), block 128: thread = one output pixel, loops over C like the reference,
// the displacement is read once per pixel, each channel's four taps are gathers (L1/L2 hits: the
// displacement field is smooth on the hot path).
// ---------------------------------------------------------------------------------------------
template <class T, bool CLAMP>
__global__ void __launch_bounds__(128) warp2d_kernel(const T* __restrict__ in, const T* __restrict__ disp,
                                                    T* __restrict__ out, int C, int H, int W,
                                                    bool normalized, T border_value) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int n = blockIdx.z;
  if (x >= W) return;
  const size_t hw = (size_t)H * W;
  const T* d = disp + (size_t)n * 2 * hw + (size_t)y * W + x;
  WarpTap<T> t = warp2d_tap<T>(x, y, __ldg(d), __ldg(d + hw), W, H, normalized);
  const T* src = in + (size_t)n * C * hw;
  T* dst = out + (size_t)n * C * hw + (size_t)y * W + x;
  // channels in chunks of four: the sixteen gathers of a chunk are in flight before the first blend
  constexpr int CH = 4;
  if (CLAMP) {
    const int x1i = (int)((unsigned)t.x0 + 1u), y1i = (int)((unsigned)t.y0 + 1u);
    const int x0 = clampi(t.x0, W), x1 = clampi(x1i, W), y0 = clampi(t.y0, H), y1 = clampi(y1i, H);
    const size_t o00 = (size_t)y0 * W + x0, o01 = (size_t)y0 * W + x1, o10 = (size_t)y1 * W + x0, o11 = (size_t)y1 * W + x1;
    for (int c0 = 0; c0 < C; c0 += CH) {
      T v[CH][4];
#pragma unroll
      for (int k = 0; k < CH; ++k)
        if (c0 + k < C) {
          const T* p = src + (size_t)(c0 + k) * hw;
          v[k][0] = __ldg(p + o00); v[k][1] = __ldg(p + o01); v[k][2] = __ldg(p + o10); v[k][3] = __ldg(p + o11);
        }
#pragma unroll
      for (int k = 0; k < CH; ++k)
        if (c0 + k < C) dst[(size_t)(c0 + k) * hw] = warp2d_blend(v[k][0], v[k][1], v[k][2], v[k][3], t);
    }
  } else {
    const bool valid = warp2d_valid(t.x0, t.y0, W, H);
    if (!valid) {
      for (int c = 0; c < C; ++c) dst[(size_t)c * hw] = border_value;
      return;
    }
    const T* p0 = src + (size_t)t.y0 * W + t.x0;
    for (int c0 = 0; c0 < C; c0 += CH) {
      T v[CH][4];
#pragma unroll
      for (int k = 0; k < CH; ++k)
        if (c0 + k < C) {
          const T* p = p0 + (size_t)(c0 + k) * hw;
          v[k][0] = __ldg(p); v[k][1] = __ldg(p + 1); v[k][2] = __ldg(p + W); v[k][3] = __ldg(p + W + 1);
        }
#pragma unroll
      for (int k = 0; k < CH; ++k)
        if (c0 + k < C) dst[(size_t)(c0 + k) * hw] = warp2d_blend(v[k][0], v[k][1], v[k][2], v[k][3], t);
    }
  }
}

// float fast path: FOUR pixels per thread.  The displacement rows are read as two float4, the results of every channel
// are stored as one float4, the index arithmetic is 32 bit (the launcher takes this path only while all tensors have
// fewer than 2^31 elements, W is a multiple of 4 and the base pointers are 16-byte aligned), and the sixteen gathers of
// a channel are in flight before the first blend.  Per-pixel arithmetic is the same sequence of IEEE operations as in
// warp2d_kernel (bit exact with the reference's CPU kernel, warp2d.cc:186-247).
template <bool CLAMP, int CU>   // CU channels per round: all their gathers (16 per channel) are in flight before the first blend
__global__ void __launch_bounds__(128) warp2d_v4_kernel(const float* __restrict__ in, const float* __restrict__ disp,
                                                       float* __restrict__ out, int C, int H, int W, bool normalized, float border_value) {
  const int x = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int y = blockIdx.y;
  const int n = blockIdx.z;
  if (x >= W) return;
  const int hw = H * W;
  const int row = y * W + x;
  const float* d = disp + n * 2 * hw + row;
  const float4 dx = __ldg(reinterpret_cast<const float4*>(d));
  const float4 dy = __ldg(reinterpret_cast<const float4*>(d + hw));
  const float vx[4] = {dx.x, dx.y, dx.z, dx.w}, vy[4] = {dy.x, dy.y, dy.z, dy.w};
  WarpTap<float> t[4];
  int o00[4], o01[4], o10[4], o11[4];
  bool valid[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    t[k] = warp2d_tap<float>(x + k, y, vx[k], vy[k], W, H, normalized);
    if (CLAMP) {
      const int x1i = (int)((unsigned)t[k].x0 + 1u), y1i = (int)((unsigned)t[k].y0 + 1u);
      const int x0 = clampi(t[k].x0, W), x1 = clampi(x1i, W), y0 = clampi(t[k].y0, H), y1 = clampi(y1i, H);
      o00[k] = y0 * W + x0; o01[k] = y0 * W + x1; o10[k] = y1 * W + x0; o11[k] = y1 * W + x1;
      valid[k] = true;
    } else {
      valid[k] = warp2d_valid(t[k].x0, t[k].y0, W, H);
      const int o = valid[k] ? t[k].y0 * W + t[k].x0 : 0;
      o00[k] = o; o01[k] = o + 1; o10[k] = o + W; o11[k] = o + W + 1;
    }
  }
  const float* src = in + n * C * hw;
  float* dst = out + n * C * hw + row;
  for (int c = 0; c < C; c += CU, src += CU * hw, dst += CU * hw) {   // (the launcher guarantees C % CU == 0)
    float v[CU][4][4];
#pragma unroll
    for (int u = 0; u < CU; ++u)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (CLAMP || valid[k]) {
          const float* q = src + u * hw;
          v[u][k][0] = __ldg(q + o00[k]); v[u][k][1] = __ldg(q + o01[k]); v[u][k][2] = __ldg(q + o10[k]); v[u][k][3] = __ldg(q + o11[k]);
        }
#pragma unroll
    for (int u = 0; u < CU; ++u) {
      float r[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) r[k] = (CLAMP || valid[k]) ? warp2d_blend(v[u][k][0], v[u][k][1], v[u][k][2], v[u][k][3], t[k]) : border_value;
      *reinterpret_cast<float4*>(dst + u * hw) = make_float4(r[0], r[1], r[2], r[3]);
    }
  }
}

template <class T>
static bool warp2d_fast(const T*, const T*, T*, int, int, int, int, int, int, T, cudaStream_t) { return false; }
template <>
bool warp2d_fast<float>(const float* in, const float* disp, float* out, int n, int c, int h, int w, int normalized, int border_mode,
                        float border_value, cudaStream_t s) {
  const int64_t total = (int64_t)n * (c > 2 ? c : 2) * h * w;
  if ((w & 3) != 0 || w < 128 || total >= (1ll << 31) || ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(disp) | reinterpret_cast<uintptr_t>(out)) & 15) != 0)
    return false;
  dim3 grid(ceil_div(w / 4, 128), h, n), block(128);
  // (CU = 3, all gathers of an RGB image in flight at once, was measured slower: 128 registers, 22 % occupancy, 77 us
  // against 62 us at [8,3,768,1024]; one channel per round keeps 48 registers)
  if (border_mode == DEMON_BORDER_CLAMP) warp2d_v4_kernel<true, 1><<<grid, block, 0, s>>>(in, disp, out, c, h, w, normalized != 0, border_value);
  else warp2d_v4_kernel<false, 1><<<grid, block, 0, s>>>(in, disp, out, c, h, w, normalized != 0, border_value);
  return true;
}

template <class T>
static int warp2d_launch(const T* in, const T* disp, T* out, int n, int c, int h, int w, int normalized,
                         int border_mode, T border_value, void* stream) {
  DEMON_REQUIRE(n >= 0 && c >= 0 && h >= 0 && w >= 0, "warp2d: negative size");
  DEMON_REQUIRE(border_mode == DEMON_BORDER_CLAMP || border_mode == DEMON_BORDER_VALUE, "warp2d: border_mode %d", border_mode);
  if ((int64_t)n * c * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(in && disp && out, "warp2d: null pointer");
  DEMON_REQUIRE(n <= 65535, "warp2d: n must be <= 65535 (got %d)", n);
  DEMON_REQUIRE(h <= 65535, "warp2d: h must be <= 65535 (got %d)", h);
  dim3 grid(ceil_div(w, 128), h, n), block(128);
  cudaStream_t s = (cudaStream_t)stream;
  if (warp2d_fast<T>(in, disp, out, n, c, h, w, normalized, border_mode, border_value, s)) {
    DEMON_LAUNCH_CHECK();
    return DEMON_OK;
  }
  if (border_mode == DEMON_BORDER_CLAMP)
    warp2d_kernel<T, true><<<grid, block, 0, s>>>(in, disp, out, c, h, w, normalized != 0, border_value);
  else
    warp2d_kernel<T, false><<<grid, block, 0, s>>>(in, disp, out, c, h, w, normalized != 0, border_value);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// depth_to_flow (replaces depthtoflow.cc:250-313 / depthtoflow_cuda.cu:62-126 + rotation_format.cu)
// grid (ceil(HW/(256*8)), N): the per-sample camera (Rodrigues etc.) is computed once per CTA by thread 0 and used for
// eight pixels per thread (a CTA per 256 pixels spent most of its time in that set-up).
// ---------------------------------------------------------------------------------------------
constexpr int kPixPerThread = 8;
template <class T>
__global__ void __launch_bounds__(256) depth_to_flow_kernel(const T* __restrict__ depth, const T* __restrict__ intrinsics,
                                                           const T* __restrict__ rotation, const T* __restrict__ translation,
                                                           T* __restrict__ flow, int H, int W, int rotation_format,
                                                           bool inverse_depth, bool normalize_flow) {
  __shared__ D2FCamera<T> cam;
  const int n = blockIdx.y;
  if (threadIdx.x == 0)
    d2f_camera(cam, intrinsics + 4 * n, rotation + (size_t)n * rotation_step(rotation_format), translation + 3 * n,
               rotation_format, W, H);
  __syncthreads();
  const int hw = H * W;
  const T* dn = depth + (size_t)n * hw;
  T* fn = flow + (size_t)n * 2 * hw;
  T dv[kPixPerThread];
#pragma unroll
  for (int k = 0; k < kPixPerThread; ++k) {   // all loads first
    const int i = (blockIdx.x * kPixPerThread + k) * 256 + threadIdx.x;
    dv[k] = (i < hw) ? __ldg(dn + i) : (T)1;
  }
#pragma unroll
  for (int k = 0; k < kPixPerThread; ++k) {
    const int i = (blockIdx.x * kPixPerThread + k) * 256 + threadIdx.x;
    if (i < hw) {
      const int y = i / W, x = i - y * W;
      T fx, fy;
      d2f_pixel(fx, fy, dv[k], x, y, cam, inverse_depth, normalize_flow);
      fn[i] = fx;
      fn[hw + i] = fy;
    }
  }
}

// float fast path: 2 x 4 consecutive pixels per thread, float4 loads and stores, 32-bit indices (H*W a multiple of 4 with W a
// multiple of 4 so that a group never crosses a row; fewer than 2^31 elements; 16-byte aligned pointers)
__global__ void __launch_bounds__(256) depth_to_flow_v4_kernel(const float* __restrict__ depth, const float* __restrict__ intrinsics,
                                                              const float* __restrict__ rotation, const float* __restrict__ translation,
                                                              float* __restrict__ flow, int H, int W, int rotation_format,
                                                              bool inverse_depth, bool normalize_flow) {
  __shared__ D2FCamera<float> cam;
  const int n = blockIdx.y;
  const int hw = H * W;
  const float* dn = depth + n * hw;
  float* fn = flow + n * 2 * hw;
  float4 dv[2];
  int idx[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {   // the depth loads are in flight while thread 0 sets the camera up
    idx[k] = ((blockIdx.x * 2 + k) * 256 + threadIdx.x) * 4;
    dv[k] = (idx[k] < hw) ? __ldg(reinterpret_cast<const float4*>(dn + idx[k])) : make_float4(1.f, 1.f, 1.f, 1.f);
  }
  if (threadIdx.x == 0)
    d2f_camera(cam, intrinsics + 4 * n, rotation + (size_t)n * rotation_step(rotation_format), translation + 3 * n, rotation_format, W, H);
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (idx[k] >= hw) continue;
    const int y = idx[k] / W, x = idx[k] - y * W;
    const float d4[4] = {dv[k].x, dv[k].y, dv[k].z, dv[k].w};
    float fx[4], fy[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) d2f_pixel(fx[j], fy[j], d4[j], x + j, y, cam, inverse_depth, normalize_flow);
    *reinterpret_cast<float4*>(fn + idx[k]) = make_float4(fx[0], fx[1], fx[2], fx[3]);
    *reinterpret_cast<float4*>(fn + hw + idx[k]) = make_float4(fy[0], fy[1], fy[2], fy[3]);
  }
}

template <class T>
static bool d2f_fast(const T*, const T*, const T*, const T*, T*, int, int, int, int, int, int, cudaStream_t) { return false; }
template <>
bool d2f_fast<float>(const float* depth, const float* k, const float* r, const float* t, float* flow, int n, int h, int w, int rf, int inv,
                     int nrm, cudaStream_t s) {
  if ((w & 3) != 0 || (int64_t)n * 2 * h * w >= (1ll << 31) || ((reinterpret_cast<uintptr_t>(depth) | reinterpret_cast<uintptr_t>(flow)) & 15) != 0) return false;
  depth_to_flow_v4_kernel<<<dim3(ceil_div(h * w, 256 * 8), n), 256, 0, s>>>(depth, k, r, t, flow, h, w, rf, inv != 0, nrm != 0);
  return true;
}

template <class T>
static int depth_to_flow_launch(const T* depth, const T* intrinsics, const T* rotation, const T* translation, T* flow,
                                int n, int h, int w, int rotation_format, int inverse_depth, int normalize_flow, void* stream) {
  DEMON_REQUIRE(rotation_format >= 0 && rotation_format <= 2, "depth_to_flow: rotation_format %d", rotation_format);
  DEMON_REQUIRE(n >= 0 && h >= 0 && w >= 0, "depth_to_flow: negative size");
  DEMON_REQUIRE(n <= 65535, "depth_to_flow: n must be <= 65535 (got %d)", n);
  if ((int64_t)n * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(depth && intrinsics && rotation && translation && flow, "depth_to_flow: null pointer");
  if (d2f_fast<T>(depth, intrinsics, rotation, translation, flow, n, h, w, rotation_format, inverse_depth, normalize_flow, (cudaStream_t)stream)) {
    DEMON_LAUNCH_CHECK();
    return DEMON_OK;
  }
  depth_to_flow_kernel<T><<<dim3(ceil_div(h * w, 256 * kPixPerThread), n), 256, 0, (cudaStream_t)stream>>>(
      depth, intrinsics, rotation, translation, flow, h, w, rotation_format, inverse_depth != 0, normalize_flow != 0);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// flow_to_depth / flow_to_depth2 (replaces flowtodepth.cc:383-481; the reference has no GPU kernel)
// ---------------------------------------------------------------------------------------------
constexpr int kF2DPixPerThread = 4;   // the double-precision camera set-up of thread 0 is shared by 512 pixels
template <class T>
__global__ void __launch_bounds__(128) flow_to_depth_kernel(const T* __restrict__ flow, const T* __restrict__ intrinsics,
                                                           const T* __restrict__ rotation, const T* __restrict__ translation,
                                                           T* __restrict__ depth, int H, int W, int rotation_format,
                                                           bool inverse_depth, bool normalized_flow) {
  __shared__ F2DCamera cam;
  const int n = blockIdx.y;
  if (threadIdx.x == 0)
    f2d_camera(cam, intrinsics + 4 * n, rotation + (size_t)n * rotation_step(rotation_format), translation + 3 * n,
               rotation_format, W, H);
  __syncthreads();
  const int hw = H * W;
  const T* f = flow + (size_t)n * 2 * hw;
  T* dn = depth + (size_t)n * hw;
  T fx[kF2DPixPerThread], fy[kF2DPixPerThread];
#pragma unroll
  for (int k = 0; k < kF2DPixPerThread; ++k) {
    const int i = (blockIdx.x * kF2DPixPerThread + k) * 128 + threadIdx.x;
    fx[k] = (i < hw) ? __ldg(f + i) : (T)0;
    fy[k] = (i < hw) ? __ldg(f + hw + i) : (T)0;
  }
#pragma unroll
  for (int k = 0; k < kF2DPixPerThread; ++k) {
    const int i = (blockIdx.x * kF2DPixPerThread + k) * 128 + threadIdx.x;
    if (i < hw) {
      const int y = i / W, x = i - y * W;
      dn[i] = f2d_pixel(fx[k], fy[k], x, y, cam, inverse_depth, normalized_flow);
    }
  }
}

template <class T>
static int flow_to_depth_launch(const T* flow, const T* intrinsics, const T* rotation, const T* translation, T* depth,
                                int n, int h, int w, int rotation_format, int inverse_depth, int normalized_flow, void* stream) {
  DEMON_REQUIRE(rotation_format >= 0 && rotation_format <= 2, "flow_to_depth: rotation_format %d", rotation_format);
  DEMON_REQUIRE(n >= 0 && h >= 0 && w >= 0, "flow_to_depth: negative size");
  DEMON_REQUIRE(n <= 65535, "flow_to_depth: n must be <= 65535 (got %d)", n);
  if ((int64_t)n * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(flow && intrinsics && rotation && translation && depth, "flow_to_depth: null pointer");
  flow_to_depth_kernel<T><<<dim3(ceil_div(h * w, 128 * kF2DPixPerThread), n), 128, 0, (cudaStream_t)stream>>>(
      flow, intrinsics, rotation, translation, depth, h, w, rotation_format, inverse_depth != 0, normalized_flow != 0);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// leaky_relu (replaces leakyrelu.cc:62-82 / leakyrelu_cuda.cu:38-47).  In the networks this op is
// fused into the convolution epilogues; the standalone kernel exists for API completeness.
// ---------------------------------------------------------------------------------------------
template <class T>
__device__ __forceinline__ T leaky(T x, T leak) {
  T a = fmul(leak, x);
  return (a < x) ? x : a;   // std::max(leak*x, x)
}

template <class T>
__global__ void __launch_bounds__(256) leaky_relu_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t size, T leak) {
  constexpr int V = 16 / sizeof(T);
  struct alignas(16) Vec { T v[V]; };
  const int64_t nvec = size / V;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (aligned) {
    for (int64_t j = i; j < nvec; j += stride) {
      Vec a = reinterpret_cast<const Vec*>(in)[j];
#pragma unroll
      for (int k = 0; k < V; ++k) a.v[k] = leaky(a.v[k], leak);
      reinterpret_cast<Vec*>(out)[j] = a;
    }
    for (int64_t j = nvec * V + i; j < size; j += stride) out[j] = leaky(in[j], leak);
  } else {
    for (int64_t j = i; j < size; j += stride) out[j] = leaky(in[j], leak);
  }
}

template <class T>
static int leaky_relu_launch(const T* in, T* out, int64_t size, T leak, void* stream) {
  DEMON_REQUIRE(size >= 0, "leaky_relu: negative size");
  if (size == 0) return DEMON_OK;
  DEMON_REQUIRE(in && out, "leaky_relu: null pointer");
  int64_t blocks = ceil_div64(ceil_div64(size, 16 / sizeof(T)), 256);
  if (blocks > 132 * 16) blocks = 132 * 16;   // 16 resident CTAs of 256 threads per SM, grid-stride beyond
  leaky_relu_kernel<T><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(in, out, size, leak);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// median3x3_downsample (replaces median3x3downsample.cc:112-184 / median3x3downsample_cuda.cu:28-99)
// grid (ceil(Wo/128), Ho, Z).  Bit exact: comparison only.
// ---------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(128) median3x3_downsample_kernel(const T* __restrict__ in, T* __restrict__ out,
                                                                  int H, int W, int Ho, int Wo, int zbase) {
  const int xo = blockIdx.x * 128 + threadIdx.x;
  const int yo = blockIdx.y;
  const int64_t z = (int64_t)zbase + blockIdx.z;
  if (xo >= Wo) return;
  const T* p = in + z * H * W;
  const int x = 2 * xo, y = 2 * yo;
  T v[9];
  int idx = 0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx)
      v[idx++] = __ldg(p + (size_t)clampi(y + dy, H) * W + clampi(x + dx, W));
  out[z * Ho * Wo + (size_t)yo * Wo + xo] = median9_reference_order(v);
}

// float fast path: FOUR outputs per thread.  Of each of the three (clamped) input rows the thread reads the eight columns
// 2*xo .. 2*xo+7 as two float4 plus the one column to the left; the four windows share these 27 values, and the result is
// one float4 store.  Taken when W is a multiple of 8 (then Wo is a multiple of 4, every group is complete and all vector
// accesses are aligned) with 16-byte aligned pointers and fewer than 2^31 elements.  The selection network is the
// reference's, compare for compare (median9_reference_order).
__global__ void __launch_bounds__(128) median3x3_v4_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int Ho, int Wo,
                                                          int zbase) {
  const int xo = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int yo = blockIdx.y;
  const int z = zbase + blockIdx.z;
  if (xo >= Wo) return;
  const float* p = in + z * (H * W);
  const int x = 2 * xo, y = 2 * yo;
  float r[3][9];   // columns x-1 .. x+7 of rows y-1, y, y+1
#pragma unroll
  for (int dy = 0; dy < 3; ++dy) {
    const float* q = p + clampi(y + dy - 1, H) * W + x;
    const float4 a = __ldg(reinterpret_cast<const float4*>(q)), b = __ldg(reinterpret_cast<const float4*>(q + 4));
    r[dy][0] = __ldg(q - (x > 0 ? 1 : 0));
    r[dy][1] = a.x; r[dy][2] = a.y; r[dy][3] = a.z; r[dy][4] = a.w;
    r[dy][5] = b.x; r[dy][6] = b.y; r[dy][7] = b.z; r[dy][8] = b.w;
  }
  float m[4];
  // Which ELEMENT the reference's selection passes pick only matters when two candidates compare equal without being
  // the same bits (+0 / -0) or do not compare at all (NaN).  Without such values among the 27 inputs the result is simply
  // the median VALUE, and any median network returns the same bits: sort the nine columns once (the four windows share
  // three of them), then median(max of the minima, median of the middles, min of the maxima): ~26 min/max per output
  // instead of 30 compare + 2 selects.  Otherwise: the reference's order, compare for compare.
  bool special = false;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int c = 0; c < 9; ++c) special |= !(fabsf(r[dy][c]) > 0.f);
  if (!special) {
    float lo[9], mid[9], hi[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) {
      const float t1 = fminf(r[0][c], r[1][c]), t2 = fmaxf(r[0][c], r[1][c]);
      lo[c] = fminf(t1, r[2][c]);
      hi[c] = fmaxf(t2, r[2][c]);
      mid[c] = fmaxf(t1, fminf(t2, r[2][c]));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = 2 * j;
      const float a = fmaxf(fmaxf(lo[c], lo[c + 1]), lo[c + 2]);
      const float b = fmaxf(fminf(mid[c], mid[c + 1]), fminf(fmaxf(mid[c], mid[c + 1]), mid[c + 2]));
      const float d = fminf(fminf(hi[c], hi[c + 1]), hi[c + 2]);
      m[j] = fmaxf(fminf(a, b), fminf(fmaxf(a, b), d));
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v[9];
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) v[3 * dy + dx] = r[dy][2 * j + dx];
      m[j] = median9_reference_order(v);
    }
  }
  *reinterpret_cast<float4*>(out + z * (Ho * Wo) + yo * Wo + xo) = make_float4(m[0], m[1], m[2], m[3]);
}

template <class T>
static bool median_fast(const T*, T*, int, int, int, int, int, int, cudaStream_t) { return false; }
template <>
bool median_fast<float>(const float* in, float* out, int h, int w, int ho, int wo, int z0, int zn, cudaStream_t s) {
  median3x3_v4_kernel<<<dim3(ceil_div(wo / 4, 128), ho, zn), 128, 0, s>>>(in, out, h, w, ho, wo, z0);
  return true;
}

template <class T>
static int median3x3_launch(const T* in, T* out, int64_t z, int h, int w, void* stream) {
  DEMON_REQUIRE(z >= 0 && h >= 0 && w >= 0, "median3x3_downsample: negative size");
  if (z * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(in && out, "median3x3_downsample: null pointer");
  const int ho = (h + 1) / 2, wo = (w + 1) / 2;
  DEMON_REQUIRE(ho <= 65535, "median3x3_downsample: (h + 1) / 2 must be <= 65535 (got h = %d)", h);
  // (the last column 2*xo+7 <= W-1 needs no clamp when W is a multiple of 8)
  const bool fast = sizeof(T) == 4 && (w & 7) == 0 && w >= 256 && z * h * w < (1ll << 31) &&
                    ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  for (int64_t z0 = 0; z0 < z; z0 += 32768) {
    int zn = (int)((z - z0 < 32768) ? (z - z0) : 32768);
    if (fast && median_fast<T>(in, out, h, w, ho, wo, (int)z0, zn, (cudaStream_t)stream)) {
      DEMON_LAUNCH_CHECK();
      continue;
    }
    median3x3_downsample_kernel<T><<<dim3(ceil_div(wo, 128), ho, zn), 128, 0, (cudaStream_t)stream>>>(in, out, h, w, ho, wo, (int)z0);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

// ---------------------------------------------------------------------------------------------
// scale_invariant_gradient forward (replaces scaleinvariantgradient.cc:148-195 /
// scaleinvariantgradient_cuda.cu:56-102).  deltas/weights travel as kernel arguments (the reference
// keeps them in a lazily initialised persistent device tensor, scaleinvariantgradient_cuda.cu:241-265).
// ---------------------------------------------------------------------------------------------
template <class T>
struct SigParams {
  int deltas[16];
  T weights[16];
  int num;
  T eps;
};

template <class T>
__global__ void __launch_bounds__(128) sig_kernel(const T* __restrict__ in, T* __restrict__ out, int H, int W, int zbase,
                                                 SigParams<T> prm) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  const int64_t z = (int64_t)zbase + blockIdx.z;
  if (x >= W) return;
  const size_t hw = (size_t)H * W;
  const T* p = in + z * hw;
  const T v0 = __ldg(p + (size_t)y * W + x);
  T gx = 0, gy = 0;
  for (int c = 0; c < prm.num; ++c) {
    const int d = prm.deltas[c];
    const T wgt = prm.weights[c];
    const T vx = (x + d >= 0 && x + d < W) ? __ldg(p + (size_t)y * W + x + d) : v0;
    const T vy = (y + d >= 0 && y + d < H) ? __ldg(p + (size_t)(y + d) * W + x) : v0;
    gx = fadd(gx, sig_term(v0, vx, wgt, prm.eps));
    gy = fadd(gy, sig_term(v0, vy, wgt, prm.eps));
  }
  T* o = out + z * 2 * hw + (size_t)y * W + x;
  o[0] = gx;
  o[hw] = gy;
}

// float fast path: FOUR consecutive pixels per thread (W a multiple of 4, 16-byte aligned pointers, fewer than 2^31
// elements).  The centre row and the row y + d are read as float4; the x neighbours x + d .. x + d + 3 come from the one or
// two aligned groups that hold them.  Per pixel and delta the SAME sequence of IEEE operations as sig_kernel
// (scaleinvariantgradient.cc:148-195): the ten divisions per pixel are what bounds the op.
__global__ void __launch_bounds__(128) sig_v4_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int zbase,
                                                    SigParams<float> prm) {
  const int x = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int y = blockIdx.y;
  const int z = zbase + blockIdx.z;
  if (x >= W) return;
  const int hw = H * W;
  const float* p = in + z * hw;
  const float* row = p + y * W;
  const float4 c4 = __ldg(reinterpret_cast<const float4*>(row + x));
  const float v0[4] = {c4.x, c4.y, c4.z, c4.w};
  float gx[4] = {0.f, 0.f, 0.f, 0.f}, gy[4] = {0.f, 0.f, 0.f, 0.f};
  for (int c = 0; c < prm.num; ++c) {
    const int d = prm.deltas[c];
    const float wgt = prm.weights[c];
    float vy[4] = {v0[0], v0[1], v0[2], v0[3]}, vx[4] = {v0[0], v0[1], v0[2], v0[3]};
    if (y + d >= 0 && y + d < H) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p + (y + d) * W + x));
      vy[0] = t.x; vy[1] = t.y; vy[2] = t.z; vy[3] = t.w;
    }
    const int b = x + d;                       // first x neighbour
    const int g0 = b & ~3, r = b - g0;         // aligned group that holds it, offset inside (arithmetic shift: fine for b < 0)
    float g[8];
    {
      const bool in0 = g0 >= 0 && g0 < W, in1 = r != 0 && g0 + 4 >= 0 && g0 + 4 < W;
      const float4 a = in0 ? __ldg(reinterpret_cast<const float4*>(row + g0)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 e = in1 ? __ldg(reinterpret_cast<const float4*>(row + g0 + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = e.x; g[5] = e.y; g[6] = e.z; g[7] = e.w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int xn = b + k;
      if (xn >= 0 && xn < W) vx[k] = (r == 0) ? g[k] : (r == 1) ? g[k + 1] : (r == 2) ? g[k + 2] : g[k + 3];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gx[k] = fadd(gx[k], sig_term(v0[k], vx[k], wgt, prm.eps));
      gy[k] = fadd(gy[k], sig_term(v0[k], vy[k], wgt, prm.eps));
    }
  }
  float* o = out + z * 2 * hw + y * W + x;
  *reinterpret_cast<float4*>(o) = make_float4(gx[0], gx[1], gx[2], gx[3]);
  *reinterpret_cast<float4*>(o + hw) = make_float4(gy[0], gy[1], gy[2], gy[3]);
}

template <class T>
static bool sig_fast(const T*, T*, int, int, int, int, const SigParams<T>&, cudaStream_t) { return false; }
template <>
bool sig_fast<float>(const float* in, float* out, int h, int w, int z0, int zn, const SigParams<float>& prm, cudaStream_t s) {
  sig_v4_kernel<<<dim3(ceil_div(w / 4, 128), h, zn), 128, 0, s>>>(in, out, h, w, z0, prm);
  return true;
}

template <class T>
static int sig_launch(const T* in, T* out, int64_t z, int h, int w, const int* deltas, const T* weights, int num, T eps,
                      void* stream) {
  DEMON_REQUIRE(z >= 0 && h >= 0 && w >= 0, "scale_invariant_gradient: negative size");
  DEMON_REQUIRE(num >= 0 && num <= 16, "scale_invariant_gradient: at most 16 deltas (got %d)", num);
  DEMON_REQUIRE(num == 0 || (deltas && weights), "scale_invariant_gradient: null deltas/weights");
  if (z * h * w == 0) return DEMON_OK;
  DEMON_REQUIRE(in && out, "scale_invariant_gradient: null pointer");
  DEMON_REQUIRE(h <= 65535, "scale_invariant_gradient: h must be <= 65535 (got %d)", h);
  SigParams<T> prm;
  prm.num = num;
  prm.eps = eps;
  for (int i = 0; i < 16; ++i) { prm.deltas[i] = i < num ? deltas[i] : 0; prm.weights[i] = i < num ? weights[i] : (T)0; }
  const bool fast = sizeof(T) == 4 && (w & 3) == 0 && w >= 128 && z * 2 * h * w < (1ll << 31) &&
                    ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  for (int64_t z0 = 0; z0 < z; z0 += 32768) {
    int zn = (int)((z - z0 < 32768) ? (z - z0) : 32768);
    if (fast && sig_fast<T>(in, out, h, w, (int)z0, zn, prm, (cudaStream_t)stream)) {
      DEMON_LAUNCH_CHECK();
      continue;
    }
    sig_kernel<T><<<dim3(ceil_div(w, 128), h, zn), 128, 0, (cudaStream_t)stream>>>(in, out, h, w, (int)z0, prm);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

}  // namespace demon

using namespace demon;

extern "C" {

const char* demon_last_error(void) { return last_error_ref().c_str(); }
const char* demon_version(void) { return "demon_b200 0.1 sm_90a"; }
int64_t demon_launch_count(void) { return g_launch_count.load(); }

int demon_warp2d_f32(const float* i, const float* d, float* o, int n, int c, int h, int w, int nm, int bm, float bv, void* s) {
  return warp2d_launch<float>(i, d, o, n, c, h, w, nm, bm, bv, s);
}
int demon_warp2d_f64(const double* i, const double* d, double* o, int n, int c, int h, int w, int nm, int bm, double bv, void* s) {
  return warp2d_launch<double>(i, d, o, n, c, h, w, nm, bm, bv, s);
}
int demon_depth_to_flow_f32(const float* d, const float* k, const float* r, const float* t, float* f, int n, int h, int w,
                            int rf, int inv, int nrm, void* s) {
  return depth_to_flow_launch<float>(d, k, r, t, f, n, h, w, rf, inv, nrm, s);
}
int demon_depth_to_flow_f64(const double* d, const double* k, const double* r, const double* t, double* f, int n, int h, int w,
                            int rf, int inv, int nrm, void* s) {
  return depth_to_flow_launch<double>(d, k, r, t, f, n, h, w, rf, inv, nrm, s);
}
int demon_flow_to_depth_f32(const float* f, const float* k, const float* r, const float* t, float* d, int n, int h, int w,
                            int rf, int inv, int nrm, void* s) {
  return flow_to_depth_launch<float>(f, k, r, t, d, n, h, w, rf, inv, nrm, s);
}
int demon_flow_to_depth_f64(const double* f, const double* k, const double* r, const double* t, double* d, int n, int h, int w,
                            int rf, int inv, int nrm, void* s) {
  return flow_to_depth_launch<double>(f, k, r, t, d, n, h, w, rf, inv, nrm, s);
}
int demon_leaky_relu_f32(const float* i, float* o, int64_t size, float leak, void* s) { return leaky_relu_launch<float>(i, o, size, leak, s); }
int demon_leaky_relu_f64(const double* i, double* o, int64_t size, double leak, void* s) { return leaky_relu_launch<double>(i, o, size, leak, s); }
int demon_median3x3_downsample_f32(const float* i, float* o, int64_t z, int h, int w, void* s) { return median3x3_launch<float>(i, o, z, h, w, s); }
int demon_median3x3_downsample_f64(const double* i, double* o, int64_t z, int h, int w, void* s) { return median3x3_launch<double>(i, o, z, h, w, s); }
int demon_scale_invariant_gradient_f32(const float* i, float* o, int64_t z, int h, int w, const int* d, const float* wt, int num,
                                       float eps, void* s) {
  return sig_launch<float>(i, o, z, h, w, d, wt, num, eps, s);
}
int demon_scale_invariant_gradient_f64(const double* i, double* o, int64_t z, int h, int w, const int* d, const double* wt, int num,
                                       double eps, void* s) {
  return sig_launch<double>(i, o, z, h, w, d, wt, num, eps, s);
}

}  // extern "C"
