// Tensor-core implicit-GEMM convolution for sm_90a (wgmma), "halo" variant: every input pixel is fetched ONCE per output
// tile.
//
// The output tile is 16 rows x 8 columns (128 GEMM rows) and, per 32-channel chunk, ONE TMA box per stride-parity plane
// brings the tile plus its halo into shared memory ((16+nqy-1) x (8+nqx-1) pixels, 128 bytes per pixel, 128-byte swizzle).
// Every filter tap is then just a different START ADDRESS inside the same shared-memory image:
//
//     GEMM row m = (y, x) of the tile  ->  halo pixel (y + qy - qy_min, x + qx - qx_min)
//
// A STEP of the main loop is one (32-channel chunk, input shift) pair.  For a plain convolution a shift is a filter tap;
// for a transposed convolution k4 s2 (four sub-pixel classes of 2x2 taps each) the 16 class-taps use only NINE distinct
// input shifts, so the A operand of a shift is loaded once and multiplied with the weight blocks of every class that uses
// it (4 classes at shift (0,0), 2 on the edges, 1 in the corners): 9 steps per chunk instead of 16.
//
// Warp roles (persistent over tiles, mbarrier rings between them, every wait bounded):
//     warpgroup 0   producer (one elected thread): the halo boxes (TMA) and the pre-swizzled weight blocks of every step
//                   (cp.async.bulk) into a ring of kRing slots
//     warpgroups 1, 2  consumers, 64 GEMM rows each: wgmma.mma_async m64nNk8 kind tf32 with the A fragment in registers
//                   (loaded from the swizzled halo image, split into A_hi = trunc_tf32(A) and A_lo = A - A_hi) and B = the
//                   weight block in shared memory; fp32 accumulators in registers; the epilogue (bias, leaky ReLU, NHWC
//                   store into the channel slice of the destination) runs on the same threads after the tile's last step
//
// K order inside a 32-channel chunk: thread (g = lane / 4, t = lane % 4) of a warp needs, for the K = 8 slice j, the
// columns t and t + 4 of its rows g and g + 8.  Slice j column kk is mapped to input channel 8 (kk % 4) + 2 j + kk / 4,
// so that a thread's four slices are the 8 CONSECUTIVE channels 8t .. 8t + 7 of its two pixels (two 16-byte loads per
// pixel); the host packs the weights in the same order.
//
// Precision (MODE): 2 = 3xTF32 = A_hi * W_lo + A_lo * W_hi + A_hi * W_hi (W split on the host), three wgmma per K = 8
// slice and class; the dropped term A_lo * W_lo is ~2^-21 relative.  0 = plain single-pass TF32.  1 = FP16: the same 8
// channels of a thread's two pixels are converted (cvt.rn.f16x2.f32, round to nearest even) into two K = 16 slices of
// m64nNk16 kind f16, slice j column kk = input channel 8 ((kk % 8) >> 1) + 4 j + 2 (kk >> 3) + (kk & 1), so that register
// R0 = (row g, channels 4j, 4j + 1), R1 = (row g + 8, same), R2 = (row g, 4j + 2, 4j + 3), R3 = (row g + 8, same) of the
// thread's eight (PTX ISA, wgmma .f16 A fragment).  The weights are packed as FP16 (round to nearest even) with 64-byte
// rows and 64-byte swizzle (TcFormat below); accumulators, epilogue and the fp32 halo staging are those of the TF32 modes.
//
// Narrow single-n-tile layers keep their whole packed weight set (<= 96 KB) RESIDENT in shared memory, loaded once per CTA
// instead of one small bulk copy per step.  Layers with few tiles split their K loop over several work items (split-K,
// halo_splitk_reduce_kernel).  Variants: PER_TAP (images that are not made of whole 16 x 8 tiles: one 128-pixel TMA box per
// step instead of a halo), CIN8 (8-channel inputs: four taps x 8 channels per K = 32 step) and FOLD (below).
//
// Fold mode (FOLD = 9 or 3: narrow 3x3 stride-1 layers, Cout 16 or 20 / 24, on images of whole 12 x 16 tiles).  At N = 16 or
// 32 a step's dozen tiny wgmma cost less than loading and splitting its A fragment, so these layers run INPUT-stationary
// with the taps in N: the GEMM rows are the pixels of the tile's 14 x 18 halo box (padded to 256 rows), the columns are
// (tap, output channel), and one K step multiplies a pixel with the weights of every folded tap:
//
//     acc[pixel][t][co] = sum_ci in[pixel][ci] * W[t][ci][co],     out[y][x][co] = sum_t acc[(y + dy_t, x + dx_t)][t][co]
//
// FOLD 9 (Cout 16): all nine taps, N = 144, one step per chunk.  FOLD 3 (Cout 24; N = 216 would not fit the registers):
// the three dx taps of a row, N = 72, and dy as three steps per chunk that shift the A rows by whole halo rows (GEMM row
// = pixel (r, c) of the 12 x 18 rows r + dy of the box).  Every pixel is loaded and split once per step instead of once
// per tap.  The epilogue (col2im) stages a third of the accumulator columns at a time in shared memory and sums the taps
// of each output in ascending tap order (deterministic), then adds the bias.
//
// Host side: tc_plan is the only place that decides whether a layer runs on this kernel and in which mode; tc_prepare
// plans and packs a layer, conv_tc_launch launches it, and the per-device launch state and timeout flag live here too.
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "conv_tc.cuh"
#include "conv_tc_ptx.cuh"
#include "wgmma_f16.cuh"
#include "wgmma_tf32.cuh"

namespace demon {

namespace {

constexpr int kRing = 4;                 // weight ring slots
constexpr int kThreads = 384;            // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr int kMaxAStages = 4;
constexpr int kTileH = 16, kTileW = 8;
constexpr int kFoldH = 12, kFoldW = 16;  // fold mode output tile: a 14 x 18 = 252-pixel halo box in 256 GEMM rows
constexpr int kMaxPlanes = 4;
constexpr int kPlanSms = 132;            // SM count the tiling model plans for (H100 SXM); the launch uses the device's count
constexpr int kSmemBudget = 224 * 1024;  // dynamic shared memory of the plan's operand stages (+ 1 KB for alignment)
constexpr int kMaxDynSmem = 226 * 1024;  // 227 KB per block on sm_90, minus the kernel's static shared memory

struct HaloPlane {
  int c_off;      // coordinate offset in dim 0 (rx * in_pitch)
  int ry;         // coordinate in dim 2
  int qx_min, qy_min;
  int cols, rows; // halo box
  int smem_off;   // byte offset of the plane inside the A region (1024-aligned)
  int bytes;      // rows * cols * 128
};

struct HaloParams {
  int tiles_x, tiles_y, B, n_tiles, total_tiles;
  uint32_t mul_n_tiles, mul_tiles_x, mul_tiles_y;   // fast_div multipliers
  int k_chunks, nplanes, nsteps, nclass;
  // split-K: a work ITEM is (tile, z), z < ksplit: kc_split = k_chunks / ksplit chunks of the tile's K loop, accumulated into
  // partial buffer z (out + z * part_stride, bias-free, no activation); halo_splitk_reduce_kernel sums the buffers.
  // ksplit == 1: an item is a tile and the epilogue writes the layer's output directly.
  int ksplit, kc_split, total_items;
  uint32_t mul_ksplit;
  long long part_stride;
  // per step (one input shift of one 32-channel chunk)
  int st_plane[kMaxTaps], st_aoff[kMaxTaps];        // halo mode: plane and byte offset of the shift's first pixel
  int st_cmask[kMaxTaps];                           // classes multiplied in this step
  int st_woff[kMaxTaps], st_wbytes[kMaxTaps];       // weight blocks of the step inside a chunk's weight image
  // per-tap mode (layers whose images are not made of whole 16x8 tiles): the A stage is ONE shift's 128-pixel tile
  // (tb images x th rows x tw columns, one TMA box per step, box coordinates carry the shift)
  int per_tap, tw, th, tb, tiles_b;
  int tap_c[kMaxTaps], tap_qx[kMaxTaps], tap_ry[kMaxTaps], tap_qy[kMaxTaps];
  // 8-channel mode (Cin == 8, e.g. the image pair): a pixel is 32 bytes in shared memory (no swizzle), the halo is loaded
  // once per tile, and one K = 32 step gathers FOUR taps x 8 channels (`nsteps` then counts these groups, g_plane / g_aoff
  // describe the real taps, -1 = missing tap -> zero columns)
  int cin8, ntaps_real;
  int g_plane[kMaxTaps], g_aoff[kMaxTaps];
  // fold mode: taps folded into N (9, 3; 0 in the other modes) and the GEMM's N = fold x (Cout rounded up to 8); the
  // epilogue's staging buffer follows the weights
  int fold, fold_n;
  HaloPlane planes[kMaxPlanes];
  int a_region_bytes;   // one halo stage (all planes)
  int sa;               // A (halo, shared memory) stages
  int w_chunk_bytes;    // weight bytes of one (n tile, chunk): sum of st_wbytes
  int w_stage_bytes;    // weight ring slot = the largest step
  int w_region_bytes;   // shared memory of the weights: kRing slots, or the whole layer when resident
  int w_resident;       // 1: ALL weight blocks of the (single) n tile live in shared memory for the whole kernel, loaded once
  int cls_bytes;        // one class block: [W_hi ; W_lo] (3xTF32) or W alone (TF32, FP16)
  int n_tile;
  int mode;             // 0 single pass TF32, 1 FP16, 2 three-instruction 3xTF32
  const unsigned char* w;
  float* out;
  int out_pitch, Ho, Wo, Hfull, Wfull, osy, osx, Cout;
  int cls_ooy[4], cls_oox[4];
  const float* bias;
  int leaky;
  int* err;
  long long* timing;   // optional [gridDim.x][16] wait-cycle counters (debug), nullptr in production
};

struct HaloMaps {
  CUtensorMap m[kMaxPlanes];
};

// Bounded wait: fast path one try_wait, slow path a spin with a cycle budget (the cycles spent there go to `acc`).  On
// timeout the error flag is raised and the kernel runs to completion with garbage; the host turns the flag into
// DEMON_E_STATE.
__device__ __forceinline__ void wait_t(uint32_t bar, uint32_t parity, int* err, long long& acc) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  for (;;) {
    if (mbar_try(bar, parity)) break;
    if (clock64() - t0 > kTimeoutCycles || *reinterpret_cast<volatile int*>(err) != 0) {
      atomicExch(err, 1);
      break;
    }
  }
  acc += clock64() - t0;
}

// x / d for small d by one multiply (mul = 2^32 / d + 1, exact while x * d < 2^32; d == 1 -> mul = 0)
__device__ __forceinline__ int fast_div(int x, int d, uint32_t mul) { return mul ? (int)__umulhi((uint32_t)x, mul) : x; }

template <bool PER_TAP, int FOLD>
__device__ __forceinline__ void halo_decode_tile(const HaloParams& p, int tile, int& nt, int& n, int& y0, int& x0) {
  int m = fast_div(tile, p.n_tiles, p.mul_n_tiles);
  nt = tile - m * p.n_tiles;
  const int m1 = fast_div(m, p.tiles_x, p.mul_tiles_x);
  const int xb = m - m1 * p.tiles_x;
  n = fast_div(m1, p.tiles_y, p.mul_tiles_y);
  const int yb = m1 - n * p.tiles_y;
  if (PER_TAP) { n *= p.tb; y0 = yb * p.th; x0 = xb * p.tw; }
  else if (FOLD) { y0 = yb * kFoldH; x0 = xb * kFoldW; }
  else { y0 = yb * kTileH; x0 = xb * kTileW; }
}

// The A fragment of one step from a thread's 8 channels of its rows g (v[0]) and g + 8 (v[1]).  TF32 modes: slice j
// (K = 8) is hi/lo[4 j + 0..3], a0 = (row g, col tq) = v[0][2j], a1 = (row g + 8, col tq), a2 = (row g, col tq + 4) =
// v[0][2j + 1], a3; A_hi = trunc_tf32(A) for 3xTF32.  FP16: slice j (K = 16) is hi[4 j + 0..3] (see the top of this file),
// lo is unused.
template <int MODE>
__device__ __forceinline__ void a_fragment(const float (&v)[2][8], uint32_t* hi, uint32_t* lo) {
  if constexpr (MODE == 1) {
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // e = 2 q + h: row g + 8 h, channels 4 j + 2 q, 4 j + 2 q + 1 (the lower one in the low half)
        const int h = e & 1, c = 4 * j + 2 * (e >> 1);
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi[4 * j + e]) : "f"(v[h][c + 1]), "f"(v[h][c]));
      }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float f[4] = {v[0][2 * j], v[1][2 * j], v[0][2 * j + 1], v[1][2 * j + 1]};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const uint32_t u = __float_as_uint(f[e]);
        hi[4 * j + e] = (MODE == 2) ? (u & 0xFFFFE000u) : u;
        lo[4 * j + e] = __float_as_uint(f[e] - __uint_as_float(u & 0xFFFFE000u));
      }
    }
  }
}

// All wgmma of ONE class block of a step: K = 32 as four K = 8 slices (TF32 modes) or two K = 16 slices (FP16).
template <int N, int MODE>
__device__ __forceinline__ void issue_block(float* acc, const uint32_t* hi, const uint32_t* lo, uint32_t wb) {
  if constexpr (MODE == 1) {
    const uint64_t w = wgmma_desc_sw64(wb);
#pragma unroll
    for (int j = 0; j < 2; ++j)   // + 32 bytes inside the swizzled 64-byte weight row per K = 16 slice
      WgmmaF16<N>::mma(acc, hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3], w + (uint64_t)(2 * j));
  } else {
    const uint64_t w_hi = wgmma_desc_sw128(wb);
    const uint64_t w_lo = wgmma_desc_sw128(wb + N * 128u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // + 32 bytes inside the swizzled weight row per K = 8 slice
      if (MODE == 2) {
        Wgmma<N>::mma(acc, hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3], w_lo + (uint64_t)(2 * j));
        Wgmma<N>::mma(acc, lo[4 * j], lo[4 * j + 1], lo[4 * j + 2], lo[4 * j + 3], w_hi + (uint64_t)(2 * j));
      }
      Wgmma<N>::mma(acc, hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3], w_hi + (uint64_t)(2 * j));
    }
  }
}

// Fold mode epilogue staging: a third of the N columns of all 256 GEMM rows per round, rows padded so that a warp's float2
// stores (8 rows x 4 column pairs) hit distinct banks
__host__ __device__ constexpr int fold_stage_pitch(int n) { return (n / 3) % 16 == 0 ? n / 3 + 8 : n / 3; }
__host__ __device__ constexpr int fold_stage_bytes(int n) { return 256 * fold_stage_pitch(n) * 4; }

// The fold-mode consumers (warpgroups 1, 2: GEMM rows 128 wg .. 128 wg + 127 as two m64 blocks).  One step (one dy of
// a chunk for FOLD 3, the whole chunk for FOLD 9) loads and splits each block's A fragment once and issues its 12
// wgmma of N = 72 / 144; the next block's pixels are read from shared memory while they run.
template <int MODE, int N, int FOLD>
__device__ __forceinline__ void fold_consumers(const HaloParams& p, unsigned char* smem, uint32_t afull0, uint32_t aempty0,
                                               uint32_t wfull0, uint32_t wempty0, uint32_t wres_bar) {
  constexpr int CO = N / FOLD;                        // columns of one tap: Cout rounded up to 8
  constexpr int BW = kFoldW + 2;                      // halo box width
  constexpr int MROWS = (FOLD == 9 ? kFoldH + 2 : kFoldH) * BW;   // GEMM rows that are pixels; rows MROWS .. 255 pad
  constexpr int TG = FOLD / 3;                        // taps per epilogue round (one dy row of taps, or one tap)
  constexpr int GC = N / 3;                           // accumulator columns per round
  constexpr int SP = fold_stage_pitch(N);
  constexpr int NQ = kFoldH * kFoldW * CO / 4;        // float4 outputs of a tile
  constexpr int OQ = (NQ + 255) / 256;                // ... per consumer thread
  static_assert(N % FOLD == 0 && CO % 8 == 0 && GC % 8 == 0, "fold geometry");
  const int ct = threadIdx.x - 128;                   // consumer thread 0 .. 255
  const int wg = ct >> 7, warp = ct >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, tq = lane & 3;
  const int m0 = 128 * wg + 16 * (warp & 3) + g;      // this thread's GEMM rows: m0 + 64 b + 8 h
  const uint32_t smem_u = smem_u32(smem);
  const uint32_t w_ring_u = smem_u + (uint32_t)(p.sa * p.a_region_bytes);
  float* stage = reinterpret_cast<float*>(smem + (size_t)p.sa * p.a_region_bytes + p.w_region_bytes);
  const float slope = p.leaky ? 0.1f : 1.0f;
  long long w_afull = 0, w_wfull = 0;
  const long long t_begin = clock64();
  int sa = 0, slot = 0;
  uint32_t pa = 0, use = 0;
  if (p.w_resident) wait_t(wres_bar, 0u, p.err, w_wfull);
  pdl_wait();   // the output buffer may still be read (or written) by the previous kernel
  float acc[2][N / 2];
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    int nt, n, y0, x0;
    halo_decode_tile<false, FOLD>(p, item, nt, n, y0, x0);
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[b][i] = 0.f;
    int l_res = 0;
    for (int kc = 0; kc < p.k_chunks; ++kc) {
      wait_t(afull0 + 8 * sa, pa, p.err, w_afull);
      const uint32_t abase = smem_u + (uint32_t)(sa * p.a_region_bytes);
      for (int s = 0; s < p.nsteps; ++s) {
        // channels 8 tq .. 8 tq + 7 of the pixels of rows m0 + 64 b and m0 + 64 b + 8 (padding rows read pixel 0)
        float v[2][8];
        auto load = [&](int b) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = m0 + 64 * b + 8 * h;
            const uint32_t row = abase + (uint32_t)((m < MROWS ? m + BW * s : 0) * 128);
            const uint32_t phase = (row >> 7) & 7u;
            const float4 a = lds128(row + (((uint32_t)(2 * tq) ^ phase) << 4));
            const float4 c = lds128(row + (((uint32_t)(2 * tq + 1) ^ phase) << 4));
            v[h][0] = a.x; v[h][1] = a.y; v[h][2] = a.z; v[h][3] = a.w; v[h][4] = c.x; v[h][5] = c.y; v[h][6] = c.z; v[h][7] = c.w;
          }
        };
        load(0);
        uint32_t wb;
        if (p.w_resident) {
          wb = w_ring_u + (uint32_t)(l_res++) * (uint32_t)p.w_stage_bytes;
        } else {
          wait_t(wfull0 + 8 * slot, use, p.err, w_wfull);
          wb = w_ring_u + (uint32_t)slot * (uint32_t)p.w_stage_bytes;
        }
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          uint32_t hi[16], lo[16];
          a_fragment<MODE>(v, hi, lo);
#pragma unroll
          for (int i = 0; i < N / 2; ++i) reg_fence(acc[b][i]);
          wgmma_fence();
          issue_block<N, MODE>(acc[b], hi, lo, wb);
          wgmma_commit();
          if (b == 0) load(1);
          wgmma_wait0();
#pragma unroll
          for (int i = 0; i < N / 2; ++i) reg_fence(acc[b][i]);
        }
        if (!p.w_resident) {
          __syncwarp();
          if (lane == 0) mbar_arrive(wempty0 + 8 * slot);
          if (++slot == kRing) { slot = 0; use ^= 1; }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(aempty0 + 8 * sa);   // this warp is done reading the halo stage
      if (++sa == p.sa) { sa = 0; pa ^= 1; }
    }
    // ---- epilogue (col2im): round r stages the columns of taps r TG .. r TG + TG - 1 of every row, then each thread adds
    // them into its float4 outputs (output pixel q / (CO / 4), channels 4 (q % (CO / 4)) ..), taps in ascending order
    float4 o[OQ];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the staging buffer's previous round (or tile) has been read
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* srow = stage + (size_t)(m0 + 64 * b + 8 * h) * SP + 2 * tq;
#pragma unroll
          for (int i = 0; i < GC / 8; ++i)
            *reinterpret_cast<float2*>(srow + 8 * i) =
                make_float2(acc[b][4 * (r * GC / 8 + i) + 2 * h], acc[b][4 * (r * GC / 8 + i) + 2 * h + 1]);
        }
      asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
      for (int j = 0; j < OQ; ++j) {
        const int q = ct + 256 * j;
        if (NQ % 256 != 0 && q >= NQ) break;
        const int pix = q / (CO / 4), c = 4 * (q % (CO / 4));
        const int y = pix / kFoldW, x = pix % kFoldW;
#pragma unroll
        for (int tl = 0; tl < TG; ++tl) {
          const int t = r * TG + tl;
          const int row = (FOLD == 9) ? (y + t / 3) * BW + x + t % 3 : y * BW + x + t;
          const float4 a = *reinterpret_cast<const float4*>(stage + (size_t)row * SP + tl * CO + c);
          if (t == 0) o[j] = a;
          else { o[j].x += a.x; o[j].y += a.y; o[j].z += a.z; o[j].w += a.w; }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < OQ; ++j) {
      const int q = ct + 256 * j;
      if (NQ % 256 != 0 && q >= NQ) break;
      const int pix = q / (CO / 4), c = 4 * (q % (CO / 4));
      if (c >= p.Cout) continue;
      const int y = pix / kFoldW, x = pix % kFoldW;
      float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bias) {
        const float2 b0 = __ldg(reinterpret_cast<const float2*>(p.bias + c)), b1 = __ldg(reinterpret_cast<const float2*>(p.bias + c + 2));
        b = make_float4(b0.x, b0.y, b1.x, b1.y);
      }
      float4 r = make_float4(o[j].x + b.x, o[j].y + b.y, o[j].z + b.z, o[j].w + b.w);
      r.x = fmaxf(slope * r.x, r.x); r.y = fmaxf(slope * r.y, r.y); r.z = fmaxf(slope * r.z, r.z); r.w = fmaxf(slope * r.w, r.w);
      *reinterpret_cast<float4*>(p.out + ((size_t)(n * p.Hfull + y0 + y) * p.Wfull + x0 + x) * p.out_pitch + c) = r;
    }
  }
  if (p.timing && threadIdx.x == 128) { p.timing[blockIdx.x * 16 + 6] = w_afull; p.timing[blockIdx.x * 16 + 3] = w_wfull; p.timing[blockIdx.x * 16 + 9] = clock64() - t_begin; }
}

template <bool PER_TAP, bool CIN8, int MODE, int N, int NCLS, int FOLD>
__global__ void __launch_bounds__(kThreads, 1) conv_tc_halo_kernel(const __grid_constant__ HaloMaps maps, const HaloParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // bars: A_full[4], A_empty[4], W_full[4], W_empty[4], W_resident
  __shared__ __align__(8) uint64_t bars[2 * kMaxAStages + 2 * kRing + 1];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t afull0 = smem_u32(&bars[0]), aempty0 = smem_u32(&bars[kMaxAStages]);
  const uint32_t wfull0 = smem_u32(&bars[2 * kMaxAStages]), wempty0 = smem_u32(&bars[2 * kMaxAStages + kRing]);
  const uint32_t wres_bar = smem_u32(&bars[2 * kMaxAStages + 2 * kRing]);
  const int a_stage_bytes = p.a_region_bytes;
  unsigned char* w_ring = smem + (size_t)p.sa * a_stage_bytes;

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < p.nplanes; ++i) asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.m[i]) : "memory");
    for (int s = 0; s < kMaxAStages; ++s) {
      mbar_init(afull0 + 8 * s, 1);
      mbar_init(aempty0 + 8 * s, kConsumerWarps);
    }
    for (int s = 0; s < kRing; ++s) {
      mbar_init(wfull0 + 8 * s, 1);
      mbar_init(wempty0 + 8 * s, kConsumerWarps);
    }
    mbar_init(wres_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const bool timed = p.timing != nullptr;
  // Programmatic dependent launch: from here on the next kernel of the stream may become resident.  The roles that read
  // what the predecessor wrote (producer: the input) or write global memory (consumers: the output) wait for it below.
  pdl_launch_dependents();

  if (warp < 4) {
    // ===== producer ===================================================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 0 || !elect_one_sync()) return;
    long long w_aempty = 0, w_wempty = 0;
    const long long t_begin = clock64();
    if (p.w_resident) {
      const uint32_t total = (uint32_t)(p.k_chunks * p.w_chunk_bytes);
      mbar_expect_tx(wres_bar, total);
      for (int kc = 0; kc < p.k_chunks; ++kc)
        bulk_load(smem_u32(w_ring + (size_t)kc * p.w_chunk_bytes), p.w + (size_t)kc * p.w_chunk_bytes, (uint32_t)p.w_chunk_bytes, wres_bar);
    }
    uint32_t a_bytes = 0;
    for (int i = 0; i < p.nplanes; ++i) a_bytes += (uint32_t)p.planes[i].bytes;
    int sa = 0, slot = 0;
    uint32_t pa = 0, use = 0;
    pdl_wait();   // the input is the previous kernel's output
    for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      const int tile = fast_div(item, p.ksplit, p.mul_ksplit);
      const int kc0 = (item - tile * p.ksplit) * p.kc_split;
      int nt, n, y0, x0;
      halo_decode_tile<PER_TAP, FOLD>(p, tile, nt, n, y0, x0);
      const unsigned char* wsrc = p.w + ((size_t)nt * p.k_chunks + kc0) * p.w_chunk_bytes;
      for (int kc = kc0; kc < kc0 + p.kc_split; ++kc, wsrc += p.w_chunk_bytes) {
        if (!PER_TAP) {
          wait_t(aempty0 + 8 * sa, pa ^ 1, p.err, w_aempty);
          const uint32_t abase = smem_u32(smem + (size_t)sa * a_stage_bytes);
          mbar_expect_tx(afull0 + 8 * sa, a_bytes);
          for (int i = 0; i < p.nplanes; ++i) {
            const HaloPlane& pl = p.planes[i];
            tma_load_5d(abase + pl.smem_off, &maps.m[i], afull0 + 8 * sa, pl.c_off + kc * 32, x0 + pl.qx_min, pl.ry, y0 + pl.qy_min, n);
          }
          if (++sa == p.sa) { sa = 0; pa ^= 1; }
        }
        for (int t = 0; t < p.nsteps; ++t) {
          if (PER_TAP) {
            wait_t(aempty0 + 8 * sa, pa ^ 1, p.err, w_aempty);
            mbar_expect_tx(afull0 + 8 * sa, 128u * 128u);
            tma_load_5d(smem_u32(smem + (size_t)sa * a_stage_bytes), &maps.m[0], afull0 + 8 * sa, p.tap_c[t] + kc * 32, x0 + p.tap_qx[t],
                        p.tap_ry[t], y0 + p.tap_qy[t], n);
            if (++sa == p.sa) { sa = 0; pa ^= 1; }
          }
          if (!p.w_resident) {
            wait_t(wempty0 + 8 * slot, use ^ 1, p.err, w_wempty);
            const uint32_t bytes = (uint32_t)p.st_wbytes[t];
            mbar_expect_tx(wfull0 + 8 * slot, bytes);
            bulk_load(smem_u32(w_ring + (size_t)slot * p.w_stage_bytes), wsrc + p.st_woff[t], bytes, wfull0 + 8 * slot);
            if (++slot == kRing) { slot = 0; use ^= 1; }
          }
        }
      }
    }
    if (timed) { p.timing[blockIdx.x * 16 + 0] = w_aempty; p.timing[blockIdx.x * 16 + 1] = w_wempty; p.timing[blockIdx.x * 16 + 8] = clock64() - t_begin; }
    return;
  }

  // ===== consumers ======================================================================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  if constexpr (FOLD != 0) {
    fold_consumers<MODE, N, FOLD>(p, smem, afull0, aempty0, wfull0, wempty0, wres_bar);
    return;
  }
  const int wg = (warp >> 2) - 1;            // 0, 1: GEMM rows 64 wg .. 64 wg + 63
  const int wq = warp & 3;                   // warp inside the warpgroup: rows + 16 wq
  const int g = lane >> 2, tq = lane & 3;
  const int m0 = 64 * wg + 16 * wq + g;      // this thread's GEMM rows m0 and m0 + 8
  // tile-relative position of the two rows
  int pos_y[2], pos_x[2], pos_n[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + 8 * h;
    pos_x[h] = PER_TAP ? (m % p.tw) : (m & 7);
    pos_y[h] = PER_TAP ? ((m / p.tw) % p.th) : (m >> 3);
    pos_n[h] = PER_TAP ? (m / (p.tw * p.th)) : 0;
  }
  const float slope = p.leaky ? 0.1f : 1.0f;
  const uint32_t w_ring_u = smem_u32(w_ring);
  long long w_afull = 0, w_wfull = 0;
  const long long t_begin = clock64();
  int sa = 0, slot = 0, l_res = 0;
  uint32_t pa = 0, use = 0;
  if (p.w_resident) wait_t(wres_bar, 0u, p.err, w_wfull);
  pdl_wait();   // the output buffer may still be read (or written) by the previous kernel
  float acc[NCLS][N / 2];
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    const int tile = fast_div(item, p.ksplit, p.mul_ksplit);
    const int z = item - tile * p.ksplit;
    int nt, n, y0, x0;
    halo_decode_tile<PER_TAP, 0>(p, tile, nt, n, y0, x0);
#pragma unroll
    for (int k = 0; k < NCLS; ++k)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[k][i] = 0.f;
    l_res = 0;
    for (int kc = 0; kc < p.kc_split; ++kc) {
      uint32_t abase = 0;
      if (!PER_TAP) {
        wait_t(afull0 + 8 * sa, pa, p.err, w_afull);
        abase = smem_u32(smem + (size_t)sa * a_stage_bytes);
      }
      for (int t = 0; t < p.nsteps; ++t) {
        if (PER_TAP) {
          wait_t(afull0 + 8 * sa, pa, p.err, w_afull);
          abase = smem_u32(smem + (size_t)sa * a_stage_bytes);
        }
        // the A fragment: channels 8 tq .. 8 tq + 7 of the two pixels (rows m0, m0 + 8)
        float v[2][8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (CIN8) {
            const int rt = 4 * t + tq;   // this thread's tap of the group of four
            const int pi = (rt < p.ntaps_real) ? p.g_plane[rt] : -1;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
            if (pi >= 0) {
              const HaloPlane& pl = p.planes[pi];
              const uint32_t px = abase + (uint32_t)(pl.smem_off + p.g_aoff[rt] + (pos_y[h] * pl.cols + pos_x[h]) * 32);
              a = lds128(px); b = lds128(px + 16);
            }
            v[h][0] = a.x; v[h][1] = a.y; v[h][2] = a.z; v[h][3] = a.w; v[h][4] = b.x; v[h][5] = b.y; v[h][6] = b.z; v[h][7] = b.w;
          } else {
            uint32_t row;
            if (PER_TAP) {
              row = abase + (uint32_t)((m0 + 8 * h) * 128);
            } else {
              const HaloPlane& pl = p.planes[p.st_plane[t]];
              row = abase + (uint32_t)(pl.smem_off + p.st_aoff[t] + (pos_y[h] * pl.cols + pos_x[h]) * 128);
            }
            const uint32_t phase = (row >> 7) & 7u;   // 128-byte swizzle: 16-byte chunk c of the pixel lives at chunk c ^ phase
            const float4 a = lds128(row + (((uint32_t)(2 * tq) ^ phase) << 4));
            const float4 b = lds128(row + (((uint32_t)(2 * tq + 1) ^ phase) << 4));
            v[h][0] = a.x; v[h][1] = a.y; v[h][2] = a.z; v[h][3] = a.w; v[h][4] = b.x; v[h][5] = b.y; v[h][6] = b.z; v[h][7] = b.w;
          }
        }
        uint32_t hi[16], lo[16];
        a_fragment<MODE>(v, hi, lo);
        uint32_t wb;
        if (p.w_resident) {
          wb = w_ring_u + (uint32_t)(l_res++) * (uint32_t)p.w_stage_bytes;
        } else {
          wait_t(wfull0 + 8 * slot, use, p.err, w_wfull);
          wb = w_ring_u + (uint32_t)slot * (uint32_t)p.w_stage_bytes;
        }
#pragma unroll
        for (int k = 0; k < NCLS; ++k)
#pragma unroll
          for (int i = 0; i < N / 2; ++i) reg_fence(acc[k][i]);
        wgmma_fence();
        if (NCLS == 1) {
          issue_block<N, MODE>(acc[0], hi, lo, wb);
        } else {
          const uint32_t cm = (uint32_t)p.st_cmask[t];
#pragma unroll
          for (int k = 0; k < NCLS; ++k)
            if (cm & (1u << k)) {
              issue_block<N, MODE>(acc[k], hi, lo, wb);
              wb += (uint32_t)p.cls_bytes;
            }
        }
        wgmma_commit();
        wgmma_wait0();
#pragma unroll
        for (int k = 0; k < NCLS; ++k)
#pragma unroll
          for (int i = 0; i < N / 2; ++i) reg_fence(acc[k][i]);
        __syncwarp();
        if (lane == 0) {
          if (!p.w_resident) mbar_arrive(wempty0 + 8 * slot);
          if (PER_TAP) mbar_arrive(aempty0 + 8 * sa);
        }
        if (!p.w_resident && ++slot == kRing) { slot = 0; use ^= 1; }
        if (PER_TAP && ++sa == p.sa) { sa = 0; pa ^= 1; }
      }
      if (!PER_TAP) {
        __syncwarp();
        if (lane == 0) mbar_arrive(aempty0 + 8 * sa);   // this warp is done reading the halo stage
        if (++sa == p.sa) { sa = 0; pa ^= 1; }
      }
    }
    // ---- epilogue: accumulator (row, col 8 i + 2 tq .. + 1) -> bias, leaky ReLU -> NHWC slice ------------------------
    float* tile_out = p.out + (size_t)z * p.part_stride + ((size_t)(n * p.Hfull + y0 * p.osy) * p.Wfull + x0 * p.osx) * p.out_pitch;
    const int cbase = nt * N;
#pragma unroll
    for (int k = 0; k < NCLS; ++k) {
      if (k >= p.nclass) break;
      float* cls_out = tile_out + (size_t)(p.cls_ooy[k] * p.Wfull + p.cls_oox[k]) * p.out_pitch;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (y0 + pos_y[h] >= p.Ho || x0 + pos_x[h] >= p.Wo || n + pos_n[h] >= p.B) continue;
        float* orow = cls_out + ((size_t)(pos_n[h] * p.Hfull + pos_y[h] * p.osy) * p.Wfull + pos_x[h] * p.osx) * p.out_pitch;
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
          const int col = cbase + 8 * i + 2 * tq;
          if (col >= p.Cout) continue;
          const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);   // (null: split-K partial sums)
          float2 o;
          o.x = acc[k][4 * i + 2 * h] + b.x;
          o.y = acc[k][4 * i + 2 * h + 1] + b.y;
          // max(slope * x, x) with slope 0.1 (leaky ReLU, helpers.py:36-38) or 1 (identity, exact)
          o.x = fmaxf(slope * o.x, o.x); o.y = fmaxf(slope * o.y, o.y);
          *reinterpret_cast<float2*>(orow + col) = o;
        }
      }
    }
  }
  if (timed && threadIdx.x == 128) { p.timing[blockIdx.x * 16 + 6] = w_afull; p.timing[blockIdx.x * 16 + 3] = w_wfull; p.timing[blockIdx.x * 16 + 9] = clock64() - t_begin; }
}

// Split-K second pass: out[pix][c] = act(bias[c] + sum_z part[z][pix][c]); the partial buffers have the geometry of the
// layer's full output image ([B][Hfull][Wfull][cpitch] floats each), so sub-pixel classes are already interleaved.
__global__ void __launch_bounds__(256) halo_splitk_reduce_kernel(const float* __restrict__ part, long long part_stride, int ksplit,
                                                                 float* __restrict__ out, int out_pitch, int cpitch, int Cout, long long npix,
                                                                 const float* __restrict__ bias, int leaky) {
  pdl_launch_dependents();
  pdl_wait();
  const int c4n = cpitch >> 2;
  const long long total = npix * c4n;
  const float slope = leaky ? 0.1f : 1.0f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long pix = i / c4n;
    const int c = (int)(i - pix * c4n) * 4;
    if (c >= Cout) continue;
    float4 acc = __ldg(reinterpret_cast<const float4*>(bias + c));
    for (int z = 0; z < ksplit; ++z) {   // fixed order: deterministic
      const float4 v = *reinterpret_cast<const float4*>(part + (size_t)z * part_stride + (size_t)pix * cpitch + c);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    acc.x = fmaxf(slope * acc.x, acc.x); acc.y = fmaxf(slope * acc.y, acc.y);
    acc.z = fmaxf(slope * acc.z, acc.z); acc.w = fmaxf(slope * acc.w, acc.w);
    *reinterpret_cast<float4*>(out + (size_t)pix * out_pitch + c) = acc;
  }
}

int floor_div_h(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

}  // namespace

// ---- host side ------------------------------------------------------------------------------------------------------
struct HaloPlan {
  HaloParams prm;
  HaloMaps maps;
  int smem_bytes;
  // weight source of every (step, class): tap index inside the class, -1 = class not in the step
  int st_tap[kMaxTaps][4];
};

static int pow2_ceil_h(int v) { int r = 1; while (r < v) r <<= 1; return r; }

// The operand format of a tensor-core precision: the kernel's MODE and the packed weight blocks it reads.  A block is
// `rows` rows (output channels) of one 32-channel chunk, K-major: 128 bytes per fp32 row (TF32 modes, 128-byte swizzle,
// wgmma_desc_sw128) or 64 bytes per FP16 row (64-byte swizzle, wgmma_desc_sw64); 3xTF32 stores [W_hi ; W_lo].  A block is
// aligned to its swizzle atom of 8 rows.
struct TcFormat {
  int mode;        // the kernel's MODE: 0 TF32, 1 FP16, 2 3xTF32
  int row_bytes;   // one packed row of a chunk
  int parts;       // weight images per block: 2 for [W_hi ; W_lo], else 1
  int block_bytes(int rows) const {
    const int atom = 8 * row_bytes;
    return (rows * row_bytes * parts + atom - 1) / atom * atom;
  }
  // byte offset of K position k (0 .. 31) of row r inside one weight image of a block, and the input channel of the chunk
  // that K position holds (the K order of the kernel's A fragment, see the top of this file)
  int offset(int r, int k) const {
    return mode == 1 ? r * 64 + (((k >> 3) ^ ((r >> 1) & 3)) << 4) + (k & 7) * 2 : r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4;
  }
  int channel(int k) const {
    if (mode == 1) { const int j = k >> 4, kk = k & 15; return 8 * ((kk & 7) >> 1) + 4 * j + 2 * (kk >> 3) + (kk & 1); }
    const int kk = k & 7;
    return 8 * (kk & 3) + 2 * (k >> 3) + (kk >> 2);
  }
};

static TcFormat tc_format(int precision) {
  if (precision == DEMON_PREC_TF32) return {0, 128, 1};
  if (precision == DEMON_PREC_FP16) return {1, 64, 1};
  return {2, 128, 2};
}
static int popcount4(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1) + ((m >> 3) & 1); }

// Steps of one chunk: the distinct input shifts of all classes, each with the mask of the classes that use it.
// max_cls: at most this many classes per step (a wide step needs a wide weight slot; a shift is repeated if necessary).
struct ShiftStep { int ry, rx, qy, qx, cmask, tap[4]; };

static bool plan_tail(const ConvProblem* probs, int nclass, HaloPlan& plan);

// The tiling of one layer (no tensor maps, no weights).  force_per_tap: per-tap mode even for images made of whole
// 16 x 8 tiles (the fallback for shapes the halo mode refuses).
static bool halo_build(const ConvProblem* probs, int nclass, const TcFormat& fmt, HaloPlan& plan, bool force_per_tap) {
  const ConvProblem& p = probs[0];
  HaloParams& prm = plan.prm;
  const int budget = kSmemBudget;
  // candidates, widest first: classes per step (a wide step needs a wide weight slot), then the N tile cap
  struct Cand { int max_cls, n_cap; };
  std::vector<Cand> cands;
  for (int mc = nclass; mc >= 1; mc = (mc > 2 ? 2 : mc - 1)) cands.push_back({mc, 256});
  cands.push_back({1, 64});
  cands.push_back({1, 32});
  bool found = false;
  for (const Cand& cand : cands) {
    const int max_cls = cand.max_cls;
    memset(&prm, 0, sizeof(prm));
    memset(plan.st_tap, -1, sizeof(plan.st_tap));
    prm.nclass = nclass;
    prm.cin8 = (p.Cin == 8) ? 1 : 0;
    const int px_bytes = prm.cin8 ? 32 : 128;   // bytes of one pixel of a halo plane in shared memory
    prm.per_tap = (force_per_tap || (p.Ho % kTileH) != 0 || (p.Wo % kTileW) != 0) ? 1 : 0;
    if (prm.cin8 && (prm.per_tap || nclass != 1)) return false;
    // ---- steps ---------------------------------------------------------------------------------------------------
    std::vector<ShiftStep> steps;
    for (int c = 0; c < nclass; ++c)
      for (int i = 0; i < probs[c].ntaps; ++i) {
        const int qy = floor_div_h(probs[c].dy[i], p.sy), ry = probs[c].dy[i] - qy * p.sy;
        const int qx = floor_div_h(probs[c].dx[i], p.sx), rx = probs[c].dx[i] - qx * p.sx;
        int si = -1;
        for (size_t k = 0; k < steps.size(); ++k)
          if (steps[k].ry == ry && steps[k].rx == rx && steps[k].qy == qy && steps[k].qx == qx && !((steps[k].cmask >> c) & 1) &&
              popcount4(steps[k].cmask) < max_cls) { si = (int)k; break; }
        if (si < 0) { steps.push_back({ry, rx, qy, qx, 0, {-1, -1, -1, -1}}); si = (int)steps.size() - 1; }
        steps[si].cmask |= 1 << c;
        steps[si].tap[c] = i;
      }
    const int nreal = (int)steps.size();
    if (nreal > kMaxTaps) return false;
    int m_tiles = 0;
    if (prm.per_tap) {
      // one 128-pixel tile per step, tb images x th rows x tw columns
      for (int t = 0; t < nreal; ++t) {
        prm.tap_qy[t] = steps[t].qy; prm.tap_ry[t] = steps[t].ry;
        prm.tap_qx[t] = steps[t].qx; prm.tap_c[t] = steps[t].rx * p.in_pitch;
      }
      prm.nplanes = 1;
      long best_tiles = -1;
      const int tw = std::min(128, pow2_ceil_h(p.Wo));
      for (int th = 1; th * tw <= 128; th <<= 1) {
        const int tb = 128 / (tw * th);
        const long tiles = (long)ceil_div(p.Wo, tw) * ceil_div(p.Ho, th) * ceil_div(p.B, tb);
        if (best_tiles < 0 || tiles <= best_tiles) {
          best_tiles = tiles;
          prm.tw = tw; prm.th = th; prm.tb = tb;
          prm.tiles_x = ceil_div(p.Wo, tw); prm.tiles_y = ceil_div(p.Ho, th); prm.tiles_b = ceil_div(p.B, tb);
        }
      }
      prm.planes[0].cols = prm.tw; prm.planes[0].rows = prm.th; prm.planes[0].bytes = 128 * 128;
      prm.a_region_bytes = 128 * 128;
      m_tiles = prm.tiles_x * prm.tiles_y * prm.tiles_b;
    } else {
      // planes: shifts grouped by stride parity
      struct PInfo { int ry, rx, qy_min, qy_max, qx_min, qx_max; };
      std::vector<PInfo> pinfo;
      std::vector<int> step_plane(nreal);
      for (int t = 0; t < nreal; ++t) {
        int pi = -1;
        for (size_t k = 0; k < pinfo.size(); ++k)
          if (pinfo[k].ry == steps[t].ry && pinfo[k].rx == steps[t].rx) pi = (int)k;
        if (pi < 0) { pinfo.push_back({steps[t].ry, steps[t].rx, steps[t].qy, steps[t].qy, steps[t].qx, steps[t].qx}); pi = (int)pinfo.size() - 1; }
        PInfo& pl = pinfo[pi];
        pl.qy_min = std::min(pl.qy_min, steps[t].qy); pl.qy_max = std::max(pl.qy_max, steps[t].qy);
        pl.qx_min = std::min(pl.qx_min, steps[t].qx); pl.qx_max = std::max(pl.qx_max, steps[t].qx);
        step_plane[t] = pi;
      }
      if ((int)pinfo.size() > kMaxPlanes) return false;
      prm.nplanes = (int)pinfo.size();
      int off = 0;
      for (int i = 0; i < prm.nplanes; ++i) {
        HaloPlane& pl = prm.planes[i];
        pl.c_off = pinfo[i].rx * p.in_pitch; pl.ry = pinfo[i].ry;
        pl.qx_min = pinfo[i].qx_min; pl.qy_min = pinfo[i].qy_min;
        pl.cols = kTileW + pinfo[i].qx_max - pinfo[i].qx_min;
        pl.rows = kTileH + pinfo[i].qy_max - pinfo[i].qy_min;
        if (pl.cols > 256 || pl.rows > 256) return false;
        pl.bytes = pl.rows * pl.cols * px_bytes;
        pl.smem_off = off;
        off += (pl.bytes + 1023) / 1024 * 1024;
      }
      prm.a_region_bytes = off;
      for (int t = 0; t < nreal; ++t) {
        const HaloPlane& pl = prm.planes[step_plane[t]];
        prm.st_plane[t] = step_plane[t];
        prm.st_aoff[t] = ((steps[t].qy - pl.qy_min) * pl.cols + (steps[t].qx - pl.qx_min)) * px_bytes;
      }
      prm.tiles_x = ceil_div(p.Wo, kTileW); prm.tiles_y = ceil_div(p.Ho, kTileH); prm.tiles_b = p.B;
      m_tiles = prm.tiles_x * prm.tiles_y * p.B;
    }
    // class masks, weight source of every (step, class)
    for (int t = 0; t < nreal; ++t) {
      prm.st_cmask[t] = steps[t].cmask;
      for (int c = 0; c < 4; ++c) plan.st_tap[t][c] = steps[t].tap[c];
    }
    prm.nsteps = nreal;
    if (prm.cin8) {   // regroup: one K step = four consecutive taps (nclass == 1: every real step is one tap of class 0)
      prm.ntaps_real = nreal;
      for (int t = 0; t < nreal; ++t) { prm.g_plane[t] = prm.st_plane[t]; prm.g_aoff[t] = prm.st_aoff[t]; }
      prm.nsteps = (nreal + 3) / 4;
      for (int t = 0; t < prm.nsteps; ++t) { prm.st_plane[t] = 0; prm.st_aoff[t] = 0; prm.st_cmask[t] = 1; }
    }
    // ---- N tile: one of the kernel's instantiations (16, 32, 64, 128), at most 64 per class when several classes share
    // a step: the accumulators live in registers, N / 2 floats per thread and class (<= 128 of the consumers' 232).
    const int cout16 = (p.Cout + 15) / 16 * 16;
    int n_tile = std::min(pow2_ceil_h(std::max(cout16, 16)), std::min(nclass > 1 ? 64 : 128, cand.n_cap));
    // narrow the N tile (down to 64) while the layer would leave SMs idle
    while (n_tile >= 128 && (long)m_tiles * ceil_div(p.Cout, n_tile) < kPlanSms) n_tile /= 2;
    prm.mode = fmt.mode;
    prm.n_tile = n_tile;
    prm.n_tiles = ceil_div(p.Cout, n_tile);
    prm.k_chunks = prm.cin8 ? 1 : p.Cin / 32;
    // ---- weights: one class block of the precision's format (TcFormat); a step holds the blocks of its classes in
    // ascending class order; the ring slot is as large as the widest step
    prm.cls_bytes = fmt.block_bytes(n_tile);
    int woff = 0, wmax = 0;
    for (int t = 0; t < prm.nsteps; ++t) {
      prm.st_woff[t] = woff;
      prm.st_wbytes[t] = popcount4(prm.st_cmask[t]) * prm.cls_bytes;
      woff += prm.st_wbytes[t];
      wmax = std::max(wmax, prm.st_wbytes[t]);
    }
    prm.w_chunk_bytes = woff;
    prm.w_stage_bytes = wmax;
    // shared memory: the weights (a ring of kRing slots, or the whole layer: see the W producer), then up to 4 halo stages
    // (at least 2).  Resident: one n tile, one class, every step the same size, <= 96 KB in all and at least 2 A stages left.
    const int w_total = prm.k_chunks * prm.w_chunk_bytes;
    prm.w_resident = 0;
    prm.w_region_bytes = kRing * wmax;
    if (!force_per_tap && nclass == 1 && prm.n_tiles == 1 && w_total <= 96 * 1024 && wmax * prm.nsteps == prm.w_chunk_bytes &&
        budget - w_total >= 2 * prm.a_region_bytes) {
      prm.w_resident = 1;
      prm.w_region_bytes = w_total;
    }
    const int rest = budget - prm.w_region_bytes;
    if (rest < 2 * prm.a_region_bytes) continue;   // next candidate: narrower steps / narrower N tile
    prm.sa = std::min(kMaxAStages, rest / prm.a_region_bytes);
    plan.smem_bytes = prm.sa * prm.a_region_bytes + prm.w_region_bytes + 1024;
    found = true;
    break;
  }
  if (!found || prm.sa < 2) return false;
  return plan_tail(probs, nclass, plan);
}

// What every mode's plan derives from its tiling: work items, split-K, the fast_div multipliers, the output.
static bool plan_tail(const ConvProblem* probs, int nclass, HaloPlan& plan) {
  const ConvProblem& p = probs[0];
  HaloParams& prm = plan.prm;
  prm.B = p.B;
  const int m_tiles = prm.tiles_x * prm.tiles_y * prm.tiles_b;
  prm.total_tiles = m_tiles * prm.n_tiles;
  // ---- split-K: layers with few tiles and a long K loop (the 6x8 / 12x16 levels; everything at batch 1) leave most SMs
  // idle and run their K loop serially.  Cost model in cycles: rounds of kPlanSms items x (steps of an item x ~600 + ~3000
  // of prologue / epilogue), + ~12000 for the second pass + the partial sums' trip through L2; a split has to win 10 %.
  prm.ksplit = 1;
  if (!prm.cin8 && !prm.fold && !prm.w_resident && prm.k_chunks >= 4) {
    // the partial sums travel to the second pass through L2 (~4000 B per cycle for write + read back)
    const long out_bytes = (long)p.B * p.Hfull * p.Wfull * ((p.Cout + 3) / 4 * 4) * 4;
    auto cost = [&](int ks) {
      const long items = (long)prm.total_tiles * ks;
      return ((items + kPlanSms - 1) / kPlanSms) * ((long)(prm.k_chunks / ks) * prm.nsteps * 600 + 3000) + (ks > 1 ? 12000 + ks * out_bytes * 2 / 4000 : 0);
    };
    long best = cost(1);
    for (int ks = 2; ks <= 8; ++ks) {
      if (prm.k_chunks % ks != 0 || prm.k_chunks / ks < 2) continue;
      const long c = cost(ks);
      if (c * 10 < best * 9 && c < cost(prm.ksplit)) prm.ksplit = ks;
    }
  }
  prm.kc_split = prm.k_chunks / prm.ksplit;
  prm.total_items = prm.total_tiles * prm.ksplit;
  prm.part_stride = 0;
  auto fd = [](int d) { return d <= 1 ? 0u : (uint32_t)((1ull << 32) / (uint64_t)d + 1ull); };
  prm.mul_n_tiles = fd(prm.n_tiles); prm.mul_tiles_x = fd(prm.tiles_x); prm.mul_tiles_y = fd(prm.tiles_y);
  prm.mul_ksplit = fd(prm.ksplit);
  if ((uint64_t)prm.total_items * (uint64_t)prm.ksplit >= (1ull << 32)) return false;
  if ((uint64_t)prm.total_tiles * (uint64_t)std::max(prm.n_tiles, std::max(prm.tiles_x, prm.tiles_y)) >= (1ull << 32)) return false;
  prm.out = p.out; prm.out_pitch = p.out_pitch; prm.Ho = p.Ho; prm.Wo = p.Wo; prm.Hfull = p.Hfull; prm.Wfull = p.Wfull;
  prm.osy = p.osy; prm.osx = p.osx; prm.Cout = p.Cout; prm.bias = p.bias; prm.leaky = p.leaky;
  for (int c = 0; c < nclass; ++c) { prm.cls_ooy[c] = probs[c].ooy; prm.cls_oox[c] = probs[c].oox; }
  return true;
}

// The fold mode's plan (see the top of this file), or false for a layer it does not take: one class of a plain 3x3
// stride-1 convolution (taps in row-major order), Cin >= 64, Cout 16 (FOLD 9, N 144) or 20 / 24 (FOLD 3, N 72: the
// kernel's two fold instantiations), an output of whole 12 x 16 tiles.  Weights resident when they fit, else the ring.
static bool fold_build(const ConvProblem* probs, int nclass, const TcFormat& fmt, HaloPlan& plan) {
  const ConvProblem& p = probs[0];
  if (nclass != 1 || p.ntaps != 9 || p.sy != 1 || p.sx != 1 || p.Cin < 64 || (p.Ho % kFoldH) != 0 || (p.Wo % kFoldW) != 0) return false;
  if (p.osy != 1 || p.osx != 1 || p.ooy != 0 || p.oox != 0) return false;
  for (int t = 0; t < 9; ++t)
    if (p.dy[t] != t / 3 - 1 || p.dx[t] != t % 3 - 1) return false;
  const int co8 = (p.Cout + 7) / 8 * 8;
  const int fold = (co8 == 16) ? 9 : (co8 == 24 ? 3 : 0);
  if (!fold) return false;
  HaloParams& prm = plan.prm;
  memset(&prm, 0, sizeof(prm));
  memset(plan.st_tap, -1, sizeof(plan.st_tap));
  prm.fold = fold;
  prm.fold_n = fold * co8;
  prm.nclass = 1;
  prm.mode = fmt.mode;
  prm.n_tile = pow2_ceil_h((p.Cout + 15) / 16 * 16);   // the output channels of a tile, as in the halo mode
  prm.n_tiles = 1;
  prm.k_chunks = p.Cin / 32;
  prm.nsteps = 9 / fold;
  prm.nplanes = 1;
  HaloPlane& pl = prm.planes[0];
  pl.qx_min = -1; pl.qy_min = -1;
  pl.cols = kFoldW + 2; pl.rows = kFoldH + 2;
  pl.bytes = pl.rows * pl.cols * 128;
  prm.a_region_bytes = (pl.bytes + 1023) / 1024 * 1024;
  prm.cls_bytes = fmt.block_bytes(prm.fold_n);
  for (int t = 0; t < prm.nsteps; ++t) {
    prm.st_cmask[t] = 1;
    prm.st_woff[t] = t * prm.cls_bytes;
    prm.st_wbytes[t] = prm.cls_bytes;
  }
  prm.w_chunk_bytes = prm.nsteps * prm.cls_bytes;
  prm.w_stage_bytes = prm.cls_bytes;
  const int w_total = prm.k_chunks * prm.w_chunk_bytes;
  const int stage = fold_stage_bytes(prm.fold_n);
  prm.w_resident = (w_total <= 96 * 1024 && kSmemBudget - w_total - stage >= 2 * prm.a_region_bytes) ? 1 : 0;
  prm.w_region_bytes = prm.w_resident ? w_total : kRing * prm.cls_bytes;
  const int rest = kSmemBudget - prm.w_region_bytes - stage;
  if (rest < 2 * prm.a_region_bytes) return false;
  prm.sa = std::min(kMaxAStages, rest / prm.a_region_bytes);
  plan.smem_bytes = prm.sa * prm.a_region_bytes + prm.w_region_bytes + stage + 1024;
  prm.tiles_x = p.Wo / kFoldW; prm.tiles_y = p.Ho / kFoldH; prm.tiles_b = p.B;
  return plan_tail(probs, nclass, plan);
}

// The shape rules of the kernel, for one problem
static bool tc_shape_supported(const ConvProblem& p) {
  const bool cin8 = p.Cin == 8 && p.in_pitch == 8;   // 8-channel mode: four taps x 8 channels per K = 32 step
  if (!cin8 && (p.Cin < 32 || (p.Cin % 32) != 0)) return false;
  if (p.Cout < 16 || (p.Cout % 4) != 0) return false;
  if ((p.in_pitch % 4) != 0 || (p.out_pitch % 4) != 0) return false;
  if ((reinterpret_cast<uintptr_t>(p.in) & 15) != 0 || (reinterpret_cast<uintptr_t>(p.out) & 15) != 0) return false;
  if (p.sy < 1 || p.sx < 1 || (p.Hi % p.sy) != 0 || (p.Wi % p.sx) != 0) return false;
  if (p.ntaps < 1 || p.ntaps > kMaxTaps) return false;
  if (p.scale != nullptr) return false;
  if (p.Ho != p.Hi / p.sy || p.Wo != p.Wi / p.sx) return false;
  return true;
}

// The one decision of the tensor-core path: whether a layer gets a plan, and in which mode.  The fold mode takes the
// narrow 3x3 layers it was made for (fold_build); the halo plan picks the
// per-tap mode itself for images not made of whole 16 x 8 tiles; shapes it refuses (e.g. more than kMaxPlanes stride-parity
// planes) get the per-tap mode forced, which takes every 32-channel multiple but no 8-channel input.
static bool tc_plan(const ConvProblem* probs, int nclass, const TcFormat& fmt, HaloPlan& plan) {
  if (nclass < 1 || nclass > 4) return false;
  for (int c = 0; c < nclass; ++c) {
    if (!tc_shape_supported(probs[c])) return false;
    if (probs[c].in != probs[0].in || probs[c].Cout != probs[0].Cout || probs[c].sy != probs[0].sy || probs[c].sx != probs[0].sx) return false;
  }
  return fold_build(probs, nclass, fmt, plan) || halo_build(probs, nclass, fmt, plan, false) ||
         halo_build(probs, nclass, fmt, plan, true);
}

// TMA descriptors: 5-D view {sx*C, W/sx, sy, H/sy, B} of the input slice, one box shape per plane
static bool encode_maps(const ConvProblem& p, HaloPlan& plan) {
  const HaloParams& prm = plan.prm;
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fp = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess)
    return false;
  EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(fp);
  const cuuint64_t cp = (cuuint64_t)p.in_pitch;
  cuuint64_t gdim[5] = {(cuuint64_t)(p.sx - 1) * cp + (cuuint64_t)p.Cin, (cuuint64_t)(p.Wi / p.sx), (cuuint64_t)p.sy,
                        (cuuint64_t)(p.Hi / p.sy), (cuuint64_t)p.B};
  cuuint64_t gstr[4] = {(cuuint64_t)p.sx * cp * 4, (cuuint64_t)p.Wi * cp * 4, (cuuint64_t)p.sy * p.Wi * cp * 4,
                        (cuuint64_t)p.Hi * p.Wi * cp * 4};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < prm.nplanes; ++i) {
    cuuint32_t box[5] = {(cuuint32_t)(prm.cin8 ? 8 : 32), (cuuint32_t)prm.planes[i].cols, 1, (cuuint32_t)prm.planes[i].rows,
                         (cuuint32_t)(prm.per_tap ? prm.tb : 1)};
    CUresult r = enc(&plan.maps.m[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(p.in), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, prm.cin8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return false;
  }
  for (int i = prm.nplanes; i < kMaxPlanes; ++i) plan.maps.m[i] = plan.maps.m[0];
  return true;
}

int tc_describe(const ConvProblem* probs, int nclass, int precision, char* buf, int buflen) {
  HaloPlan plan;
  if (!tc_plan(probs, nclass, tc_format(precision), plan)) return 0;
  const HaloParams& q = plan.prm;
  // per-tap mode: a pixel tile is tb images x th rows x tw columns (halo mode: 1 x 16 x 8, fold mode 1 x 12 x 16; the fold
  // mode's kind is "halo", its halo box, and `fold` the taps it puts into N)
  int n = snprintf(buf, buflen,
                   "halo %s mode %d n_tile %d x%d steps %d x %d chunks sa %d fold %d a_stage %d w_slot %d smem %d tiles %d ksplit %d wres %d tb %d th %d tw %d |",
                   q.per_tap ? "per-tap" : (q.cin8 ? "cin8" : "halo"), q.mode, q.n_tile, q.n_tiles, q.nsteps, q.k_chunks, q.sa, q.fold,
                   q.a_region_bytes, q.w_stage_bytes, plan.smem_bytes, q.total_tiles, q.ksplit, q.w_resident, q.per_tap ? q.tb : 1,
                   q.per_tap ? q.th : (q.fold ? kFoldH : kTileH), q.per_tap ? q.tw : (q.fold ? kFoldW : kTileW));
  for (int t = 0; t < q.nsteps && n < buflen - 32; ++t)
    n += snprintf(buf + n, buflen - n, " [c%x w%d+%d]", q.st_cmask[t], q.st_woff[t], q.st_wbytes[t]);
  return n;
}

static float tf32_round_h(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7F800000u) == 0x7F800000u) return x;
  u += 0x00000FFFu + ((u >> 13) & 1u);
  u &= 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

int tc_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision) {
  const ConvProblem& p = probs[0];
  const TcFormat fmt = tc_format(precision);
  std::unique_ptr<HaloPlan> plan(new HaloPlan());
  if (!tc_plan(probs, nclass, fmt, *plan)) return kTcNoPlan;
  if (!encode_maps(p, *plan)) return fail(DEMON_E_CUDA, "tc_prepare: tensor map encode failed");
  const HaloParams& prm = plan->prm;
  // weights: [n tile][chunk][step][class of the step] blocks of the precision's format (TcFormat: [W_hi | W_lo], W or FP16
  // W), n_tile rows x 32 K positions, K-major, pre-swizzled; K position k of a row holds input channel fmt.channel(k).
  // Fold mode: fold_n rows per block, row (tap of the step, co) with the tap's columns co8 = fold_n / fold apart.
  const int rows = prm.fold ? prm.fold_n : prm.n_tile;
  const size_t total = (size_t)prm.n_tiles * prm.k_chunks * prm.w_chunk_bytes;
  std::vector<unsigned char> packed(total, 0);
  for (int nt = 0; nt < prm.n_tiles; ++nt)
    for (int kc = 0; kc < prm.k_chunks; ++kc)
      for (int tt = 0; tt < prm.nsteps; ++tt) {
        int idx = 0;
        for (int cls = 0; cls < 4; ++cls) {
          if (!((prm.st_cmask[tt] >> cls) & 1)) continue;
          unsigned char* blk = packed.data() + ((size_t)nt * prm.k_chunks + kc) * prm.w_chunk_bytes + prm.st_woff[tt] + (size_t)idx * prm.cls_bytes;
          ++idx;
          for (int r = 0; r < rows; ++r) {
            int tap = prm.cin8 ? 0 : plan->st_tap[tt][cls], co = nt * prm.n_tile + r;
            if (prm.fold) {
              const int co8 = prm.fold_n / prm.fold;
              tap = (prm.fold == 3 ? 3 * tt : 0) + r / co8;   // taps in row-major order: 3 dy + dx
              co = r % co8;
            }
            for (int k = 0; k < 32; ++k) {
              const int kphys = fmt.channel(k);
              float w = 0.f;
              if (prm.cin8) {   // channel index = (tap within the group of four, channel)
                const int rt = 4 * tt + kphys / 8;
                if (co < p.Cout && rt < prm.ntaps_real) w = w_hosts[0][((size_t)plan->st_tap[rt][0] * 8 + (kphys & 7)) * p.Cout_pad + co];
              } else if (co < p.Cout) {
                w = w_hosts[cls][((size_t)tap * p.Cin + kc * 32 + kphys) * p.Cout_pad + co];
              }
              const size_t off = (size_t)fmt.offset(r, k);
              if (fmt.mode == 1) {   // FP16, round to nearest even; a weight FP16 cannot hold is refused, not made infinite
                if (!(std::fabs(w) <= 65504.f)) return kTcWeightRange;
                const __half h = __float2half_rn(w);
                memcpy(blk + off, &h, 2);
                continue;
              }
              const float hi = (fmt.mode == 2) ? tf32_round_h(w) : w;
              const float lo = w - hi;
              memcpy(blk + off, &hi, 4);
              if (fmt.mode == 2) memcpy(blk + (size_t)rows * 128 + off, &lo, 4);
            }
          }
        }
      }
  void* dw = nullptr;
  cudaError_t e = cudaMalloc(&dw, total);
  if (e == cudaSuccess) {
    e = cudaMemcpy(dw, packed.data(), total, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) cudaFree(dw);
  }
  if (e != cudaSuccess) return fail(DEMON_E_CUDA, "tc_prepare: %s", cudaGetErrorString(e));
  plan->prm.w = static_cast<const unsigned char*>(dw);
  t.per_tap = prm.per_tap != 0;
  t.splitk_bytes = (prm.ksplit > 1) ? (size_t)prm.ksplit * p.B * p.Hfull * p.Wfull * ((p.Cout + 3) / 4 * 4) * sizeof(float) : 0;
  t.plan = plan.release();
  return DEMON_OK;
}

void tc_layer_free(TcLayer& t) {
  if (t.plan) {
    cudaFree(const_cast<unsigned char*>(t.plan->prm.w));
    delete t.plan;
  }
  t.plan = nullptr;
}

// Per-DEVICE launch state (one process may drive several GPUs): the dynamic shared-memory attribute has to be set on
// every device a kernel is launched on, the SM count and the pipeline-timeout flag live on the device.
// tc_device_state() returns the state of the CURRENT device (cudaGetDevice), creating it on first use.
struct TcDeviceState {
  int device = -1;
  int sms = 132;
  int* err_dev = nullptr;   // device int: set to 1 by a bounded mbarrier wait that timed out
};

static TcDeviceState& tc_device_state() {
  constexpr int kMaxDevices = 64;
  static TcDeviceState states[kMaxDevices];
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) dev = 0;
  std::lock_guard<std::mutex> lock(mu);
  TcDeviceState& s = states[dev];
  if (s.device != dev) {
    s = TcDeviceState();
    s.device = dev;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    s.sms = sms > 0 ? sms : 132;
    if (cudaMalloc(&s.err_dev, sizeof(int)) == cudaSuccess) cudaMemset(s.err_dev, 0, sizeof(int));
    else s.err_dev = nullptr;
  }
  return s;
}

int tc_read_error_flag(bool clear) {
  TcDeviceState& ds = tc_device_state();
  if (!ds.err_dev) return 0;
  int v = 0;
  cudaMemcpy(&v, ds.err_dev, sizeof(int), cudaMemcpyDeviceToHost);
  if (v && clear) cudaMemset(ds.err_dev, 0, sizeof(int));
  return v;
}

static long long* g_timing_dev = nullptr;
void tc_halo_enable_timing(bool on) {
  if (on && !g_timing_dev) { cudaMalloc(&g_timing_dev, 256 * 16 * sizeof(long long)); }
  if (g_timing_dev) cudaMemset(g_timing_dev, 0, 256 * 16 * sizeof(long long));
  if (!on && g_timing_dev) { cudaFree(g_timing_dev); g_timing_dev = nullptr; }
}
int tc_halo_read_timing(long long* host, int nblocks) {
  if (!g_timing_dev) return -1;
  cudaMemcpy(host, g_timing_dev, (size_t)nblocks * 16 * sizeof(long long), cudaMemcpyDeviceToHost);
  return 0;
}

template <bool PER_TAP, bool CIN8, int MODE, int N, int NCLS, int FOLD = 0>
static int launch_variant(const HaloPlan* plan, const HaloParams& prm, int grid, cudaStream_t stream) {
  TcDeviceState& ds = tc_device_state();
  static int attr_device = -1;   // per instantiation: the device whose shared-memory limit was raised last
  if (attr_device != ds.device) {
    DEMON_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_halo_kernel<PER_TAP, CIN8, MODE, N, NCLS, FOLD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    attr_device = ds.device;
  }
  cudaError_t le = launch_pdl(conv_tc_halo_kernel<PER_TAP, CIN8, MODE, N, NCLS, FOLD>, dim3(grid), dim3(kThreads), (size_t)plan->smem_bytes, stream, plan->maps, prm);
  if (le != cudaSuccess) return fail(DEMON_E_CUDA, "conv_tc_halo launch: %s", cudaGetErrorString(le));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

template <bool PER_TAP, bool CIN8, int MODE, int NCLS>
static int launch_n(const HaloPlan* plan, const HaloParams& prm, int grid, cudaStream_t stream) {
  switch (prm.n_tile) {
    case 16: return launch_variant<PER_TAP, CIN8, MODE, 16, NCLS>(plan, prm, grid, stream);
    case 32: return launch_variant<PER_TAP, CIN8, MODE, 32, NCLS>(plan, prm, grid, stream);
    case 64: return launch_variant<PER_TAP, CIN8, MODE, 64, NCLS>(plan, prm, grid, stream);
    default: break;
  }
  if (NCLS == 1 && prm.n_tile == 128) return launch_variant<PER_TAP, CIN8, MODE, (NCLS == 1 ? 128 : 64), NCLS>(plan, prm, grid, stream);
  return fail(DEMON_E_STATE, "conv_tc_halo: no kernel for N tile %d with %d classes", prm.n_tile, prm.nclass);
}

template <bool PER_TAP, bool CIN8, int NCLS>
static int launch_mode(const HaloPlan* plan, const HaloParams& prm, int grid, cudaStream_t stream) {
  switch (prm.mode) {
    case 0: return launch_n<PER_TAP, CIN8, 0, NCLS>(plan, prm, grid, stream);
    case 1: return launch_n<PER_TAP, CIN8, 1, NCLS>(plan, prm, grid, stream);
    default: return launch_n<PER_TAP, CIN8, 2, NCLS>(plan, prm, grid, stream);
  }
}

template <int FOLD, int N>
static int launch_fold(const HaloPlan* plan, const HaloParams& prm, int grid, cudaStream_t stream) {
  if (prm.fold_n != N) return fail(DEMON_E_STATE, "conv_tc_halo: no fold kernel for %d taps at N %d", prm.fold, prm.fold_n);
  switch (prm.mode) {
    case 0: return launch_variant<false, false, 0, N, 1, FOLD>(plan, prm, grid, stream);
    case 1: return launch_variant<false, false, 1, N, 1, FOLD>(plan, prm, grid, stream);
    default: return launch_variant<false, false, 2, N, 1, FOLD>(plan, prm, grid, stream);
  }
}

int conv_tc_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream) {
  const HaloPlan* plan = t.plan;
  HaloParams prm = plan->prm;
  prm.out = probs[0].out;          // the output slice may be re-pointed between calls (caller-owned result buffers)
  prm.out_pitch = probs[0].out_pitch;
  TcDeviceState& ds = tc_device_state();
  if (!ds.err_dev) return fail(DEMON_E_CUDA, "tensor-core path: no error flag on device %d", ds.device);
  prm.err = ds.err_dev;
  prm.timing = g_timing_dev;
  const int cpitch = (prm.Cout + 3) / 4 * 4;
  const long long npix = (long long)prm.B * prm.Hfull * prm.Wfull;
  float* const final_out = prm.out;
  const int final_pitch = prm.out_pitch;
  if (prm.ksplit > 1) {   // partial sums into the caller's scratch, bias and activation in the second pass
    if (!probs[0].partial) return fail(DEMON_E_STATE, "conv_tc_halo: split-K layer launched without a scratch buffer");
    prm.out = probs[0].partial;
    prm.out_pitch = cpitch;
    prm.part_stride = npix * cpitch;
    prm.bias = nullptr;
    prm.leaky = 0;
  }
  const int grid = std::min(prm.total_items, ds.sms);
  int rc;
  if (prm.fold) rc = prm.fold == 9 ? launch_fold<9, 144>(plan, prm, grid, stream) : launch_fold<3, 72>(plan, prm, grid, stream);
  else if (prm.cin8) rc = launch_mode<false, true, 1>(plan, prm, grid, stream);
  else if (prm.per_tap) rc = prm.nclass == 1 ? launch_mode<true, false, 1>(plan, prm, grid, stream) : launch_mode<true, false, 4>(plan, prm, grid, stream);
  else rc = prm.nclass == 1 ? launch_mode<false, false, 1>(plan, prm, grid, stream) : launch_mode<false, false, 4>(plan, prm, grid, stream);
  if (rc != DEMON_OK || prm.ksplit == 1) return rc;
  const long long total = npix * (cpitch / 4);
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)ds.sms * 8);
  cudaError_t le = launch_pdl(halo_splitk_reduce_kernel, dim3(blocks), dim3(256), 0, stream, (const float*)probs[0].partial, prm.part_stride,
                              prm.ksplit, final_out, final_pitch, cpitch, prm.Cout, npix, plan->prm.bias, plan->prm.leaky);
  if (le != cudaSuccess) return fail(DEMON_E_CUDA, "halo_splitk_reduce launch: %s", cudaGetErrorString(le));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

}  // namespace demon
