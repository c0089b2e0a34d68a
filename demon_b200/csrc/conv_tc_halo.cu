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
// Precision: 3xTF32 = A_hi * W_lo + A_lo * W_hi + A_hi * W_hi (W split on the host), three wgmma per K = 8 slice and
// class; the dropped term A_lo * W_lo is ~2^-21 relative.  nsplit = 1 is plain single-pass TF32.
//
// Narrow single-n-tile layers keep their whole packed weight set (<= 96 KB) RESIDENT in shared memory, loaded once per CTA
// instead of one small bulk copy per step.  Layers with few tiles split their K loop over several work items (split-K,
// halo_splitk_reduce_kernel).  Variants: PER_TAP (images that are not made of whole 16 x 8 tiles: one 128-pixel TMA box per
// step instead of a halo) and CIN8 (8-channel inputs: four taps x 8 channels per K = 32 step).
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "conv_tc.cuh"
#include "conv_tc_ptx.cuh"
#include "wgmma_tf32.cuh"

namespace demon {

namespace {

constexpr int kRing = 4;                 // weight ring slots
constexpr int kThreads = 384;            // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr int kMaxAStages = 4;
constexpr int kTileH = 16, kTileW = 8;
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
  HaloPlane planes[kMaxPlanes];
  int a_region_bytes;   // one halo stage (all planes)
  int sa;               // A (halo, shared memory) stages
  int w_chunk_bytes;    // weight bytes of one (n tile, chunk): sum of st_wbytes
  int w_stage_bytes;    // weight ring slot = the largest step
  int w_region_bytes;   // shared memory of the weights: kRing slots, or the whole layer when resident
  int w_resident;       // 1: ALL weight blocks of the (single) n tile live in shared memory for the whole kernel, loaded once
  int cls_bytes;        // one class block: [W_hi ; W_lo] (3xTF32) or W alone
  int n_tile, nsplit;
  int mode;             // 0 single pass TF32, 2 three-instruction 3xTF32
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

template <bool PER_TAP>
__device__ __forceinline__ void halo_decode_tile(const HaloParams& p, int tile, int& nt, int& n, int& y0, int& x0) {
  int m = fast_div(tile, p.n_tiles, p.mul_n_tiles);
  nt = tile - m * p.n_tiles;
  const int m1 = fast_div(m, p.tiles_x, p.mul_tiles_x);
  const int xb = m - m1 * p.tiles_x;
  n = fast_div(m1, p.tiles_y, p.mul_tiles_y);
  const int yb = m1 - n * p.tiles_y;
  if (PER_TAP) { n *= p.tb; y0 = yb * p.th; x0 = xb * p.tw; }
  else { y0 = yb * kTileH; x0 = xb * kTileW; }
}

// All wgmma of ONE class block of a step: K = 32 as four K = 8 slices.  hi/lo[8 j + 0..3] = the A fragment of slice j.
template <int N, int MODE>
__device__ __forceinline__ void issue_block(float* acc, const uint32_t* hi, const uint32_t* lo, uint32_t wb) {
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

template <bool PER_TAP, bool CIN8, int MODE, int N, int NCLS>
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
      halo_decode_tile<PER_TAP>(p, tile, nt, n, y0, x0);
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
    halo_decode_tile<PER_TAP>(p, tile, nt, n, y0, x0);
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
        // slice j: a0 = (row g, col tq) = v[0][2j], a1 = (row g + 8, col tq), a2 = (row g, col tq + 4) = v[0][2j + 1], a3
        uint32_t hi[16], lo[16];
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
static int popcount4(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1) + ((m >> 3) & 1); }

static bool w_resident_enabled() {   // DEMON_W_RESIDENT=0: weights always through the 4-slot ring (A/B measurements)
  static const bool v = []() { const char* e = getenv("DEMON_W_RESIDENT"); return !(e && e[0] == '0'); }();
  return v;
}

static bool splitk_enabled() {   // DEMON_TC_SPLITK=0: never split the K loop of a tensor-core layer (A/B measurements)
  static const bool v = []() { const char* e = getenv("DEMON_TC_SPLITK"); return !(e && e[0] == '0'); }();
  return v;
}

// Steps of one chunk: the distinct input shifts of all classes, each with the mask of the classes that use it.
// max_cls: at most this many classes per step (a wide step needs a wide weight slot; a shift is repeated if necessary).
struct ShiftStep { int ry, rx, qy, qx, cmask, tap[4]; };

static bool halo_build(const ConvProblem* probs, int nclass, int nsplit, HaloPlan& plan, bool encode, bool force_per_tap) {
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
    prm.nsplit = nsplit;
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
    prm.mode = (nsplit == 1) ? 0 : 2;
    prm.n_tile = n_tile;
    prm.n_tiles = ceil_div(p.Cout, n_tile);
    prm.k_chunks = prm.cin8 ? 1 : p.Cin / 32;
    // ---- weights: one class block = [W_hi ; W_lo] (3xTF32) or W alone, 1024-byte aligned; a step holds the blocks of its
    // classes in ascending class order; the ring slot is as large as the widest step
    prm.cls_bytes = (nsplit == 3) ? n_tile * 256 : (n_tile * 128 + 1023) / 1024 * 1024;
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
    if (w_resident_enabled() && !force_per_tap && nclass == 1 && prm.n_tiles == 1 && w_total <= 96 * 1024 && wmax * prm.nsteps == prm.w_chunk_bytes &&
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
  prm.B = p.B;
  const int m_tiles = prm.tiles_x * prm.tiles_y * prm.tiles_b;
  prm.total_tiles = m_tiles * prm.n_tiles;
  // ---- split-K: layers with few tiles and a long K loop (the 6x8 / 12x16 levels; everything at batch 1) leave most SMs
  // idle and run their K loop serially.  Cost model in cycles: rounds of kPlanSms items x (steps of an item x ~600 + ~3000
  // of prologue / epilogue), + ~12000 for the second pass + the partial sums' trip through L2; a split has to win 10 %.
  prm.ksplit = 1;
  if (splitk_enabled() && !prm.cin8 && !prm.w_resident && prm.k_chunks >= 4) {
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
  if (!encode) return true;
  // TMA descriptors: 5-D view {sx*C, W/sx, sy, H/sy, B} of the input slice, one box shape per plane
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

bool tc_halo_supported(const ConvProblem* probs, int nclass) {
  if (nclass < 1 || nclass > 4) return false;
  for (int c = 0; c < nclass; ++c) {
    ConvProblem q = probs[c];
    if (q.Cin == 8 && q.in_pitch == 8) q.Cin = 32;   // 8-channel mode: everything but the channel rule must hold
    if (!tc_layer_supported(q)) return false;
    if (probs[c].in != probs[0].in || probs[c].Cout != probs[0].Cout || probs[c].sy != probs[0].sy || probs[c].sx != probs[0].sx) return false;
  }
  HaloPlan plan;
  return halo_build(probs, nclass, 3, plan, false, false);
}

// debug: the plan halo_build chooses for a layer, as text (no device needed)
int tc_halo_describe(const ConvProblem* probs, int nclass, int nsplit, char* buf, int buflen) {
  HaloPlan plan;
  if (!halo_build(probs, nclass, nsplit, plan, false, false)) return snprintf(buf, buflen, "halo: unsupported");
  const HaloParams& q = plan.prm;
  int n = snprintf(buf, buflen, "halo %s mode %d n_tile %d x%d steps %d x %d chunks sa %d a_stage %d w_slot %d smem %d tiles %d ksplit %d wres %d |",
                   q.per_tap ? "per-tap" : (q.cin8 ? "cin8" : "halo"), q.mode, q.n_tile, q.n_tiles, q.nsteps, q.k_chunks, q.sa,
                   q.a_region_bytes, q.w_stage_bytes, plan.smem_bytes, q.total_tiles, q.ksplit, q.w_resident);
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

static int prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision, bool per_tap) {
  const ConvProblem& p = probs[0];
  const int nsplit = (precision == DEMON_PREC_TF32) ? 1 : 3;
  HaloPlan* plan = new HaloPlan();
  if (!halo_build(probs, nclass, nsplit, *plan, true, per_tap)) {
    delete plan;
    return fail(DEMON_E_CUDA, "tc_halo_prepare: could not build the plan (tensor map encode failed?)");
  }
  const HaloParams& prm = plan->prm;
  // weights: [n tile][chunk][step][class of the step] blocks of [W_hi | W_lo], n_tile rows x 32 fp32, K-major, pre-swizzled;
  // K position k of a row holds input channel kphys (the K order of the kernel's A fragment, see the top of this file)
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
          const int tap = prm.cin8 ? 0 : plan->st_tap[tt][cls];
          for (int r = 0; r < prm.n_tile; ++r) {
            const int co = nt * prm.n_tile + r;
            for (int k = 0; k < 32; ++k) {
              const int kk = k & 7, kphys = 8 * (kk & 3) + 2 * (k >> 3) + (kk >> 2);
              float w = 0.f;
              if (prm.cin8) {   // channel index = (tap within the group of four, channel)
                const int rt = 4 * tt + kphys / 8;
                if (co < p.Cout && rt < prm.ntaps_real) w = w_hosts[0][((size_t)plan->st_tap[rt][0] * 8 + (kphys & 7)) * p.Cout_pad + co];
              } else if (co < p.Cout) {
                w = w_hosts[cls][((size_t)tap * p.Cin + kc * 32 + kphys) * p.Cout_pad + co];
              }
              const float hi = (nsplit == 3) ? tf32_round_h(w) : w;
              const float lo = w - hi;
              const size_t off = (size_t)r * 128 + (size_t)(((k >> 2) ^ (r & 7)) << 4) + (size_t)(k & 3) * 4;
              memcpy(blk + off, &hi, 4);
              if (nsplit == 3) memcpy(blk + (size_t)prm.n_tile * 128 + off, &lo, 4);
            }
          }
        }
      }
  void* dw = nullptr;
  cudaError_t e = cudaMalloc(&dw, total);
  if (e == cudaSuccess) e = cudaMemcpy(dw, packed.data(), total, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { delete plan; return fail(DEMON_E_CUDA, "tc_halo_prepare: %s", cudaGetErrorString(e)); }
  plan->prm.w = static_cast<const unsigned char*>(dw);
  t.w_packed = dw;
  t.halo_plan = plan;
  t.per_tap = prm.per_tap;
  t.nclass = nclass;
  t.n_tile = prm.n_tile; t.n_tiles = prm.n_tiles; t.k_chunks = prm.k_chunks; t.nsplit = nsplit;
  t.th = kTileH; t.tw = kTileW; t.tb = 1; t.stages = prm.sa; t.smem_bytes = plan->smem_bytes;
  t.ksplit = prm.ksplit;
  t.splitk_bytes = (prm.ksplit > 1) ? (size_t)prm.ksplit * p.B * p.Hfull * p.Wfull * ((p.Cout + 3) / 4 * 4) * sizeof(float) : 0;
  return DEMON_OK;
}

int tc_halo_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision) {
  return prepare(t, probs, w_hosts, nclass, precision, false);
}

int tc_layer_prepare(TcLayer& t, const ConvProblem* probs, const float* const* w_hosts, int nclass, int precision) {
  DEMON_REQUIRE(nclass >= 1 && nclass <= 4, "tc_layer_prepare: nclass %d", nclass);
  for (int c = 0; c < nclass; ++c) DEMON_REQUIRE(tc_layer_supported(probs[c]), "tc_layer_prepare: unsupported shape");
  return prepare(t, probs, w_hosts, nclass, precision, true);
}

void tc_halo_free(TcLayer& t) {
  if (t.halo_plan) delete static_cast<HaloPlan*>(t.halo_plan);
  t.halo_plan = nullptr;
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

template <bool PER_TAP, bool CIN8, int MODE, int N, int NCLS>
static int launch_variant(const HaloPlan* plan, const HaloParams& prm, int grid, cudaStream_t stream) {
  TcDeviceState& ds = tc_device_state();
  static int attr_device = -1;   // per instantiation: the device whose shared-memory limit was raised last
  if (attr_device != ds.device) {
    DEMON_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_halo_kernel<PER_TAP, CIN8, MODE, N, NCLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    attr_device = ds.device;
  }
  cudaError_t le = launch_pdl(conv_tc_halo_kernel<PER_TAP, CIN8, MODE, N, NCLS>, dim3(grid), dim3(kThreads), (size_t)plan->smem_bytes, stream, plan->maps, prm);
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
  return prm.mode == 0 ? launch_n<PER_TAP, CIN8, 0, NCLS>(plan, prm, grid, stream) : launch_n<PER_TAP, CIN8, 2, NCLS>(plan, prm, grid, stream);
}

int conv_tc_halo_launch(const TcLayer& t, const ConvProblem* probs, cudaStream_t stream) {
  HaloPlan* plan = static_cast<HaloPlan*>(t.halo_plan);
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
  if (prm.cin8) rc = launch_mode<false, true, 1>(plan, prm, grid, stream);
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
