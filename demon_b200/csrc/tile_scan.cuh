// The single-CTA exclusive scan of per-tile counts shared by the marching cubes, the indexed mesh (csrc/fusion.cu) and
// the mesh components (csrc/mesh.cu).  The tiles are summed in a fixed order, so the result does not depend on
// scheduling.
#pragma once
#include <cstdint>

namespace demon {
namespace {

constexpr int kScanThreads = 1024;

// One CTA: tile_first[t] = the counts of tiles 0..t-1, and *total = all of them.
__global__ void __launch_bounds__(kScanThreads) tile_offsets_kernel(const int* __restrict__ tile_counts, int tiles,
                                                                    int64_t* __restrict__ tile_first, int64_t* __restrict__ total) {
  __shared__ int64_t s_sum[kScanThreads];
  const int seg = (tiles + kScanThreads - 1) / kScanThreads;
  const int b = threadIdx.x * seg, e = min(tiles, b + seg);
  int64_t s = 0;
  for (int q = b; q < e; ++q) s += tile_counts[q];
  s_sum[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {   // 1024 additions: not worth a tree
    int64_t run = 0;
    for (int q = 0; q < kScanThreads; ++q) {
      const int64_t v = s_sum[q];
      s_sum[q] = run;
      run += v;
    }
    *total = run;
  }
  __syncthreads();
  int64_t run = s_sum[threadIdx.x];
  for (int q = b; q < e; ++q) {
    tile_first[q] = run;
    run += tile_counts[q];
  }
}

}  // namespace
}  // namespace demon
