// Connected components of an indexed mesh and the removal of the small ones (include/demon_b200.h: demon_mesh_*).
//
// * cc_union_kernel: one thread per face unions (v0, v1) and (v1, v2) in a lock-free union-find over parent [V].  A tree's
//   root is its smallest vertex: a union hooks the larger of two roots under the smaller with atomicCAS (which fails, and
//   is retried from the new roots, when another thread hooked that root first), so every hook joins two trees whose roots
//   are their minima under the smaller root.  find halves the path it walks; a halving store writes an ancestor of the
//   vertex, which is smaller, so the invariant holds whatever the interleaving.
// * parent is read inside a kernel with relaxed device-scope loads.  Other threads write it through L2, and on Hopper a
//   plain load may keep hitting a stale L1 line: a CAS retry loop fed by stale reads need not make progress.
// * cc_flatten_kernel writes each vertex's root; the roots, in ascending index, are the components.  A tile scan of the
//   root flags (cc_rank_kernel, tile_offsets_kernel) gives each root its rank, and cc_label_kernel relabels every vertex
//   by its root's rank.  So the labels depend only on the faces, not on the order the unions ran in.
// * cc_sizes_kernel counts faces and vertices per component with integer atomics, aggregated over the lanes of a warp that
//   share a component.
// * The filter keeps a component by its triangle count (and the caller's selection): cc_filter_count_kernel counts the
//   kept vertices and faces per tile, and cc_filter_vertex_kernel / cc_filter_face_kernel write them at their scanned
//   offsets, so the output is a boolean-mask compaction in the input's order.
#include "common.cuh"
#include "tile_scan.cuh"
#include <cuda/atomic>
#include <cstdint>

namespace demon {
namespace {

constexpr int kCcThreads = 256;
constexpr int kCcWarps = kCcThreads / 32;
constexpr int kCcRounds = 8;
constexpr int kCcTile = kCcThreads * kCcRounds;   // round r of thread i handles item tile * kCcTile + r * kCcThreads + i

using ParentRef = cuda::atomic_ref<int, cuda::thread_scope_device>;

__device__ __forceinline__ int parent_of(int* parent, int x) { return ParentRef(parent[x]).load(cuda::memory_order_relaxed); }

// The root of x's tree, halving the path on the way: each visited vertex is pointed at its grandparent.
__device__ __forceinline__ int find_root(int* parent, int x) {
  int p = parent_of(parent, x);
  while (p != x) {
    const int g = parent_of(parent, p);
    if (g != p) ParentRef(parent[x]).store(g, cuda::memory_order_relaxed);   // x is not a root, and stays one
    x = g;
    p = parent_of(parent, x);
  }
  return x;
}

__device__ __forceinline__ void unite(int* parent, int a, int b) {
  for (;;) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    const int lo = min(a, b), hi = max(a, b);
    if (atomicCAS(parent + hi, hi, lo) == hi) return;
  }
}

__global__ void __launch_bounds__(kCcThreads) cc_init_kernel(int* __restrict__ parent, int nv) {
  const long v = (long)blockIdx.x * kCcThreads + threadIdx.x;
  if (v < nv) parent[v] = (int)v;
}

__global__ void __launch_bounds__(kCcThreads) cc_union_kernel(const int* __restrict__ faces, long nf, int* parent) {
  const long f = (long)blockIdx.x * kCcThreads + threadIdx.x;
  if (f >= nf) return;
  const int v0 = __ldg(faces + 3 * f), v1 = __ldg(faces + 3 * f + 1), v2 = __ldg(faces + 3 * f + 2);
  unite(parent, v0, v1);
  unite(parent, v1, v2);
}

// The number of set flags of one block's round, and the number set in lanes below this one.
struct Ballot {
  int below, warp_total;
  __device__ __forceinline__ explicit Ballot(bool flag) {
    const unsigned b = __ballot_sync(0xffffffffu, flag);
    const unsigned lane = threadIdx.x & 31;
    below = __popc(b & ((1u << lane) - 1u));
    warp_total = __popc(b);
  }
};

// Tile t's count of the items i < n with flag(i).
template <class Flag>
__device__ __forceinline__ void tile_count(long tile, long n, Flag flag, int* __restrict__ tile_counts) {
  __shared__ int s_warp[kCcWarps];
  const long base = tile * kCcTile + threadIdx.x;
  int c = 0;
  for (int r = 0; r < kCcRounds; ++r) {
    const long i = base + r * kCcThreads;
    c += Ballot(i < n && flag(i)).warp_total;
  }
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
#pragma unroll
    for (int q = 0; q < kCcWarps; ++q) s += s_warp[q];
    tile_counts[tile] = s;
  }
}

// emit(i, k) for each item i < n of tile t with flag(i), k its rank among all flagged items (tile_first[t] plus the
// flagged items before it in the tile).
template <class Flag, class Emit>
__device__ __forceinline__ void tile_ranks(long tile, long n, const int64_t* __restrict__ tile_first, Flag flag, Emit emit) {
  __shared__ int s_warp[kCcWarps];
  const int warp = threadIdx.x >> 5;
  const long base = tile * kCcTile + threadIdx.x;
  long row = tile_first[tile];
  for (int r = 0; r < kCcRounds; ++r) {
    const long i = base + r * kCcThreads;
    const bool f = i < n && flag(i);
    const Ballot b(f);
    __syncthreads();   // s_warp of the previous round has been read
    if ((threadIdx.x & 31) == 0) s_warp[warp] = b.warp_total;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int q = 0; q < kCcWarps; ++q) {
      const int v = s_warp[q];
      total += v;
      before += q < warp ? v : 0;
    }
    if (f) emit(i, row + before + b.below);
    row += total;
  }
}

// labels[v] = the root of v; tile_counts: the roots of each tile.
__global__ void __launch_bounds__(kCcThreads) cc_flatten_kernel(int* parent, int nv, int* __restrict__ labels, int* __restrict__ tile_counts) {
  tile_count(blockIdx.x, nv, [&](long v) {
    const int root = find_root(parent, (int)v);
    labels[v] = root;
    return root == v;
  }, tile_counts);
}

// parent[root] = the root's rank among the roots (the component's label).
__global__ void __launch_bounds__(kCcThreads) cc_rank_kernel(const int* __restrict__ labels, int nv, const int64_t* __restrict__ tile_first,
                                                             int* __restrict__ parent) {
  tile_ranks(blockIdx.x, nv, tile_first, [&](long v) { return labels[v] == v; }, [&](long v, long k) { parent[v] = (int)k; });
}

__global__ void __launch_bounds__(kCcThreads) cc_label_kernel(int* __restrict__ labels, int nv, const int* __restrict__ parent) {
  const long v = (long)blockIdx.x * kCcThreads + threadIdx.x;
  if (v < nv) labels[v] = parent[labels[v]];
}

// counters[c] += 1 for each active lane's component c: one atomic per distinct c in the warp.
__device__ __forceinline__ void count_aggregated(unsigned long long* counters, bool active, int c) {
  const unsigned act = __ballot_sync(0xffffffffu, active);
  if (!active) return;
  const unsigned peers = __match_any_sync(act, c);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(counters + c, (unsigned long long)__popc(peers));
}

__global__ void __launch_bounds__(kCcThreads) cc_sizes_kernel(const int* __restrict__ faces, long nf, const int* __restrict__ labels, int nv,
                                                              unsigned long long* triangles, unsigned long long* vertices) {
  const long i = (long)blockIdx.x * kCcThreads + threadIdx.x;
  count_aggregated(triangles, i < nf, i < nf ? __ldg(labels + __ldg(faces + 3 * i)) : 0);
  count_aggregated(vertices, i < nv, i < nv ? __ldg(labels + i) : 0);
}

// Whether component c is kept: at least min_triangles triangles, and selected when the caller passes a selection.
struct Keep {
  const int64_t* triangles;
  int64_t min_triangles;
  const uint8_t* select;
  __device__ __forceinline__ bool operator()(int c) const {
    return __ldg(triangles + c) >= min_triangles && (!select || __ldg(select + c));
  }
};

struct FilterArgs {
  const int* faces;
  long nf;
  const int* labels;
  int nv;
  Keep keep;
  __device__ __forceinline__ bool vertex_kept(long v) const { return keep(__ldg(labels + v)); }
  __device__ __forceinline__ bool face_kept(long f) const { return keep(__ldg(labels + __ldg(faces + 3 * f))); }
};

// Blocks 0 .. vtiles-1 count the kept vertices of their tiles, the rest the kept faces.
__global__ void __launch_bounds__(kCcThreads) cc_filter_count_kernel(FilterArgs a, int vtiles, int* __restrict__ vcounts, int* __restrict__ fcounts) {
  if ((int)blockIdx.x < vtiles)
    tile_count(blockIdx.x, a.nv, [&](long v) { return a.vertex_kept(v); }, vcounts);
  else
    tile_count(blockIdx.x - vtiles, a.nf, [&](long f) { return a.face_kept(f); }, fcounts);
}

// Each kept vertex's new index into remap, and its attributes copied bit for bit.
__global__ void __launch_bounds__(kCcThreads) cc_filter_vertex_kernel(FilterArgs a, const int64_t* __restrict__ vfirst, int* __restrict__ remap,
                                                                      const unsigned* __restrict__ vertices, const unsigned* __restrict__ normals,
                                                                      const uint8_t* __restrict__ colors, unsigned* __restrict__ out_vertices,
                                                                      unsigned* __restrict__ out_normals, uint8_t* __restrict__ out_colors) {
  tile_ranks(blockIdx.x, a.nv, vfirst, [&](long v) { return a.vertex_kept(v); }, [&](long v, long k) {
    remap[v] = (int)k;
#pragma unroll
    for (int q = 0; q < 3; ++q) out_vertices[3 * k + q] = __ldg(vertices + 3 * v + q);
    if (normals) {
#pragma unroll
      for (int q = 0; q < 3; ++q) out_normals[3 * k + q] = __ldg(normals + 3 * v + q);
    }
    if (colors) {
#pragma unroll
      for (int q = 0; q < 3; ++q) out_colors[3 * k + q] = __ldg(colors + 3 * v + q);
    }
  });
}

// Each kept face at its rank, every corner replaced by its vertex's new index.
__global__ void __launch_bounds__(kCcThreads) cc_filter_face_kernel(FilterArgs a, const int64_t* __restrict__ ffirst, const int* __restrict__ remap,
                                                                    int* __restrict__ out_faces) {
  tile_ranks(blockIdx.x, a.nf, ffirst, [&](long f) { return a.face_kept(f); }, [&](long f, long k) {
#pragma unroll
    for (int q = 0; q < 3; ++q) out_faces[3 * k + q] = __ldg(remap + __ldg(a.faces + 3 * f + q));
  });
}

long cc_tiles(long n) { return (n + kCcTile - 1) / kCcTile; }

// The scratch of V vertices and F faces: vertex tile_first int64 [vt], face tile_first int64 [ft], parent (the
// components) or remap (the filter) int [V], vertex tile counts int [vt], face tile counts int [ft].
struct CcScratch {
  int64_t* vfirst;
  int64_t* ffirst;
  int* parent;
  int* vcounts;
  int* fcounts;
  int vtiles, ftiles;
  CcScratch(void* scratch, int nv, long nf) : vtiles((int)cc_tiles(nv)), ftiles((int)cc_tiles(nf)) {
    vfirst = static_cast<int64_t*>(scratch);
    ffirst = vfirst + vtiles;
    parent = reinterpret_cast<int*>(ffirst + ftiles);
    vcounts = parent + nv;
    fcounts = vcounts + vtiles;
  }
  static int64_t bytes(int nv, long nf) {
    return (cc_tiles(nv) + cc_tiles(nf)) * (int64_t)(sizeof(int64_t) + sizeof(int)) + (int64_t)nv * sizeof(int);
  }
};

int check_mesh(const char* name, const int* faces, int64_t nf, int nv) {
  DEMON_REQUIRE(nv >= 0 && nf >= 0 && nf <= (INT64_C(1) << 40), "%s: bad mesh of %d vertices and %lld faces", name, nv, (long long)nf);
  DEMON_REQUIRE(nv > 0 || nf == 0, "%s: %lld faces but no vertices", name, (long long)nf);
  DEMON_REQUIRE(faces || nf == 0, "%s: null faces", name);
  return DEMON_OK;
}

int check_filter(const char* name, const int* faces, int64_t nf, const int* labels, int nv, const int64_t* triangles, int64_t min_triangles) {
  if (int rc = check_mesh(name, faces, nf, nv)) return rc;
  DEMON_REQUIRE(min_triangles >= 0, "%s: min_triangles must be >= 0, got %lld", name, (long long)min_triangles);
  DEMON_REQUIRE(nv == 0 || (labels && triangles), "%s: null pointer", name);
  return DEMON_OK;
}

}  // namespace
}  // namespace demon

using namespace demon;

extern "C" {

int64_t demon_mesh_components_scratch_bytes(int num_vertices, int64_t num_faces) {
  if (num_vertices < 0 || num_faces < 0 || num_faces > (INT64_C(1) << 40)) return 0;
  return CcScratch::bytes(num_vertices, num_faces);
}

int demon_mesh_components_count(const int* faces, int64_t num_faces, int num_vertices, void* scratch, int* labels, int64_t* components,
                                void* stream) {
  if (int rc = check_mesh("mesh_components_count", faces, num_faces, num_vertices)) return rc;
  DEMON_REQUIRE(components, "mesh_components_count: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (num_vertices == 0) {
    DEMON_CHECK_CUDA(cudaMemsetAsync(components, 0, sizeof(int64_t), st));
    return DEMON_OK;
  }
  DEMON_REQUIRE(scratch && labels, "mesh_components_count: null pointer");
  const CcScratch sc(scratch, num_vertices, num_faces);
  cc_init_kernel<<<(unsigned)ceil_div64(num_vertices, kCcThreads), kCcThreads, 0, st>>>(sc.parent, num_vertices);
  DEMON_LAUNCH_CHECK();
  if (num_faces) {
    cc_union_kernel<<<(unsigned)ceil_div64(num_faces, kCcThreads), kCcThreads, 0, st>>>(faces, num_faces, sc.parent);
    DEMON_LAUNCH_CHECK();
  }
  cc_flatten_kernel<<<sc.vtiles, kCcThreads, 0, st>>>(sc.parent, num_vertices, labels, sc.vcounts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(sc.vcounts, sc.vtiles, sc.vfirst, components);
  DEMON_LAUNCH_CHECK();
  cc_rank_kernel<<<sc.vtiles, kCcThreads, 0, st>>>(labels, num_vertices, sc.vfirst, sc.parent);
  DEMON_LAUNCH_CHECK();
  cc_label_kernel<<<(unsigned)ceil_div64(num_vertices, kCcThreads), kCcThreads, 0, st>>>(labels, num_vertices, sc.parent);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_mesh_component_sizes(const int* faces, int64_t num_faces, const int* labels, int num_vertices, int64_t components,
                               int64_t* triangles, int64_t* vertices, void* stream) {
  if (int rc = check_mesh("mesh_component_sizes", faces, num_faces, num_vertices)) return rc;
  DEMON_REQUIRE(components >= 0 && components <= num_vertices && (components > 0) == (num_vertices > 0),
                "mesh_component_sizes: %lld components of %d vertices", (long long)components, num_vertices);
  if (num_vertices == 0) return DEMON_OK;
  DEMON_REQUIRE(labels && triangles && vertices, "mesh_component_sizes: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  DEMON_CHECK_CUDA(cudaMemsetAsync(triangles, 0, components * sizeof(int64_t), st));
  DEMON_CHECK_CUDA(cudaMemsetAsync(vertices, 0, components * sizeof(int64_t), st));
  const int64_t n = num_faces > num_vertices ? num_faces : num_vertices;
  cc_sizes_kernel<<<(unsigned)ceil_div64(n, kCcThreads), kCcThreads, 0, st>>>(faces, num_faces, labels, num_vertices,
                                                                              reinterpret_cast<unsigned long long*>(triangles),
                                                                              reinterpret_cast<unsigned long long*>(vertices));
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_mesh_filter_count(const int* faces, int64_t num_faces, const int* labels, int num_vertices, const int64_t* triangles,
                            int64_t min_triangles, const uint8_t* select, void* scratch, int64_t* counts, void* stream) {
  if (int rc = check_filter("mesh_filter_count", faces, num_faces, labels, num_vertices, triangles, min_triangles)) return rc;
  DEMON_REQUIRE(counts, "mesh_filter_count: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (num_vertices == 0) {
    DEMON_CHECK_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), st));
    return DEMON_OK;
  }
  DEMON_REQUIRE(scratch, "mesh_filter_count: null pointer");
  const CcScratch sc(scratch, num_vertices, num_faces);
  const FilterArgs a{faces, (long)num_faces, labels, num_vertices, Keep{triangles, min_triangles, select}};
  cc_filter_count_kernel<<<sc.vtiles + sc.ftiles, kCcThreads, 0, st>>>(a, sc.vtiles, sc.vcounts, sc.fcounts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(sc.vcounts, sc.vtiles, sc.vfirst, counts);
  DEMON_LAUNCH_CHECK();
  tile_offsets_kernel<<<1, kScanThreads, 0, st>>>(sc.fcounts, sc.ftiles, sc.ffirst, counts + 1);
  DEMON_LAUNCH_CHECK();
  return DEMON_OK;
}

int demon_mesh_filter(const int* faces, int64_t num_faces, const int* labels, int num_vertices, const int64_t* triangles,
                      int64_t min_triangles, const uint8_t* select, void* scratch, const float* vertices, const float* normals,
                      const uint8_t* colors, float* out_vertices, float* out_normals, uint8_t* out_colors, int* out_faces, void* stream) {
  if (int rc = check_filter("mesh_filter", faces, num_faces, labels, num_vertices, triangles, min_triangles)) return rc;
  DEMON_REQUIRE(!normals == !out_normals && !colors == !out_colors, "mesh_filter: an attribute and its output go together");
  if (num_vertices == 0) return DEMON_OK;
  DEMON_REQUIRE(scratch && vertices && out_vertices, "mesh_filter: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const CcScratch sc(scratch, num_vertices, num_faces);
  const FilterArgs a{faces, (long)num_faces, labels, num_vertices, Keep{triangles, min_triangles, select}};
  cc_filter_vertex_kernel<<<sc.vtiles, kCcThreads, 0, st>>>(a, sc.vfirst, sc.parent, reinterpret_cast<const unsigned*>(vertices),
                                                            reinterpret_cast<const unsigned*>(normals), colors,
                                                            reinterpret_cast<unsigned*>(out_vertices), reinterpret_cast<unsigned*>(out_normals),
                                                            out_colors);
  DEMON_LAUNCH_CHECK();
  if (num_faces && out_faces) {
    cc_filter_face_kernel<<<sc.ftiles, kCcThreads, 0, st>>>(a, sc.ffirst, sc.parent, out_faces);
    DEMON_LAUNCH_CHECK();
  }
  return DEMON_OK;
}

}  // extern "C"
