// map.h — host-side handle of the hash-voxel map.
#pragma once
#include <algorithm>
#include <list>
#include <unordered_map>
#include <vector>

#include "lsd_common.cuh"

// iVox's LRU bookkeeping (ivox3d.h:231-256: grids_cache_ list + grids_map_), mirrored on the host when
// lsd_map_enable_lru is on.  The order of an LRU list is sequential by nature (one touch per inserted point, at most one
// eviction per inserted point); the point data stays on the device, only the voxel keys of each insert batch are replayed
// here and the resulting evictions are applied to the table by map_evict_kernel.
struct LruMirror {
  size_t capacity = 0;
  double max_distance = 100.0;      // IVox::Options::max_distance_
  double distance = 0.0;            // travel_distance handed to AddPoints
  struct Node { unsigned long long key; double d0; };
  std::list<Node> cache;            // front = most recently touched
  std::unordered_map<unsigned long long, std::list<Node>::iterator> idx;
  unsigned long long n_evicted = 0;
  unsigned long long tombstones = 0;   // lines retired since the last rehash
};

struct lsd_map {
  lsd::MapView view{};
  unsigned long long n_lines = 0;
  int device = 0;
  cudaStream_t stream = nullptr;
  void* scratch = nullptr;  // staging for the host-pointer entry points
  size_t scratch_bytes = 0;
  long long launches = 0;   // kernels launched on behalf of this handle
  int knn_shape = 0;        // lsd_knn_set_shape: 0 auto, 1 warp/query, 2 thread/query, 3 brick pages (TMA)
  // brick layout (lsd_map_enable_bricks, brick.cuh): directory size and the per-batch binning scratch
  unsigned long long n_bricks = 0;
  unsigned* bin_count = nullptr;   // [n_bricks], zero between batches
  int* bin_base = nullptr;         // [n_bricks]
  void* bscratch = nullptr;        // q_slot, q_rank, sorted, work items, counters of the batch in flight
  size_t bscratch_bytes = 0;
  LruMirror* lru = nullptr;        // lsd_map_enable_lru
  unsigned long long dropped_seen = 0;   // counters[2] at the last look (lsd_map_saturated)
  bool incomplete = false;   // a matcher's point map (build_point_map, reg.cu) refused points: its grid search is not exact
};

namespace lsd {
lsd_status_t upload_stencils();
lsd_status_t launch_insert(lsd_map* m, const float4* d_pts, int n, int id0, cudaStream_t st);
lsd_status_t launch_knn(lsd_map* m, const float4* d_q, int nq, int k, float max_sq, int stencil, int* d_idx, float* d_d2,
                        int* d_cnt, cudaStream_t st);
__device__ void map_insert_point(const MapView& mv, float x, float y, float z, int id);
// LRU replay of one AddPoints batch (host points in AddPoints order, ids id0 + i or ids[i]) and the eviction it causes
lsd_status_t map_lru_touch(lsd_map* m, const float4* pts_host, const int* ids_or_null, int n, int id0, cudaStream_t st);
}  // namespace lsd
