// map.cu — hash-voxel map build/insert (K2) and batched k-NN query (K3) + their C ABI.
//
// Replaces faster_lio::IVox (reference: slam/mapping/fastlio/include/ivox3d/ivox3d.h):
//   AddPoints :231-256  -> map_insert_kernel      (open addressing, 64-bit atomicCAS claim,
//                                                  atomicAdd slot claim, float4 stores)
//   GetClosestPoint :139-171 -> knn_query_kernel   (knn.cuh)
// The table is sized for the whole map in HBM (80 GB on an H100); the reference's capacity / LRU eviction
// (ivox3d.h:246-255) is available on request (lsd_map_enable_lru: map_lru_touch + map_evict_kernel below).
#include <stdarg.h>
#include <stdlib.h>

#include <mutex>

#include "knn.cuh"
#include "map.h"

namespace lsd {

// ------------------------------------------------------------------ error plumbing
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
lsd_status_t cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
  bool nodev = e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice;
  cudaGetLastError();
  return nodev ? LSD_ERR_NO_DEVICE : LSD_ERR_CUDA;
}
static thread_local int g_device = 0;
lsd_status_t ensure_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device available (%s): liblsdreg has no CPU fallback", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return LSD_ERR_NO_DEVICE;
  }
  LSD_CUDA(cudaSetDevice(g_device));
  return LSD_OK;
}

// ------------------------------------------------------------------ stencil tables (ivox3d.h:178-215)
static Stencil h_stencils[5];
static std::once_flag g_stencil_once;
static void build_stencils() {
  static const signed char n18[19][3] = {{0,0,0},{-1,0,0},{1,0,0},{0,1,0},{0,-1,0},{0,0,-1},{0,0,1},{1,1,0},{-1,1,0},
    {1,-1,0},{-1,-1,0},{1,0,1},{-1,0,1},{1,0,-1},{-1,0,-1},{0,1,1},{0,-1,1},{0,1,-1},{0,-1,-1}};
  memset(h_stencils, 0, sizeof(h_stencils));
  h_stencils[0].n = 1;
  h_stencils[1].n = 7; memcpy(h_stencils[1].off, n18, 7 * 3);
  h_stencils[2].n = 19; memcpy(h_stencils[2].off, n18, 19 * 3);
  static const signed char corners[8][3] = {{1,1,1},{-1,1,1},{1,-1,1},{1,1,-1},{-1,-1,1},{-1,1,-1},{1,-1,-1},{-1,-1,-1}};   // ivox3d.h:196-198
  h_stencils[3].n = 27; memcpy(h_stencils[3].off, n18, 19 * 3); memcpy(h_stencils[3].off[19], corners, 8 * 3);
  for (int i = -2; i <= 2; i++) for (int j = -2; j <= 2; j++) for (int k = -1; k <= 1; k++) {
    signed char* o = h_stencils[4].off[h_stencils[4].n++]; o[0] = i; o[1] = j; o[2] = k; }
}
const Stencil* host_stencil(int type) {
  std::call_once(g_stencil_once, build_stencils);
  int s = stencil_slot(type);
  return s < 0 ? nullptr : &h_stencils[s];
}
lsd_status_t upload_stencils() {
  std::call_once(g_stencil_once, build_stencils);
  LSD_CUDA(cudaMemcpyToSymbol(c_stencils, h_stencils, sizeof(h_stencils)));
  return LSD_OK;
}

// K best candidates of one thread in registers, canonical ascending (d2, id) order (thread-per-query shapes)
template <int K>
struct TopK {
  float d[K]; int id[K];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < K; i++) { d[i] = 3.0e38f; id[i] = 0x7fffffff; }
  }
  // insert (d2, pid) keeping ascending (d2, id) order; fully unrolled compare-exchange chain (registers only)
  __device__ __forceinline__ bool push(float d2, int pid) {
    if (!(d2 < d[K - 1] || (d2 == d[K - 1] && pid < id[K - 1]))) return false;
    d[K - 1] = d2; id[K - 1] = pid;
#pragma unroll
    for (int i = K - 1; i > 0; i--) {
      const bool sw = d[i] < d[i - 1] || (d[i] == d[i - 1] && id[i] < id[i - 1]);
      const float td = d[i]; const int ti = id[i];
      d[i] = sw ? d[i - 1] : d[i]; id[i] = sw ? id[i - 1] : id[i];
      d[i - 1] = sw ? td : d[i - 1]; id[i - 1] = sw ? ti : id[i - 1];
    }
    return true;
  }
};

}  // namespace lsd
#include "brick.cuh"
namespace lsd {

// ------------------------------------------------------------------ K2: insert
__device__ __forceinline__ long long find_or_claim(const MapView& mv, unsigned long long key, bool* fresh) {
  const unsigned long long h = hash_key(key);
  unsigned long long s = h & mv.mask;
  *fresh = false;
  for (unsigned probe = 0; probe < kMaxProbe; probe++) {
    unsigned long long* kp = &mv.lines[s].key;
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(kp);
    if (cur == key) return (long long)s;
    if (cur == 0ull) {
      unsigned long long old = atomicCAS(kp, 0ull, key);
      if (old == 0ull) { mv.tags[s] = (unsigned char)slot_tag(h); *fresh = true; return (long long)s; }
      if (old == key) return (long long)s;
    }
    s = (s + 1) & mv.mask;
  }
  return -1;
}

// Insert one point (device function shared with map_incremental in lio.cu).
__device__ void map_insert_point(const MapView& mv, float x, float y, float z, int id) {
  int3 c = pos2grid(x, y, z, mv.inv_res);
  if (!coord_ok(c.x, c.y, c.z)) { atomicAdd(&mv.counters[2], 1ull); return; }
  if (!shard_relevant(mv, c.x, c.y)) return;  // another rank's tile and not in our halo
  unsigned long long key0 = pack_key(c.x, c.y, c.z, 0);
  bool fresh;
  long long s = find_or_claim(mv, key0, &fresh);
  if (s < 0) { atomicAdd(&mv.counters[2], 1ull); return; }
  if (fresh) atomicAdd(&mv.counters[0], 1ull);
  unsigned pos = atomicAdd(&mv.lines[s].count, 1u);
  unsigned L = pos / kPtsPerLine, j = pos % kPtsPerLine;
  if (L > 0) {
    if (L > (unsigned)kMaxLevel) { atomicAdd(&mv.counters[2], 1ull); return; }
    s = find_or_claim(mv, key0 | ((unsigned long long)L << 57), &fresh);
    if (s < 0) { atomicAdd(&mv.counters[2], 1ull); return; }
  }
  mv.lines[s].pts[j] = make_float4(x, y, z, __int_as_float(id));
  atomicAdd(&mv.counters[1], 1ull);
  if (mv.bricks.keys) brick_insert_point(mv.bricks, c.x, c.y, c.z, make_float4(x, y, z, __int_as_float(id)));
}

__global__ void __launch_bounds__(256) map_insert_kernel(MapView mv, const float4* __restrict__ pts, int n, int id0) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = __ldg(pts + i);  // coalesced 16-byte loads
  map_insert_point(mv, p.x, p.y, p.z, id0 + i);
}

// ------------------------------------------------------------------ K3: batched k-NN query
constexpr int kKnnWarps = 8;
constexpr int kThreadKnnMin = 1 << 16;  // from this many queries on, lsd_knn_query* uses the thread-per-query kernel
template <int K>
__global__ void __launch_bounds__(kKnnWarps * 32, 5) knn_query_kernel(MapView mv, const float4* __restrict__ q, int nq, float max_sq,
                                                                   int stencil, int* __restrict__ out_idx,
                                                                   float* __restrict__ out_d2, int* __restrict__ out_cnt) {
  __shared__ __align__(16) unsigned char s_list[kKnnWarps * kWarpListBytes];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpList wl = make_warp_list(s_list, warp);
  const LaneStencil ls = lane_stencil(stencil_slot(stencil));
  for (int i = blockIdx.x * kKnnWarps + warp; i < nq; i += gridDim.x * kKnnWarps) {
    const float4 p = __ldg(q + i);
    Neighbor nb;
    const int nf = knn_search_warp<K>(mv, stencil, ls, p.x, p.y, p.z, max_sq, wl, nb);
    if (lane < K) {
      out_idx[(size_t)i * K + lane] = lane < nf ? nb.id : -1;
      out_d2[(size_t)i * K + lane] = lane < nf ? nb.d2 : -1.0f;
    }
    if (lane == 0) out_cnt[i] = nf;
  }
}

// ---- batched variant: one THREAD per query.
// With millions of queries in flight there is no need to spread one query over a warp: a thread walks
// its stencil cells serially (tag probe in L2, line fetch only for voxels that exist) and keeps the K best
// in registers, in canonical (d2, id) order.  ~12x fewer warp instructions per query than the warp-per-query
// kernel, which stays the right shape for a single scan's 10-40 k queries (latency, not throughput).
// resolve `key` through the tag array (see warp_scan_cells); returns the line or nullptr
__device__ __forceinline__ const CellLine* tag_find(const MapView& mv, unsigned long long key, uint4* hdr) {
  constexpr unsigned long long k01 = 0x0101010101010101ull, k7f = 0x7f7f7f7f7f7f7f7full;
  const unsigned long long hh = hash_key(key);
  const unsigned long long tagv = (unsigned long long)slot_tag(hh) * k01;
  unsigned long long s = hh & mv.mask;
  for (unsigned walked = 0; walked < kMaxProbe;) {
    const unsigned pos = (unsigned)(s & 7ull), nv = 8u - pos;
    const unsigned long long v = __ldg(reinterpret_cast<const unsigned long long*>(mv.tags + (s & ~7ull))) >> (8u * pos);
    const unsigned long long ze = ~(((v & k7f) + k7f) | v | k7f);
    const unsigned long long x = v ^ tagv;
    unsigned long long zm = ~(((x & k7f) + k7f) | x | k7f);
    const unsigned fe = ze ? (unsigned)(__ffsll((long long)ze) - 1) >> 3 : 8u;
    while (zm) {
      const unsigned fm = (unsigned)(__ffsll((long long)zm) - 1) >> 3;
      if (fm >= fe) break;
      zm &= zm - 1ull;
      const CellLine* cl = mv.lines + ((s + fm) & mv.mask);
      const uint4 h = ldg_u4(cl);
      if (((unsigned long long)h.x | ((unsigned long long)h.y << 32)) == key) { *hdr = h; return cl; }
    }
    if (fe < nv) return nullptr;
    walked += nv;
    s = (s + nv) & mv.mask;
  }
  return nullptr;
}

template <int K>
__global__ void __launch_bounds__(256) knn_query_thread_kernel(MapView mv, const float4* __restrict__ q, int nq, float max_sq,
                                                               int st_slot, int* __restrict__ out_idx, float* __restrict__ out_d2,
                                                               int* __restrict__ out_cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const float4 p = __ldg(q + i);
  const int3 c = pos2grid(p.x, p.y, p.z, mv.inv_res);
  const Stencil& st = c_stencils[st_slot];
  TopK<K> best;
  best.init();
  int found = 0;
#pragma unroll 1
  for (int o = 0; o < st.n; o++) {
    const int x = c.x + st.off[o][0], y = c.y + st.off[o][1], z = c.z + st.off[o][2];
    if (!coord_ok(x, y, z)) continue;
    const unsigned long long key = pack_key(x, y, z, 0);
    uint4 h;
    const CellLine* ln = tag_find(mv, key, &h);
    if (!ln) continue;
    const unsigned cnt = h.z;
    const unsigned n0 = min(cnt, (unsigned)kPtsPerLine);
#pragma unroll 1
    for (unsigned j = 0; j < n0; j++) {
      const float4 a = ldg_f4(&ln->pts[j]);
      const float d2 = dist2(p.x, p.y, p.z, a.x, a.y, a.z);
      if (d2 < max_sq) { found++; best.push(d2, __float_as_int(a.w)); }
    }
    if (cnt > (unsigned)kPtsPerLine) {  // overflow levels (rare in a 0.5 m-thinned map)
      const int levels = min((int)((cnt - 1) / kPtsPerLine), kMaxLevel);
      for (int L = 1; L <= levels; L++) {
        uint4 hl;
        const CellLine* ll = tag_find(mv, key | ((unsigned long long)L << 57), &hl);
        if (!ll) continue;
        const int n = (int)min(cnt - (unsigned)(L * kPtsPerLine), (unsigned)kPtsPerLine);
        for (int j = 0; j < n; j++) {
          const float4 a = ldg_f4(&ll->pts[j]);
          const float d2 = dist2(p.x, p.y, p.z, a.x, a.y, a.z);
          if (d2 < max_sq) { found++; best.push(d2, __float_as_int(a.w)); }
        }
      }
    }
  }
  const int nf = min(found, K);
#pragma unroll
  for (int r = 0; r < K; r++) {
    out_idx[(size_t)i * K + r] = r < nf ? best.id[r] : -1;
    out_d2[(size_t)i * K + r] = r < nf ? best.d[r] : -1.0f;
  }
  out_cnt[i] = nf;
}

// ------------------------------------------------------------------ box delete
// KD_TREE::Delete_Point_Boxes (ikd_Tree.cpp:536-556; Delete_by_range :648-672): a point is deleted iff
// min <= p < max on every axis, for any box.  Deleted points keep their slot and get NaN coordinates: every
// distance to them is NaN, every `d2 < max_sq` test false, so no query can return them and no table entry moves.
constexpr int kMaxDeleteBoxes = 16;
struct DeleteBoxes { int n; float b[kMaxDeleteBoxes][6]; };

__global__ void __launch_bounds__(256) map_delete_boxes_kernel(MapView mv, unsigned long long n_lines, DeleteBoxes bx,
                                                               unsigned long long* __restrict__ n_deleted) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_lines) return;
  CellLine* ln = mv.lines + s;
  const unsigned long long key = ln->key;
  if (key == 0ull) return;
  const int level = (int)(key >> 57);
  unsigned total = ln->count;
  if (level > 0) {  // points 7L.. of a crowded voxel: the voxel's total count lives in its level-0 line
    uint4 h;
    const CellLine* base = tag_find(mv, key & ((1ull << 57) - 1ull), &h);
    if (!base) return;
    total = h.z;
  }
  const int n = (int)min(total > (unsigned)(level * kPtsPerLine) ? total - (unsigned)(level * kPtsPerLine) : 0u, (unsigned)kPtsPerLine);
  unsigned del = 0;
  for (int j = 0; j < n; j++) {
    const float4 p = ln->pts[j];
    bool inside = false;
    for (int b = 0; b < bx.n && !inside; b++)
      inside = bx.b[b][0] <= p.x && bx.b[b][3] > p.x && bx.b[b][1] <= p.y && bx.b[b][4] > p.y && bx.b[b][2] <= p.z && bx.b[b][5] > p.z;
    if (inside) {  // NaN coordinates compare false with everything, including the box test of a later delete
      ln->pts[j] = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000), p.w);
      del++;
    }
  }
  if (del) { atomicAdd(n_deleted, (unsigned long long)del); atomicAdd(&mv.counters[1], (unsigned long long)(0ull - del)); }
}

// Fill the brick pages from the voxel lines (lsd_map_enable_bricks on a map that already holds points): one thread per
// line, every stored point (tombstones included: NaN coordinates can never be a candidate) goes to its bricks.
__global__ void __launch_bounds__(256) brick_rebuild_kernel(MapView mv, unsigned long long n_lines) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_lines) return;
  const CellLine* ln = mv.lines + s;
  const unsigned long long key = ln->key;
  if (key == 0ull) return;
  const int level = (int)(key >> 57);
  unsigned total = ln->count;
  if (level > 0) {
    uint4 h;
    if (!tag_find(mv, key & ((1ull << 57) - 1ull), &h)) return;
    total = h.z;
  }
  const int n = (int)min(total > (unsigned)(level * kPtsPerLine) ? total - (unsigned)(level * kPtsPerLine) : 0u, (unsigned)kPtsPerLine);
  const int cx = (int)((key >> 38) & 0x7ffffull) - kCoordBias, cy = (int)((key >> 19) & 0x7ffffull) - kCoordBias,
            cz = (int)(key & 0x7ffffull) - kCoordBias;
  for (int j = 0; j < n; j++) brick_insert_point(mv.bricks, cx, cy, cz, ln->pts[j]);
}

static lsd_status_t brick_scratch(lsd_map* m, size_t bytes) {
  if (m->bscratch_bytes >= bytes) return LSD_OK;
  if (m->bscratch) LSD_CUDA(cudaFree(m->bscratch));
  m->bscratch = nullptr; m->bscratch_bytes = 0;
  LSD_CUDA(cudaMalloc(&m->bscratch, bytes));
  m->bscratch_bytes = bytes;
  return LSD_OK;
}

// Batched fixed-stencil k-NN over the brick pages: bin the batch by home brick (3 small kernels), then the persistent
// TMA-staged search (brick.cuh).  Everything on `st`, no host synchronisation.
static lsd_status_t launch_knn_bricks(lsd_map* m, const float4* d_q, int nq, int k, float max_sq, int st_slot, int* d_idx, float* d_d2,
                                      int* d_cnt, cudaStream_t st) {
  const BrickView& bv = m->view.bricks;
  const size_t n_work_max = std::min<size_t>((size_t)m->n_bricks, (size_t)nq) + (size_t)nq / kBrickQC + 2;
  const size_t o_slot = 0, o_rank = o_slot + (size_t)nq * 4, o_sorted = (o_rank + (size_t)nq * 4 + 31) & ~(size_t)31,
               o_work = o_sorted + (size_t)nq * sizeof(BrickQuery), o_ctr = o_work + n_work_max * sizeof(BrickWork), total = o_ctr + 64;
  lsd_status_t s = brick_scratch(m, total);
  if (s) return s;
  char* base = static_cast<char*>(m->bscratch);
  int* q_slot = reinterpret_cast<int*>(base + o_slot);
  int* q_rank = reinterpret_cast<int*>(base + o_rank);
  BrickQuery* sorted = reinterpret_cast<BrickQuery*>(base + o_sorted);
  BrickWork* work = reinterpret_cast<BrickWork*>(base + o_work);
  unsigned* ctr = reinterpret_cast<unsigned*>(base + o_ctr);
  LSD_CUDA(cudaMemsetAsync(ctr, 0, 16, st));
  const int gq = (nq + 255) / 256;
  brick_bin_kernel<<<gq, 256, 0, st>>>(bv, m->view.inv_res, d_q, nq, k, q_slot, q_rank, m->bin_count, d_idx, d_d2, d_cnt, ctr + 3);
  brick_plan_kernel<<<(unsigned)((m->n_bricks + 255) / 256), 256, 0, st>>>(bv, m->n_bricks, m->bin_count, m->bin_base, work, ctr);
  brick_scatter_kernel<<<gq, 256, 0, st>>>(d_q, q_slot, q_rank, m->bin_base, nq, sorted, ctr);
  const int grid = (int)std::min<size_t>(lsd::kNumSms * 5, (n_work_max + kBrickWarps - 1) / kBrickWarps);   // 5 CTAs x 4 warps x 2 x 4.6 KB per SM
  if (k == 1) brick_knn_kernel<1><<<grid, kBrickWarps * 32, 0, st>>>(bv, m->view.inv_res, st_slot, max_sq, sorted, nq, work, ctr, d_idx, d_d2, d_cnt);
  else brick_knn_kernel<5><<<grid, kBrickWarps * 32, 0, st>>>(bv, m->view.inv_res, st_slot, max_sq, sorted, nq, work, ctr, d_idx, d_d2, d_cnt);
  LSD_CUDA(cudaGetLastError());
  m->launches += 4;
  return LSD_OK;
}

static lsd_status_t map_scratch(lsd_map* m, size_t bytes) {
  if (m->scratch_bytes >= bytes) return LSD_OK;
  if (m->scratch) LSD_CUDA(cudaFree(m->scratch));
  m->scratch = nullptr; m->scratch_bytes = 0;
  LSD_CUDA(cudaMalloc(&m->scratch, bytes));
  m->scratch_bytes = bytes;
  return LSD_OK;
}

// ------------------------------------------------------------------ LRU eviction (IVox::AddPoints, ivox3d.h:246-255)
// One thread per evicted voxel: its level-0 line and every overflow line are retired (key = kTombKey: the probe chains that
// run through them stay intact, no query can match them), the counters follow (`points` loses the live points only: a
// box delete already took its tombstones off).
// A voxel evicted and re-created inside one batch keeps exactly what iVox keeps: the points the batch added to it after
// its last eviction.  The host lists them, keep[k0, k1) sorted by their (x, y, z, id) bit patterns; the kernel looks every
// stored point up in that list, retires the lines and re-inserts the points it found (they claim fresh lines).  A listed
// point the map had refused (voxel or table full) is not found, stays refused and is counted in `dropped` once.
struct MapEvict { unsigned long long key; int k0, k1; };
__host__ __device__ __forceinline__ bool keep_less(const uint4& a, const uint4& b) {
  return a.x != b.x ? a.x < b.x : a.y != b.y ? a.y < b.y : a.z != b.z ? a.z < b.z : a.w < b.w;
}
__device__ __forceinline__ bool is_tombstone(const float4& p) {   // map_delete_boxes_kernel's pattern
  return __float_as_uint(p.x) == 0x7fc00000u && __float_as_uint(p.y) == 0x7fc00000u && __float_as_uint(p.z) == 0x7fc00000u;
}
__global__ void __launch_bounds__(128) map_evict_kernel(MapView mv, const MapEvict* __restrict__ ev, int n_ev,
                                                        const uint4* __restrict__ keep, unsigned char* __restrict__ found) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_ev) return;
  const unsigned long long key0 = ev[e].key;
  const int k0 = ev[e].k0, k1 = ev[e].k1;
  uint4 h;
  const CellLine* base = tag_find(mv, key0, &h);
  if (!base) return;
  const unsigned total = h.z;
  const int levels = total > (unsigned)kPtsPerLine ? min((int)((total - 1) / kPtsPerLine), kMaxLevel) : 0;
  unsigned long long stored = 0;
  for (int L = 0; L <= levels; L++) {
    CellLine* ln = const_cast<CellLine*>(base);
    if (L > 0) { uint4 hl; ln = const_cast<CellLine*>(tag_find(mv, key0 | ((unsigned long long)L << 57), &hl)); if (!ln) continue; }
    const int n = (int)min(total - (unsigned)(L * kPtsPerLine), (unsigned)kPtsPerLine);
    for (int j = 0; j < n; j++) {
      const float4 p = ln->pts[j];
      if (is_tombstone(p)) continue;
      stored++;
      if (k0 == k1) continue;
      const uint4 u = make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), __float_as_uint(p.w));
      int lo = k0, hi = k1;                                  // first listed entry not below u
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (keep_less(keep[mid], u)) lo = mid + 1; else hi = mid; }
      for (; lo < k1 && !keep_less(u, keep[lo]); lo++)       // equal entries (exact duplicates): the first one not yet found
        if (!found[lo]) { found[lo] = 1; break; }
    }
    ln->count = 0u;
    ln->key = kTombKey;
  }
  atomicAdd(&mv.counters[0], ~0ull);                       // cells - 1
  atomicAdd(&mv.counters[1], 0ull - stored);
  __threadfence();
  for (int q = k0; q < k1; q++)
    if (found[q]) map_insert_point(mv, __uint_as_float(keep[q].x), __uint_as_float(keep[q].y), __uint_as_float(keep[q].z), (int)keep[q].w);
}

// Fresh table without the retired lines: every live line is copied to its place in the new table (whole 128-byte lines:
// level-0 and overflow lines alike keep their keys).
__global__ void __launch_bounds__(256) map_rehash_kernel(MapView src, unsigned long long n_src, MapView dst) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_src) return;
  const CellLine* ln = src.lines + s;
  const unsigned long long key = ln->key;
  if (key == 0ull || key == kTombKey) return;
  bool fresh;
  const long long d = find_or_claim(dst, key, &fresh);
  if (d < 0) { atomicAdd(&dst.counters[2], 1ull); return; }
  CellLine* out = dst.lines + d;
  out->count = ln->count;
#pragma unroll
  for (int j = 0; j < kPtsPerLine; j++) out->pts[j] = ln->pts[j];
}

// pos2grid as the device evaluates it.  The device's float -> int conversion saturates and turns NaN into 0, so a point with
// a NaN coordinate lands in voxel 0 along that axis (x86's conversion gives INT_MIN for both).  The LRU mirror must file
// every point where map_insert_point filed it.
static __host__ int device_f2i(float v) {
  if (v != v) return 0;
  if (v >= 2147483648.0f) return 0x7fffffff;
  if (v < -2147483648.0f) return (int)0x80000000;
  return (int)v;
}
static __host__ int3 pos2grid_host(float x, float y, float z, float inv_res) {
  return make_int3(device_f2i(roundf(x * inv_res)), device_f2i(roundf(y * inv_res)), device_f2i(roundf(z * inv_res)));
}

static lsd_status_t map_rehash(lsd_map* m, cudaStream_t st) {
  MapView nv = m->view;
  nv.lines = nullptr; nv.tags = nullptr;
  LSD_CUDA(cudaMalloc(&nv.lines, m->n_lines * sizeof(CellLine)));
  LSD_CUDA(cudaMalloc(&nv.tags, m->n_lines));
  LSD_CUDA(cudaMemsetAsync(nv.lines, 0, m->n_lines * sizeof(CellLine), st));
  LSD_CUDA(cudaMemsetAsync(nv.tags, 0, m->n_lines, st));
  nv.bricks.keys = nullptr;                                  // (the brick layout is not combined with the LRU)
  map_rehash_kernel<<<(unsigned)((m->n_lines + 255) / 256), 256, 0, st>>>(m->view, m->n_lines, nv);
  LSD_CUDA(cudaGetLastError());
  LSD_CUDA(cudaStreamSynchronize(st));
  cudaFree(m->view.lines); cudaFree(m->view.tags);
  m->view.lines = nv.lines; m->view.tags = nv.tags;
  m->launches++;
  if (m->lru) m->lru->tombstones = 0;
  return LSD_OK;
}

lsd_status_t map_lru_touch(lsd_map* m, const float4* pts, const int* ids, int n, int id0, cudaStream_t st) {
  LruMirror* L = m->lru;
  if (!L || n <= 0) return LSD_OK;
  std::vector<MapEvict> ev;
  std::vector<std::vector<int>> survivors;                   // per entry of ev: batch positions added after its last eviction
  std::unordered_map<unsigned long long, size_t> in_batch;   // key -> its entry in ev (evicted during this batch)
  const float inv = m->view.inv_res;
  for (int i = 0; i < n; i++) {
    const float4 p = pts[i];
    const int3 c = pos2grid_host(p.x, p.y, p.z, inv);
    if (!coord_ok(c.x, c.y, c.z)) continue;                  // the device dropped it too
    const unsigned long long key = pack_key(c.x, c.y, c.z, 0);
    auto it = L->idx.find(key);
    if (it == L->idx.end()) {
      L->cache.push_front({key, L->distance});
      L->idx[key] = L->cache.begin();
    } else {
      L->cache.splice(L->cache.begin(), L->cache, it->second);
    }
    auto b = in_batch.find(key);
    if (b != in_batch.end()) survivors[b->second].push_back(i);   // evicted earlier in this batch and alive again
    if (L->idx.size() > L->capacity && (L->distance - L->cache.back().d0) > L->max_distance) {
      const unsigned long long k = L->cache.back().key;
      L->idx.erase(k);
      L->cache.pop_back();
      auto e = in_batch.find(k);
      if (e != in_batch.end()) survivors[e->second].clear();     // evicted again: nothing added so far survives
      else { in_batch[k] = ev.size(); ev.push_back({k, 0, 0}); survivors.emplace_back(); }
      L->n_evicted++;
    }
  }
  if (ev.empty()) return LSD_OK;
  // the points to keep, as the device stores them: (x, y, z, id) bit patterns, sorted per voxel for the kernel's lookup
  std::vector<uint4> keep;
  for (size_t e = 0; e < ev.size(); e++) {
    ev[e].k0 = (int)keep.size();
    for (int i : survivors[e]) {
      uint4 u;
      memcpy(&u, &pts[i], 12);
      u.w = ids ? (unsigned)ids[i] : (unsigned)id0 + (unsigned)i;
      keep.push_back(u);
    }
    ev[e].k1 = (int)keep.size();
    std::sort(keep.begin() + ev[e].k0, keep.end(), keep_less);
  }
  const size_t o_keep = (ev.size() * sizeof(MapEvict) + 15) & ~(size_t)15, o_found = o_keep + keep.size() * sizeof(uint4);
  lsd_status_t s = map_scratch(m, o_found + keep.size() + 1);
  if (s) return s;
  char* sc = static_cast<char*>(m->scratch);
  LSD_CUDA(cudaMemcpyAsync(sc, ev.data(), ev.size() * sizeof(MapEvict), cudaMemcpyHostToDevice, st));
  if (!keep.empty()) {
    LSD_CUDA(cudaMemcpyAsync(sc + o_keep, keep.data(), keep.size() * sizeof(uint4), cudaMemcpyHostToDevice, st));
    LSD_CUDA(cudaMemsetAsync(sc + o_found, 0, keep.size(), st));
  }
  map_evict_kernel<<<(unsigned)((ev.size() + 127) / 128), 128, 0, st>>>(m->view, reinterpret_cast<const MapEvict*>(sc), (int)ev.size(),
                                                                        reinterpret_cast<const uint4*>(sc + o_keep),
                                                                        reinterpret_cast<unsigned char*>(sc + o_found));
  LSD_CUDA(cudaGetLastError());
  LSD_CUDA(cudaStreamSynchronize(st));                        // `ev` and `keep` live on this stack frame
  m->launches++;
  L->tombstones += ev.size();
  // retired lines keep their slots: rebuild the table before they crowd the probe chains
  if ((L->idx.size() + L->tombstones) * 2 > m->n_lines) return map_rehash(m, st);
  return LSD_OK;
}

lsd_status_t launch_insert(lsd_map* m, const float4* d_pts, int n, int id0, cudaStream_t st) {
  if (n <= 0) return LSD_OK;
  map_insert_kernel<<<(n + 255) / 256, 256, 0, st>>>(m->view, d_pts, n, id0);
  LSD_CUDA(cudaGetLastError());
  m->launches++;
  return LSD_OK;
}

lsd_status_t launch_knn(lsd_map* m, const float4* d_q, int nq, int k, float max_sq, int stencil, int* d_idx, float* d_d2,
                        int* d_cnt, cudaStream_t st) {
  if (nq <= 0) return LSD_OK;
  if (stencil != LSD_STENCIL_EXACT && stencil_slot(stencil) < 0) { set_error("unknown stencil %d", stencil); return LSD_ERR_INVALID; }
  if (m->view.shard_world > 1 && stencil_reach(stencil, max_sq, m->view.inv_res) > m->view.shard_reach) {
    // a wider search than the halo would silently miss the neighbours in voxels this shard does not hold
    set_error("k-NN on a tile-sharded map: stencil %d reaches %d voxels, the shard's halo only %d", stencil,
              stencil_reach(stencil, max_sq, m->view.inv_res), m->view.shard_reach);
    return LSD_ERR_INVALID;
  }
  const int shape = m->knn_shape;  // 0 auto, 1 warp/query, 2 thread/query, 3 brick pages (lsd_knn_set_shape)
  {
    // brick pages: fixed stencils of reach 1 (CENTER / NEARBY6 / 18 / 26), k in {1, 5}; auto from kThreadKnnMin queries on
    const int ss = stencil_slot(stencil);
    const bool can = m->view.bricks.keys && ss >= 0 && ss <= 3 && (k == 1 || k == 5);
    if (shape == 3 && !can) { set_error("lsd_knn_set_shape(3): bricks not enabled on this map, or stencil / k not served by the brick pages"); return LSD_ERR_INVALID; }
    if (can && (shape == 3 || (shape == 0 && nq >= kThreadKnnMin))) return launch_knn_bricks(m, d_q, nq, k, max_sq, ss, d_idx, d_d2, d_cnt, st);
  }
  if (stencil != LSD_STENCIL_EXACT && k <= 5 && shape != 1 && (nq >= kThreadKnnMin || shape == 2)) {  // throughput shape: one thread per query
    const int ss = stencil_slot(stencil), gb = (nq + 255) / 256;
    if (k == 1) knn_query_thread_kernel<1><<<gb, 256, 0, st>>>(m->view, d_q, nq, max_sq, ss, d_idx, d_d2, d_cnt);
    else if (k == 5) knn_query_thread_kernel<5><<<gb, 256, 0, st>>>(m->view, d_q, nq, max_sq, ss, d_idx, d_d2, d_cnt);
    else { set_error("k must be 1, 5 or 20 (got %d)", k); return LSD_ERR_INVALID; }
    LSD_CUDA(cudaGetLastError());
    m->launches++;
    return LSD_OK;
  }
  dim3 g(std::min((nq + kKnnWarps - 1) / kKnnWarps, lsd::kNumSms * 8)), b(kKnnWarps * 32);
  switch (k) {
    case 1: knn_query_kernel<1><<<g, b, 0, st>>>(m->view, d_q, nq, max_sq, stencil, d_idx, d_d2, d_cnt); break;
    case 5: knn_query_kernel<5><<<g, b, 0, st>>>(m->view, d_q, nq, max_sq, stencil, d_idx, d_d2, d_cnt); break;
    case 20: knn_query_kernel<20><<<g, b, 0, st>>>(m->view, d_q, nq, max_sq, stencil, d_idx, d_d2, d_cnt); break;
    default: set_error("k must be 1, 5 or 20 (got %d)", k); return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaGetLastError());
  m->launches++;
  return LSD_OK;
}

}  // namespace lsd

using namespace lsd;

// ==================================================================== C ABI
extern "C" {

const char* lsd_version(void) { return "lsdreg 0.1.0 (sm_90a)"; }
const char* lsd_last_error(void) { return g_err; }

lsd_status_t lsd_init(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) { cudaGetLastError(); set_error("no CUDA device: liblsdreg has no CPU fallback"); return LSD_ERR_NO_DEVICE; }
  if (device < 0 || device >= n) { set_error("device %d out of range (%d devices)", device, n); return LSD_ERR_INVALID; }
  g_device = device;
  LSD_CUDA(cudaSetDevice(device));
  // L2 fetch granularity stays at the driver default: 32-byte fetches halve the DRAM bytes of a hash probe but
  // can make the batched k-NN slower.
  // LSD_L2_FETCH_GRANULARITY=32|64|128 overrides it for A/B measurements.
  if (const char* e = getenv("LSD_L2_FETCH_GRANULARITY")) {
    const size_t g = (size_t)atoi(e);
    if (g == 32 || g == 64 || g == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, g);
    cudaGetLastError();
  }
  return LSD_OK;
}

lsd_status_t lsd_map_create(lsd_map_t** out, float resolution, int log2_lines) {
  if (!out || resolution <= 0.f || log2_lines < 10 || log2_lines > 28) { set_error("lsd_map_create: bad arguments"); return LSD_ERR_INVALID; }
  lsd_status_t s = ensure_device();
  if (s) return s;
  s = upload_stencils();
  if (s) return s;
  lsd_map* m = new lsd_map();
  m->device = g_device;
  m->n_lines = 1ull << log2_lines;
  m->view.mask = m->n_lines - 1;
  m->view.res = resolution;
  m->view.inv_res = (float)(1.0 / (double)resolution);  // ivox3d.h:58
  m->view.shard_rank = 0; m->view.shard_world = 1; m->view.shard_tile = 32; m->view.shard_reach = 1;
  cudaError_t e = cudaMalloc(&m->view.lines, m->n_lines * sizeof(CellLine));
  if (e == cudaSuccess) e = cudaMalloc(&m->view.tags, m->n_lines);
  if (e == cudaSuccess) e = cudaMalloc(&m->view.counters, 4 * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { lsd_status_t r = cuda_fail(e, "lsd_map_create alloc", __FILE__, __LINE__); delete m; return r; }
  *out = m;
  return lsd_map_clear(m);
}

lsd_status_t lsd_map_destroy(lsd_map_t* m) {
  if (!m) return LSD_OK;
  cudaSetDevice(m->device);
  if (m->stream) cudaStreamSynchronize(m->stream); else cudaDeviceSynchronize();
  cudaFree(m->view.lines); cudaFree(m->view.tags); cudaFree(m->view.counters); cudaFree(m->scratch);
  cudaFree(m->view.bricks.keys); cudaFree(m->view.bricks.totals); cudaFree(m->view.bricks.pages); cudaFree(m->view.bricks.counters);
  cudaFree(m->bin_count); cudaFree(m->bin_base); cudaFree(m->bscratch);
  delete m->lru;
  if (m->stream) cudaStreamDestroy(m->stream);
  delete m;
  return LSD_OK;
}

lsd_status_t lsd_map_set_shard(lsd_map_t* m, int rank, int world, int tile_cells, int reach_cells) {
  if (!m || world < 1 || rank < 0 || rank >= world || tile_cells < 1 || reach_cells < 0 || 2 * reach_cells >= tile_cells) {
    set_error("lsd_map_set_shard: need 0 <= rank < world and 2*reach < tile");
    return LSD_ERR_INVALID;
  }
  if (world > 1 && m->view.bricks.keys) { set_error("lsd_map_set_shard: the brick layout is not available on a tile-sharded map"); return LSD_ERR_INVALID; }
  m->view.shard_rank = rank; m->view.shard_world = world; m->view.shard_tile = tile_cells; m->view.shard_reach = reach_cells;
  return LSD_OK;
}

lsd_status_t lsd_map_clear(lsd_map_t* m) {
  if (!m) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  LSD_CUDA(cudaMemsetAsync(m->view.lines, 0, m->n_lines * sizeof(CellLine), m->stream));
  LSD_CUDA(cudaMemsetAsync(m->view.tags, 0, m->n_lines, m->stream));
  LSD_CUDA(cudaMemsetAsync(m->view.counters, 0, 4 * sizeof(unsigned long long), m->stream));
  if (m->view.bricks.keys) {
    LSD_CUDA(cudaMemsetAsync(m->view.bricks.keys, 0, m->n_bricks * 8, m->stream));
    LSD_CUDA(cudaMemsetAsync(m->view.bricks.totals, 0, m->n_bricks * 4, m->stream));
    LSD_CUDA(cudaMemsetAsync(m->view.bricks.pages, 0, m->n_bricks * (size_t)kPageBytes, m->stream));
    LSD_CUDA(cudaMemsetAsync(m->view.bricks.counters, 0, 4 * sizeof(unsigned long long), m->stream));
  }
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  if (m->lru) { m->lru->cache.clear(); m->lru->idx.clear(); m->lru->tombstones = 0; }
  m->dropped_seen = 0;
  return LSD_OK;
}

// iVox's capacity / LRU (ivox3d.h:51-52,246-255; the reference runs with capacity 100 000 voxels, max_distance 100 m,
// laserMapping.cpp:1063-1064).  See include/lsdreg.h.
lsd_status_t lsd_map_enable_lru(lsd_map_t* m, uint64_t capacity, double max_distance) {
  if (!m || capacity < 1 || !(max_distance >= 0.0)) { set_error("lsd_map_enable_lru: bad arguments"); return LSD_ERR_INVALID; }
  if (m->view.shard_world > 1 || m->view.bricks.keys) { set_error("lsd_map_enable_lru: not available on a tile-sharded map or together with the brick layout"); return LSD_ERR_INVALID; }
  uint64_t cells = 0;
  lsd_status_t s = lsd_map_stats(m, &cells, nullptr, nullptr);
  if (s) return s;
  if (cells != 0) { set_error("lsd_map_enable_lru: the map must be empty (the LRU order of points already stored is unknown)"); return LSD_ERR_INVALID; }
  if (!m->lru) m->lru = new LruMirror();
  m->lru->capacity = (size_t)capacity;
  m->lru->max_distance = max_distance;
  return LSD_OK;
}
lsd_status_t lsd_map_set_travel_distance(lsd_map_t* m, double distance) {
  if (!m) return LSD_ERR_INVALID;
  if (m->lru) m->lru->distance = distance;
  return LSD_OK;
}
lsd_status_t lsd_map_evict(lsd_map_t* m, uint64_t* n_evicted_total) {
  if (!m || !m->lru) { set_error("lsd_map_evict: lsd_map_enable_lru was not called"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(m->device));
  if (m->stream) LSD_CUDA(cudaStreamSynchronize(m->stream));   // evictions are applied inside the insert calls; this is the fence + the count
  if (n_evicted_total) *n_evicted_total = m->lru->n_evicted;
  return LSD_OK;
}
// Did the map refuse points since the last call (table full along a probe chain, > 127 overflow lines in a voxel, voxel
// coordinates beyond +-2^18)?  A map that stopped growing degrades odometry silently; callers should treat 1 as an alarm.
lsd_status_t lsd_map_saturated(lsd_map_t* m, int* saturated, uint64_t* n_dropped_total) {
  if (!m || !saturated) return LSD_ERR_INVALID;
  uint64_t d = 0;
  lsd_status_t s = lsd_map_stats(m, nullptr, nullptr, &d);
  if (s) return s;
  *saturated = d > m->dropped_seen ? 1 : 0;
  m->dropped_seen = d;
  if (n_dropped_total) *n_dropped_total = d;
  return LSD_OK;
}

lsd_status_t lsd_map_enable_bricks(lsd_map_t* m, int log2_bricks) {
  if (!m || log2_bricks < 8 || log2_bricks > 24) { set_error("lsd_map_enable_bricks: log2_bricks must be in [8, 24]"); return LSD_ERR_INVALID; }
  if (m->view.shard_world > 1) { set_error("lsd_map_enable_bricks: not available on a tile-sharded map"); return LSD_ERR_INVALID; }
  if (m->view.bricks.keys) { set_error("lsd_map_enable_bricks: already enabled"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(m->device));
  const unsigned long long n = 1ull << log2_bricks;
  BrickView bv;
  memset(&bv, 0, sizeof(bv));
  cudaError_t e = cudaMalloc(&bv.keys, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&bv.totals, n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&bv.pages, n * (size_t)kPageBytes);
  if (e == cudaSuccess) e = cudaMalloc(&bv.counters, 4 * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&m->bin_count, n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&m->bin_base, n * 4);
  if (e != cudaSuccess) {
    cudaFree(bv.keys); cudaFree(bv.totals); cudaFree(bv.pages); cudaFree(bv.counters); cudaFree(m->bin_count); cudaFree(m->bin_base);
    m->bin_count = nullptr; m->bin_base = nullptr;
    return cuda_fail(e, "lsd_map_enable_bricks alloc", __FILE__, __LINE__);
  }
  bv.mask = n - 1;
  LSD_CUDA(cudaMemsetAsync(bv.keys, 0, n * 8, m->stream));
  LSD_CUDA(cudaMemsetAsync(bv.totals, 0, n * 4, m->stream));
  LSD_CUDA(cudaMemsetAsync(bv.pages, 0, n * (size_t)kPageBytes, m->stream));
  LSD_CUDA(cudaMemsetAsync(bv.counters, 0, 4 * sizeof(unsigned long long), m->stream));
  LSD_CUDA(cudaMemsetAsync(m->bin_count, 0, n * 4, m->stream));
  m->n_bricks = n;
  m->view.bricks = bv;
  // points already in the map
  brick_rebuild_kernel<<<(unsigned)((m->n_lines + 255) / 256), 256, 0, m->stream>>>(m->view, m->n_lines);
  LSD_CUDA(cudaGetLastError());
  m->launches++;
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  return LSD_OK;
}

lsd_status_t lsd_map_brick_stats(lsd_map_t* m, uint64_t* n_pages, uint64_t* n_replicas, uint64_t* n_dropped) {
  if (!m || !m->view.bricks.keys) { set_error("lsd_map_brick_stats: bricks not enabled"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(m->device));
  unsigned long long h[4];
  LSD_CUDA(cudaMemcpyAsync(h, m->view.bricks.counters, sizeof(h), cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  if (n_pages) *n_pages = h[0];
  if (n_replicas) *n_replicas = h[1];
  if (n_dropped) *n_dropped = h[2];
  return LSD_OK;
}


lsd_status_t lsd_map_insert_dev(lsd_map_t* m, const float* xyzi_dev, int n, int32_t id0) {
  if (!m || (n > 0 && !xyzi_dev) || n < 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  lsd_status_t s = launch_insert(m, reinterpret_cast<const float4*>(xyzi_dev), n, id0, m->stream);
  if (s || !m->lru || n == 0) return s;
  std::vector<float4> h((size_t)n);                            // the LRU order is replayed on the host (map.h::LruMirror)
  LSD_CUDA(cudaMemcpyAsync(h.data(), xyzi_dev, (size_t)n * 16, cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  return map_lru_touch(m, h.data(), nullptr, n, id0, m->stream);
}

lsd_status_t lsd_map_insert(lsd_map_t* m, const float* xyzi_host, int n, int32_t id0) {
  if (!m || (n > 0 && !xyzi_host) || n < 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  const int chunk = 1 << 22;  // 64 MB staging
  lsd_status_t s = map_scratch(m, (size_t)std::min(n, chunk) * 16);
  if (s) return s;
  for (int o = 0; o < n; o += chunk) {
    int c = std::min(chunk, n - o);
    LSD_CUDA(cudaMemcpyAsync(m->scratch, xyzi_host + (size_t)o * 4, (size_t)c * 16, cudaMemcpyHostToDevice, m->stream));
    s = launch_insert(m, reinterpret_cast<const float4*>(m->scratch), c, id0 + o, m->stream);
    if (s) return s;
    LSD_CUDA(cudaStreamSynchronize(m->stream));
    if (m->lru) { s = map_lru_touch(m, reinterpret_cast<const float4*>(xyzi_host) + o, nullptr, c, id0 + o, m->stream); if (s) return s; }
  }
  return LSD_OK;
}

lsd_status_t lsd_map_stats(lsd_map_t* m, uint64_t* n_cells, uint64_t* n_points, uint64_t* n_dropped) {
  if (!m) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  unsigned long long h[4];
  LSD_CUDA(cudaMemcpyAsync(h, m->view.counters, sizeof(h), cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  if (n_cells) *n_cells = h[0];
  if (n_points) *n_points = h[1];
  if (n_dropped) *n_dropped = h[2];
  return LSD_OK;
}

lsd_status_t lsd_map_dump(lsd_map_t* m, int32_t* voxel3, float* xyz3, int32_t* ids, uint8_t* tombstone, uint64_t cap,
                          uint64_t* n_points) {
  if (!m || !n_points || (cap > 0 && (!voxel3 || !xyz3 || !ids || !tombstone))) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  std::vector<CellLine> t((size_t)m->n_lines);
  LSD_CUDA(cudaMemcpyAsync(t.data(), m->view.lines, (size_t)m->n_lines * sizeof(CellLine), cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  std::unordered_map<unsigned long long, size_t> over;   // overflow line key -> slot
  for (size_t s = 0; s < t.size(); s++)
    if (t[s].key != 0ull && t[s].key != kTombKey && (t[s].key >> 57) != 0ull) over[t[s].key] = s;
  uint64_t k = 0;
  for (size_t s = 0; s < t.size(); s++) {
    const unsigned long long key = t[s].key;
    if (key == 0ull || key == kTombKey || (key >> 57) != 0ull) continue;
    const int v[3] = {(int)((key >> 38) & 0x7ffffull) - kCoordBias, (int)((key >> 19) & 0x7ffffull) - kCoordBias,
                      (int)(key & 0x7ffffull) - kCoordBias};
    const unsigned total = t[s].count;
    const int levels = total > (unsigned)kPtsPerLine ? std::min((int)((total - 1) / kPtsPerLine), kMaxLevel) : 0;
    for (int L = 0; L <= levels; L++) {
      const CellLine* ln = &t[s];
      if (L > 0) {
        auto it = over.find(key | ((unsigned long long)L << 57));
        if (it == over.end()) continue;
        ln = &t[it->second];
      }
      const int n = (int)std::min(total - (unsigned)(L * kPtsPerLine), (unsigned)kPtsPerLine);
      for (int j = 0; j < n; j++, k++) {
        if (k >= cap) continue;
        const float4 p = ln->pts[j];
        unsigned b[3];
        memcpy(b, &p, 12);
        for (int d = 0; d < 3; d++) voxel3[3 * k + d] = v[d];
        xyz3[3 * k] = p.x; xyz3[3 * k + 1] = p.y; xyz3[3 * k + 2] = p.z;
        memcpy(&ids[k], &p.w, 4);
        tombstone[k] = b[0] == 0x7fc00000u && b[1] == 0x7fc00000u && b[2] == 0x7fc00000u;
      }
    }
  }
  *n_points = k;
  return LSD_OK;
}

lsd_status_t lsd_map_delete_boxes(lsd_map_t* m, const float* boxes6_host, int n_boxes, uint64_t* n_deleted) {
  if (!m || n_boxes < 0 || (n_boxes > 0 && !boxes6_host)) return LSD_ERR_INVALID;
  if (n_deleted) *n_deleted = 0;
  if (n_boxes == 0) return LSD_OK;
  LSD_CUDA(cudaSetDevice(m->device));
  unsigned long long total = 0;
  for (int o = 0; o < n_boxes; o += kMaxDeleteBoxes) {
    DeleteBoxes bx;
    bx.n = std::min(kMaxDeleteBoxes, n_boxes - o);
    memcpy(bx.b, boxes6_host + 6 * (size_t)o, (size_t)bx.n * 6 * sizeof(float));
    LSD_CUDA(cudaMemsetAsync(&m->view.counters[3], 0, sizeof(unsigned long long), m->stream));
    map_delete_boxes_kernel<<<(unsigned)((m->n_lines + 255) / 256), 256, 0, m->stream>>>(m->view, m->n_lines, bx, &m->view.counters[3]);
    LSD_CUDA(cudaGetLastError());
    m->launches++;
    if (m->view.bricks.keys) {   // the replicas in the brick pages get the same tombstones
      BrickBoxes bb;
      bb.n = bx.n; memcpy(bb.b, bx.b, sizeof(bb.b));
      brick_delete_boxes_kernel<<<(unsigned)((m->n_bricks * 8 + 255) / 256), 256, 0, m->stream>>>(m->view.bricks, m->n_bricks, bb);
      LSD_CUDA(cudaGetLastError());
      m->launches++;
    }
    unsigned long long h = 0;
    LSD_CUDA(cudaMemcpyAsync(&h, &m->view.counters[3], sizeof(h), cudaMemcpyDeviceToHost, m->stream));
    LSD_CUDA(cudaStreamSynchronize(m->stream));
    total += h;
  }
  if (n_deleted) *n_deleted = total;
  return LSD_OK;
}

lsd_status_t lsd_map_stream(lsd_map_t* m, void** cuda_stream_out) {
  if (!m || !cuda_stream_out) return LSD_ERR_INVALID;
  *cuda_stream_out = static_cast<void*>(m->stream);
  return LSD_OK;
}

lsd_status_t lsd_knn_set_shape(lsd_map_t* m, int shape) {
  if (!m || shape < 0 || shape > 3) return LSD_ERR_INVALID;
  m->knn_shape = shape;
  return LSD_OK;
}
lsd_status_t lsd_knn_query_dev(lsd_map_t* m, const float* q_dev, int nq, int k, float max_sq, int stencil,
                               int32_t* out_idx_dev, float* out_d2_dev, int32_t* out_cnt_dev) {
  if (!m || nq < 0 || (nq > 0 && (!q_dev || !out_idx_dev || !out_d2_dev || !out_cnt_dev))) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(m->device));
  return launch_knn(m, reinterpret_cast<const float4*>(q_dev), nq, k, max_sq, stencil, out_idx_dev, out_d2_dev, out_cnt_dev, m->stream);
}

lsd_status_t lsd_knn_query(lsd_map_t* m, const float* q_host, int nq, int k, float max_sq, int stencil,
                           int32_t* out_idx, float* out_d2, int32_t* out_cnt) {
  if (!m || nq < 0 || (nq > 0 && (!q_host || !out_idx || !out_d2 || !out_cnt))) return LSD_ERR_INVALID;
  if (nq == 0) return LSD_OK;
  LSD_CUDA(cudaSetDevice(m->device));
  size_t bq = (size_t)nq * 16, bi = (size_t)nq * k * 4, bc = (size_t)nq * 4;
  lsd_status_t s = map_scratch(m, bq + 2 * bi + bc + 256);
  if (s) return s;
  char* base = static_cast<char*>(m->scratch);
  float4* dq = reinterpret_cast<float4*>(base);
  int* didx = reinterpret_cast<int*>(base + bq);
  float* dd2 = reinterpret_cast<float*>(base + bq + bi);
  int* dcnt = reinterpret_cast<int*>(base + bq + 2 * bi);
  LSD_CUDA(cudaMemcpyAsync(dq, q_host, bq, cudaMemcpyHostToDevice, m->stream));
  s = launch_knn(m, dq, nq, k, max_sq, stencil, didx, dd2, dcnt, m->stream);
  if (s) return s;
  LSD_CUDA(cudaMemcpyAsync(out_idx, didx, bi, cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaMemcpyAsync(out_d2, dd2, bi, cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaMemcpyAsync(out_cnt, dcnt, bc, cudaMemcpyDeviceToHost, m->stream));
  LSD_CUDA(cudaStreamSynchronize(m->stream));
  return LSD_OK;
}

}  // extern "C"
