// voxelgrid.cu — K1: voxel-grid centroid downsample, sort-free.
//
// Replaces pcl::VoxelGrid<PointXYZINormal>::filter as called by the LIO front-end
// (reference: slam/mapping/fastlio/src/laserMapping.cpp:1206-1207, leaf 0.5 m :1027,:1073) and by
// localization (hdl_localization_nodelet.cpp:333-344).  PCL semantics kept (PCL 1.9.1
// filters/impl/voxel_grid.hpp; not vendored in the reference tree):
//   bbox -> min_b = floor(min * inv_leaf); leaf index = (ijk - min_b) . (1, dx, dx*dy);
//   one centroid of all channels per occupied leaf; output in ascending leaf-index order;
//   grids above INT32_MAX leaves are refused (PCL warns and returns the input).
// PCL gets the order from a std::sort of (leaf, point) pairs and sums fp32 in that order.  Here the OUTPUT
// order comes from a rank over an occupancy bitmap (popcount prefix scan); the centroids are, by default,
// the sequential fp32 sums in input order of the restated filter (oracle/lsd_oracle.c::orc_voxelgrid, the
// arithmetic the reference arm runs), bit for bit — or, with LSD_VG_SUMS=fixed, exact 64-bit fixed-point
// atomics (round 1: independent of thread order, one fp32 ulp from the former for half the leaves, 2.2 x faster).
//
// Pipeline (all sizes stay on the device, no host round trip):
//   vg_minmax -> vg_mark (+grid setup) -> vg_scan (word scan; last block scans the chunk totals)
//   -> vg_count (+ the last block scans the per-leaf counts) -> vg_scatter -> vg_sum (+scratch cleanup)
//   [fixed-point: -> vg_accum -> vg_finalize (+scratch cleanup)].  A single cooperative kernel with grid barriers
//   was measured and rejected: no faster (the barriers cost what the launches do) and cooperative
//   launches serialise badly behind an in-flight H2D copy (e2e 3.5 ms/scan vs 0.39 ms).
#include "lsd_common.cuh"
#include "voxelgrid.h"

namespace lsd {

constexpr int kScanChunk = 1024;  // bitmap words per scan block
constexpr double kFix = 67108864.0;  // 2^26 fixed-point scale (1.5e-8 m)

__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__device__ __forceinline__ void vg_setup(const int* __restrict__ bbox, float leaf, long long max_cells, VgGrid* g) {
  const float inv = 1.0f / leaf;
  float mn[3], mx[3];
  for (int d = 0; d < 3; d++) { mn[d] = ord2f(bbox[d]); mx[d] = ord2f(bbox[3 + d]); }
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  g->inv = inv;
  g->status = 0;
  // each factor is bounded first: (long long)(huge float) and the triple product must not wrap past the test below
  const bool sane = dx >= 1 && dy >= 1 && dz >= 1 && dx <= 2147483647ll && dy <= 2147483647ll && dz <= 2147483647ll;
  if (!sane || dx * dy > 2147483647ll || dx * dy * dz > 2147483647ll) g->status = LSD_ERR_GRID_OVERFLOW;  // PCL: "Leaf size is too small"
  if (mn[0] > mx[0]) g->status = LSD_ERR_INVALID;   // no finite point at all: empty output
  for (int d = 0; d < 3; d++) {
    g->minb[d] = g->status ? 0 : (int)floorf(mn[d] * inv);
    g->divb[d] = g->status ? 1 : (int)floorf(mx[d] * inv) - g->minb[d] + 1;
  }
  const long long cells = (long long)g->divb[0] * g->divb[1] * g->divb[2];
  if (g->status == 0 && cells > max_cells) g->status = LSD_ERR_CAPACITY;
  g->mul[0] = 1; g->mul[1] = g->divb[0]; g->mul[2] = g->divb[0] * g->divb[1];
  g->n_words = g->status ? 0 : (int)((cells + 31) >> 5);
}

__device__ __forceinline__ bool vg_finite(const float4& p) {
  return fabsf(p.x) <= 3.0e38f && fabsf(p.y) <= 3.0e38f && fabsf(p.z) <= 3.0e38f;   // false for NaN and +-Inf
}

__device__ __forceinline__ int leaf_index(const VgGrid& g, const float4& p) {
  const int i0 = (int)(floorf(p.x * g.inv) - (float)g.minb[0]);
  const int i1 = (int)(floorf(p.y * g.inv) - (float)g.minb[1]);
  const int i2 = (int)(floorf(p.z * g.inv) - (float)g.minb[2]);
  return i0 * g.mul[0] + i1 * g.mul[1] + i2 * g.mul[2];
}

// block-wide exclusive scan helper over `count` ints starting at base (256 threads)
__device__ __forceinline__ int block_scan_step(int v, int* warp_tot, int* carry, int* incl_out) {
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= o) inc += t; }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
  __syncthreads();
  int woff = 0;
  for (int k = 0; k < (int)(threadIdx.x >> 5); k++) woff += warp_tot[k];
  const int c = *carry;
  *incl_out = c + woff + inc;
  __syncthreads();
  if (threadIdx.x == blockDim.x - 1) *carry = c + woff + inc;
  __syncthreads();
  return c + woff + inc - v;  // exclusive
}

// ---- kernel 1: bounding box.  Block-level reduction, then 6 atomics per block.
__global__ void __launch_bounds__(256) vg_minmax_kernel(const float4* __restrict__ in, int n, int* __restrict__ bbox) {
  pdl_enter();
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(in + i);
    if (!vg_finite(p)) continue;   // pcl::VoxelGrid skips non-finite points (!is_dense branch); one Inf would blow the grid up
    mn[0] = fminf(mn[0], p.x); mx[0] = fmaxf(mx[0], p.x);
    mn[1] = fminf(mn[1], p.y); mx[1] = fmaxf(mx[1], p.y);
    mn[2] = fminf(mn[2], p.z); mx[2] = fmaxf(mx[2], p.z);
  }
  __shared__ float smn[8][3], smx[8][3];
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5][d] = mn[d]; smx[threadIdx.x >> 5][d] = mx[d]; }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float a = smn[0][threadIdx.x], b = smx[0][threadIdx.x];
    for (int w = 1; w < 8; w++) { a = fminf(a, smn[w][threadIdx.x]); b = fmaxf(b, smx[w][threadIdx.x]); }
    atomicMin(&bbox[threadIdx.x], f2ord(a));
    atomicMax(&bbox[3 + threadIdx.x], f2ord(b));
  }
}

// ---- kernel 2: grid description (every block derives it; block 0 publishes it), mark leaves
__global__ void __launch_bounds__(256) vg_mark_kernel(const float4* __restrict__ in, int n, float leaf, long long max_cells,
                                                      const int* __restrict__ bbox, VgGrid* __restrict__ gp,
                                                      unsigned* __restrict__ bitmap, int* __restrict__ vidx) {
  pdl_enter();
  __shared__ VgGrid g;
  if (threadIdx.x == 0) { vg_setup(bbox, leaf, max_cells, &g); if (blockIdx.x == 0) *gp = g; }
  __syncthreads();
  if (g.status) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(in + i);
    int idx = vg_finite(p) ? leaf_index(g, p) : -1;
    if (idx < 0 || (idx >> 5) >= g.n_words) idx = -1;   // cannot happen for a finite point inside the bbox; never index past the bitmap
    vidx[i] = idx;
    if (idx < 0) continue;
    const unsigned bit = 1u << (idx & 31);
    unsigned* w = bitmap + (idx >> 5);
    if (!(*reinterpret_cast<volatile unsigned*>(w) & bit)) atomicOr(w, bit);
  }
}

// ---- kernel 3: per chunk of kScanChunk bitmap words, exclusive popcount prefix + chunk total; the
// last block to finish scans the chunk totals and writes the output count.
__global__ void __launch_bounds__(256) vg_scan_kernel(const VgGrid* __restrict__ gp, const unsigned* __restrict__ bitmap,
                                                      int* __restrict__ word_prefix, int* __restrict__ chunk_sum,
                                                      unsigned* __restrict__ done, int* __restrict__ m_out, int n_in) {
  pdl_enter();
  __shared__ int warp_tot[8];
  __shared__ int carry;
  __shared__ bool is_last;
  const int n_words = gp->n_words, status = gp->status;
  const int n_chunks = (n_words + kScanChunk - 1) / kScanChunk;
  for (int chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = chunk * kScanChunk; base < min((chunk + 1) * kScanChunk, n_words); base += 256) {
      const int w = base + threadIdx.x;
      const int v = w < n_words ? __popc(bitmap[w]) : 0;
      int incl;
      const int ex = block_scan_step(v, warp_tot, &carry, &incl);
      if (w < n_words) word_prefix[w] = ex;
    }
    if (threadIdx.x == 0) chunk_sum[chunk] = carry;
    __syncthreads();
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_chunks; base += 256) {
    const int i = base + threadIdx.x;
    const int v = i < n_chunks ? __ldcg(chunk_sum + i) : 0;
    int incl;
    const int ex = block_scan_step(v, warp_tot, &carry, &incl);
    if (i < n_chunks) chunk_sum[i] = ex;
  }
  if (threadIdx.x == 0) {
    *m_out = status == LSD_ERR_GRID_OVERFLOW ? n_in : (status ? 0 : carry);
    *done = 0u;
  }
}

// ---- kernel 4: rank of each point's leaf = its output slot; exact fixed-point channel sums
__global__ void __launch_bounds__(256) vg_accum_kernel(const float4* __restrict__ in, int n, const VgGrid* __restrict__ gp,
                                                       const unsigned* __restrict__ bitmap, const int* __restrict__ vidx,
                                                       const int* __restrict__ word_prefix, const int* __restrict__ chunk_off,
                                                       long long* __restrict__ sums, int* __restrict__ cnt,
                                                       int* __restrict__ out_vidx, float4* __restrict__ out) {
  pdl_enter();
  const int status = gp->status;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(in + i);
    if (status == LSD_ERR_GRID_OVERFLOW) { out[i] = p; continue; }  // PCL: output = input
    if (status) return;
    const int idx = vidx[i];
    if (idx < 0) continue;   // non-finite point
    const int w = idx >> 5;
    const int rank = chunk_off[w / kScanChunk] + word_prefix[w] + __popc(bitmap[w] & ((1u << (idx & 31)) - 1u));
    long long* s = sums + 4 * (size_t)rank;
    atomicAdd(reinterpret_cast<unsigned long long*>(s + 0), (unsigned long long)__double2ll_rn((double)p.x * kFix));
    atomicAdd(reinterpret_cast<unsigned long long*>(s + 1), (unsigned long long)__double2ll_rn((double)p.y * kFix));
    atomicAdd(reinterpret_cast<unsigned long long*>(s + 2), (unsigned long long)__double2ll_rn((double)p.z * kFix));
    atomicAdd(reinterpret_cast<unsigned long long*>(s + 3), (unsigned long long)__double2ll_rn((double)p.w * kFix));
    atomicAdd(cnt + rank, 1);
    out_vidx[rank] = idx;
  }
}

// ---- kernel 5: centroids; scratch (bitmap words, sums, counts, bbox) returns to its idle state so
// the next call needs no memset proportional to the grid volume.
__global__ void __launch_bounds__(256) vg_finalize_kernel(const VgGrid* __restrict__ gp, const int* __restrict__ m_ptr,
                                                          long long* __restrict__ sums, int* __restrict__ cnt,
                                                          const int* __restrict__ out_vidx, unsigned* __restrict__ bitmap,
                                                          float4* __restrict__ out, int* __restrict__ bbox) {
  pdl_enter();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    bbox[0] = bbox[1] = bbox[2] = 0x7f7f7f7f;
    bbox[3] = bbox[4] = bbox[5] = (int)0x80808080;
  }
  if (gp->status) return;
  const int m = *m_ptr;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    long long* s = sums + 4 * (size_t)r;
    const double c = (double)cnt[r];
    float4 o;
    o.x = (float)((double)s[0] / kFix / c);
    o.y = (float)((double)s[1] / kFix / c);
    o.z = (float)((double)s[2] / kFix / c);
    o.w = (float)((double)s[3] / kFix / c);
    out[r] = o;
    s[0] = s[1] = s[2] = s[3] = 0;
    cnt[r] = 0;
    bitmap[out_vidx[r] >> 5] = 0u;
  }
}

// ---- the centroids as a sequential fp32 sum in INPUT order (kernels 4a-4c instead of 4 and 5) ----------------------------------
// pcl::VoxelGrid adds a leaf's points one by one into fp32 accumulators, in the order std::sort leaves equal keys in, and divides
// by the count; the restated filter the oracle and the reference arm use (oracle/lsd_oracle.c::orc_voxelgrid,
// oracle/ref_shim_fastlio/pcl/filters/voxel_grid.h) fixes that order to the input order.  Reproducing THAT arithmetic — instead
// of the exact fixed-point sums above, one fp32 ulp away for half the leaves — is what lets a whole scan agree with the
// reference arm to the last bits of the double-precision sums (DESIGN.md section 4): a counting sort by leaf (count + exclusive
// scan of the counts, scatter), then every leaf sorts its members' input indices and adds its points in that order.  The scatter
// leaves a leaf's members in arrival order, so the sort is what fixes the order of the additions.  Two size classes: a leaf of
// at most kVgSmall points is one thread's (a sorting network in registers); a crowded one is a warp's (bitonic sort of the
// indices in shared memory, the points gathered with all loads in flight, each channel one sequential fp32 chain); a big one
// (more than kVgCap) is a block's (the sort in the block's shared memory, in place in global memory above kVgBig).
constexpr int kVgSmall = 8;     // leaves of up to this many points: one thread each
constexpr int kVgCap = 512;     // crowded leaves up to this many points: one warp each, sorting in its share of shared memory
constexpr int kVgWarps = 8;     // warps per 256-thread block
constexpr int kVgBig = kVgWarps * kVgCap;   // big leaves up to this many points sort in the whole block's shared memory
constexpr int kVgTile = 2048;   // per-leaf counts per tile of vg_count_kernel's closing scan

__global__ void __launch_bounds__(256) vg_count_kernel(const float4* __restrict__ in, int n, const VgGrid* __restrict__ gp,
                                                       const unsigned* __restrict__ bitmap, int* __restrict__ vidx,
                                                       const int* __restrict__ word_prefix, const int* __restrict__ chunk_off,
                                                       int* __restrict__ cnt, int* __restrict__ slot, int* __restrict__ out_vidx,
                                                       float4* __restrict__ out, const int* __restrict__ m_ptr, int* __restrict__ off,
                                                       int* __restrict__ crowd, int* __restrict__ crowd_n, unsigned* __restrict__ done) {
  pdl_enter();
  __shared__ int warp_tot[8];
  __shared__ int carry, n_list, n_big;
  __shared__ bool is_last;
  __shared__ int tile[kVgTile];
  const int status = gp->status;
  if (status) {
    if (status == LSD_ERR_GRID_OVERFLOW)   // PCL: output = input
      for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = __ldg(in + i);
    return;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int idx = vidx[i];
    if (idx < 0) continue;   // non-finite point
    const int w = idx >> 5;
    const int rank = chunk_off[w / kScanChunk] + word_prefix[w] + __popc(bitmap[w] & ((1u << (idx & 31)) - 1u));
    vidx[i] = rank;          // from here on: the point's output slot
    slot[i] = atomicAdd(cnt + rank, 1);   // and its place in the leaf's segment (arrival order)
    out_vidx[rank] = idx;
  }
  // the last block to finish: exclusive scan of the per-leaf counts (off[m] = total) and the lists of crowded leaves (more than
  // kVgSmall points, from the front of `crowd`) and of big leaves (more than kVgCap, from its back).  Tiles of kVgTile counts,
  // read coalesced into shared memory, each thread then scanning a contiguous run of kVgTile / 256.
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) { is_last = atomicAdd(done, 1u) == gridDim.x - 1; carry = 0; n_list = 0; n_big = 0; }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int m = *m_ptr;
  constexpr int per = kVgTile / 256;
  for (int base = 0; base < m; base += kVgTile) {
#pragma unroll
    for (int u = 0; u < per; u++) { const int r = base + u * 256 + threadIdx.x; tile[u * 256 + threadIdx.x] = r < m ? __ldcg(cnt + r) : 0; }
    __syncthreads();
    int v[per], s = 0;
#pragma unroll
    for (int u = 0; u < per; u++) { v[u] = tile[threadIdx.x * per + u]; s += v[u]; }
    int incl;
    int run = block_scan_step(s, warp_tot, &carry, &incl);   // ends with a barrier: the tile may be overwritten after it
#pragma unroll
    for (int u = 0; u < per; u++) {
      const int r = base + threadIdx.x * per + u;
      if (r < m) {
        off[r] = run;
        if (v[u] > kVgCap) crowd[m - 1 - atomicAdd(&n_big, 1)] = r;
        else if (v[u] > kVgSmall) crowd[atomicAdd(&n_list, 1)] = r;
      }
      run += v[u];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { off[m] = carry; crowd_n[0] = n_list; crowd_n[1] = n_big; *done = 0u; }
}
__global__ void __launch_bounds__(256) vg_scatter_kernel(int n, const VgGrid* __restrict__ gp, const int* __restrict__ vidx,
                                                         const int* __restrict__ slot, const int* __restrict__ off, int* __restrict__ seg) {
  pdl_enter();
  if (gp->status) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int r = vidx[i];
    if (r < 0) continue;
    seg[off[r] + slot[i]] = i;
  }
}

// Ascending sort of s[0, n) by one warp (kBlock = false) or the whole block: bitonic with the first comparator of every merge
// flipped, so that every comparator puts the smaller value first and positions >= n act as +infinity that never moves (their
// comparators are skipped).
template <bool kBlock, class T>
__device__ __forceinline__ void sort_ids(T* s, int n) {
  const int tid = kBlock ? (int)threadIdx.x : (int)(threadIdx.x & 31), nt = kBlock ? (int)blockDim.x : 32;
  int lg = 0;
  while ((1 << lg) < n) lg++;
  const int pairs = (1 << lg) >> 1;
  for (int lsz = 1; lsz <= lg; lsz++) {
    for (int ls = lsz - 1; ls >= 0; ls--) {
      for (int i = tid; i < pairs; i += nt) {
        const int hi = (i >> ls) << (ls + 1), lo = i & ((1 << ls) - 1);
        const int a = hi + lo, b = ls == lsz - 1 ? hi + (2 << ls) - 1 - lo : a + (1 << ls);
        if (b < n) {
          const int x = s[a], y = s[b];
          if (x > y) { s[a] = y; s[b] = x; }
        }
      }
      if (kBlock) __syncthreads(); else __syncwarp();
    }
  }
}

// Sum of in[ids[0]], in[ids[1]], ... in that order, by one warp: 256 points requested at a time, then broadcast one by one;
// every lane adds all four channels (the same sequential fp32 chains), lane 0's result is used.
template <class T>
__device__ __forceinline__ float4 warp_sum_in_order(const float4* __restrict__ in, T* ids, int k, int lane) {
  float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
  for (int t0 = 0; t0 < k; t0 += 32 * 8) {
    float4 p[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int t = t0 + 32 * u + lane;
      p[u] = t < k ? __ldg(in + ids[t]) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int nj = min(32, k - t0 - 32 * u);
      for (int j = 0; j < nj; j++) {
        ax += __shfl_sync(0xffffffffu, p[u].x, j);
        ay += __shfl_sync(0xffffffffu, p[u].y, j);
        az += __shfl_sync(0xffffffffu, p[u].z, j);
        aw += __shfl_sync(0xffffffffu, p[u].w, j);
      }
    }
  }
  return make_float4(ax, ay, az, aw);
}

#define VG_CE(i, j) { const int lo_ = min(id[i], id[j]), hi_ = max(id[i], id[j]); id[i] = lo_; id[j] = hi_; }

// One launch for all classes: blocks take the big leaves, warps the crowded ones, threads the rest (the last threads of the grid first,
// so the warps busy with crowded leaves take none when there are fewer leaves than threads).  Every leaf writes only its own
// output slot.  Scratch returns to its idle state: counts, bitmap words and bbox.
__global__ void __launch_bounds__(256) vg_sum_kernel(const float4* __restrict__ in, const VgGrid* __restrict__ gp,
                                                     const int* __restrict__ m_ptr, const int* __restrict__ off, int* __restrict__ cnt,
                                                     int* seg, const int* __restrict__ crowd, const int* __restrict__ crowd_n,
                                                     const int* __restrict__ out_vidx, unsigned* __restrict__ bitmap,
                                                     float4* __restrict__ out, int* __restrict__ bbox) {
  pdl_enter();
  __shared__ int s_ids[kVgWarps][kVgCap];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    bbox[0] = bbox[1] = bbox[2] = 0x7f7f7f7f;
    bbox[3] = bbox[4] = bbox[5] = (int)0x80808080;
  }
  if (gp->status) return;
  const int m = *m_ptr, n_crowd = crowd_n[0], n_big = crowd_n[1], lane = threadIdx.x & 31;
  for (int j = blockIdx.x; j < n_big; j += gridDim.x) {   // big leaves: one block each, listed from the back of `crowd`
    const int r = crowd[m - 1 - j], base = off[r], k = off[r + 1] - base;
    int* sb = &s_ids[0][0];
    if (k <= kVgBig) {
      for (int t = threadIdx.x; t < k; t += blockDim.x) sb[t] = seg[base + t];
      __syncthreads();
      sort_ids<true>(sb, k);
    } else {        // rare: sorted in place in global memory
      sort_ids<true>(static_cast<volatile int*>(seg + base), k);
      sb = nullptr;
    }
    if (threadIdx.x < 32) {
      const float4 o = sb ? warp_sum_in_order(in, sb, k, lane) : warp_sum_in_order(in, static_cast<volatile int*>(seg + base), k, lane);
      const float ck = (float)k;
      if (lane == 0) out[r] = make_float4(o.x / ck, o.y / ck, o.z / ck, o.w / ck);
    }
    __syncthreads();   // the sum has read the buffer before the next big leaf overwrites it
  }
  int* sid = s_ids[threadIdx.x >> 5];
  for (int c = blockIdx.x * kVgWarps + (threadIdx.x >> 5); c < n_crowd; c += gridDim.x * kVgWarps) {   // crowded: one warp each
    const int r = crowd[c], base = off[r], k = off[r + 1] - base;
    for (int t = lane; t < k; t += 32) sid[t] = seg[base + t];
    __syncwarp();
    sort_ids<false>(sid, k);
    const float4 o = warp_sum_in_order(in, sid, k, lane);
    __syncwarp();   // every lane has read sid before the next leaf overwrites it
    const float ck = (float)k;
    if (lane == 0) out[r] = make_float4(o.x / ck, o.y / ck, o.z / ck, o.w / ck);
  }
  const int nt = gridDim.x * blockDim.x;
  for (int r = nt - 1 - (int)(blockIdx.x * blockDim.x + threadIdx.x); r < m; r += nt) {
    const int base = off[r], k = off[r + 1] - base;
    cnt[r] = 0;
    bitmap[out_vidx[r] >> 5] = 0u;
    if (k > kVgSmall) continue;
    int id[kVgSmall];
#pragma unroll
    for (int u = 0; u < kVgSmall; u++) id[u] = u < k ? seg[base + u] : 0x7fffffff;
    VG_CE(0, 2) VG_CE(1, 3) VG_CE(4, 6) VG_CE(5, 7)     // optimal 19-comparator network for 8 keys
    VG_CE(0, 4) VG_CE(1, 5) VG_CE(2, 6) VG_CE(3, 7)
    VG_CE(0, 1) VG_CE(2, 3) VG_CE(4, 5) VG_CE(6, 7)
    VG_CE(2, 4) VG_CE(3, 5)
    VG_CE(1, 4) VG_CE(3, 6)
    VG_CE(1, 2) VG_CE(3, 4) VG_CE(5, 6)
    float4 p[kVgSmall];
#pragma unroll
    for (int u = 0; u < kVgSmall; u++) p[u] = u < k ? __ldg(in + id[u]) : make_float4(0.f, 0.f, 0.f, 0.f);
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
#pragma unroll
    for (int u = 0; u < kVgSmall; u++)
      if (u < k) { ax += p[u].x; ay += p[u].y; az += p[u].z; aw += p[u].w; }
    const float ck = (float)k;
    out[r] = make_float4(ax / ck, ay / ck, az / ck, aw / ck);
  }
}
#undef VG_CE
static_assert(kVgSmall == 8, "vg_sum_kernel's sorting network is written for 8 keys");

lsd_status_t vg_run(lsd_voxelgrid* g, const float4* d_in, int n, float leaf, float4* d_out, int* d_m, cudaStream_t st) {
  if (n > g->max_points) { set_error("voxelgrid: %d points exceed capacity %d", n, g->max_points); return LSD_ERR_CAPACITY; }
  if (n <= 0) { LSD_CUDA(cudaMemsetAsync(d_m, 0, sizeof(int), st)); return LSD_OK; }
  const int nb = std::min((n + 255) / 256, 4 * lsd::kNumSms);
  const int pdl = g->pdl;
  LSD_LAUNCH(pdl, vg_minmax_kernel, std::min(nb, lsd::kNumSms), 256, st, d_in, n, g->bbox);
  LSD_LAUNCH(pdl, vg_mark_kernel, nb, 256, st, d_in, n, leaf, g->max_cells, g->bbox, g->grid, g->bitmap, g->vidx);
  LSD_LAUNCH(pdl, vg_scan_kernel, g->scan_blocks, 256, st, g->grid, g->bitmap, g->word_prefix, g->chunk_sum, g->done, d_m, n);
  if (g->input_order_sums) {
    LSD_LAUNCH(pdl, vg_count_kernel, nb, 256, st, d_in, n, g->grid, g->bitmap, g->vidx, g->word_prefix, g->chunk_sum, g->cnt, g->slot,
               g->out_vidx, d_out, d_m, g->off, g->crowd, g->crowd_n, g->done + 1);
    LSD_LAUNCH(pdl, vg_scatter_kernel, nb, 256, st, n, g->grid, g->vidx, g->slot, g->off, g->seg);
    LSD_LAUNCH(pdl, vg_sum_kernel, nb, 256, st, d_in, g->grid, d_m, g->off, g->cnt, g->seg, g->crowd, g->crowd_n, g->out_vidx, g->bitmap,
               d_out, g->bbox);
    LSD_CUDA(cudaGetLastError());
    g->launches += vg_launches(g);
    return LSD_OK;
  }
  LSD_LAUNCH(pdl, vg_accum_kernel, nb, 256, st, d_in, n, g->grid, g->bitmap, g->vidx, g->word_prefix, g->chunk_sum, g->sums, g->cnt,
             g->out_vidx, d_out);
  LSD_LAUNCH(pdl, vg_finalize_kernel, nb, 256, st, g->grid, d_m, g->sums, g->cnt, g->out_vidx, g->bitmap, d_out, g->bbox);
  LSD_CUDA(cudaGetLastError());
  g->launches += vg_launches(g);
  return LSD_OK;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

lsd_status_t lsd_voxelgrid_create(lsd_voxelgrid_t** out, int max_points, int log2_max_cells) {
  if (!out || max_points <= 0 || log2_max_cells < 10 || log2_max_cells > 31) { set_error("lsd_voxelgrid_create: bad arguments"); return LSD_ERR_INVALID; }
  lsd_status_t s = ensure_device();
  if (s) return s;
  lsd_voxelgrid* g = new lsd_voxelgrid();
  cudaGetDevice(&g->device);
  g->max_points = max_points;
  g->max_cells = log2_max_cells == 31 ? 2147483647ll : (1ll << log2_max_cells);
  const size_t words = (size_t)((g->max_cells + 31) >> 5);
  const size_t chunks = (words + kScanChunk - 1) / kScanChunk;
  g->scan_blocks = (int)std::min<size_t>(chunks, 2 * lsd::kNumSms);
  cudaError_t e = cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking);
  auto A = [&](void** p, size_t b) { if (e == cudaSuccess) e = cudaMalloc(p, b); if (e == cudaSuccess) e = cudaMemset(*p, 0, b); };
  A((void**)&g->bbox, 8 * sizeof(int));
  A((void**)&g->grid, sizeof(VgGrid));
  A((void**)&g->bitmap, words * 4);
  A((void**)&g->word_prefix, words * 4);
  A((void**)&g->chunk_sum, (chunks + 1) * 4);
  A((void**)&g->vidx, (size_t)max_points * 4);
  A((void**)&g->out_vidx, (size_t)max_points * 4);
  A((void**)&g->sums, (size_t)max_points * 4 * 8);
  A((void**)&g->cnt, (size_t)max_points * 4);
  A((void**)&g->off, ((size_t)max_points + 1) * 4);
  A((void**)&g->slot, (size_t)max_points * 4);
  A((void**)&g->seg, (size_t)max_points * 4);
  A((void**)&g->crowd, (size_t)max_points * 4);
  A((void**)&g->crowd_n, 64);
  { const char* ev = getenv("LSD_VG_SUMS"); g->input_order_sums = (ev && ev[0] == 'f') ? 0 : 1; }   // "fixed": the exact fixed-point sums
  A((void**)&g->io_in, (size_t)max_points * 16);
  A((void**)&g->io_out, (size_t)max_points * 16);
  A((void**)&g->d_m, 64);
  A((void**)&g->done, 64);
  if (e == cudaSuccess) e = cudaMemset(g->bbox, 0x7f, 3 * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(g->bbox + 3, 0x80, 3 * sizeof(int));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { lsd_status_t r = cuda_fail(e, "lsd_voxelgrid_create", __FILE__, __LINE__); lsd_voxelgrid_destroy(g); return r; }
  *out = g;
  return LSD_OK;
}

lsd_status_t lsd_voxelgrid_destroy(lsd_voxelgrid_t* g) {
  if (!g) return LSD_OK;
  cudaSetDevice(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  void* ptrs[] = {g->bbox, g->grid, g->bitmap, g->word_prefix, g->chunk_sum, g->vidx, g->out_vidx, g->sums, g->cnt, g->io_in, g->io_out, g->d_m, g->done,
                  g->off, g->slot, g->seg, g->crowd, g->crowd_n};
  for (void* p : ptrs) cudaFree(p);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
  return LSD_OK;
}

lsd_status_t lsd_voxelgrid_filter_dev(lsd_voxelgrid_t* g, const float* in_dev, int n, float leaf, float* out_dev, int* m_dev) {
  if (!g || n < 0 || leaf <= 0.f || (n > 0 && (!in_dev || !out_dev)) || !m_dev) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(g->device));
  return vg_run(g, reinterpret_cast<const float4*>(in_dev), n, leaf, reinterpret_cast<float4*>(out_dev), m_dev, g->stream);
}

lsd_status_t lsd_voxelgrid_filter(lsd_voxelgrid_t* g, const float* in_host, int n, float leaf, float* out_host, int* m) {
  if (!g || n < 0 || leaf <= 0.f || (n > 0 && (!in_host || !out_host)) || !m) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(g->device));
  if (n > g->max_points) { set_error("voxelgrid: %d points exceed capacity %d", n, g->max_points); return LSD_ERR_CAPACITY; }
  LSD_CUDA(cudaMemcpyAsync(g->io_in, in_host, (size_t)n * 16, cudaMemcpyHostToDevice, g->stream));
  lsd_status_t s = vg_run(g, g->io_in, n, leaf, g->io_out, g->d_m, g->stream);
  if (s) return s;
  int hm[2] = {0, 0};
  LSD_CUDA(cudaMemcpyAsync(&hm[0], g->d_m, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
  LSD_CUDA(cudaMemcpyAsync(&hm[1], &g->grid->status, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
  LSD_CUDA(cudaStreamSynchronize(g->stream));
  *m = hm[0];
  if (hm[0] > 0) LSD_CUDA(cudaMemcpy(out_host, g->io_out, (size_t)hm[0] * 16, cudaMemcpyDeviceToHost));
  if (hm[1] == LSD_ERR_CAPACITY) { set_error("voxelgrid: grid exceeds the handle's max_cells"); return LSD_ERR_CAPACITY; }
  return hm[1] == LSD_ERR_GRID_OVERFLOW ? LSD_ERR_GRID_OVERFLOW : LSD_OK;
}

}  // extern "C"
