// knn.cuh — warp-cooperative k-NN over the hash-voxel map (K3).
//
// One WARP per query.  Lane L owns stencil cell L: it requests that voxel's header and first three
// points (two 32-byte sectors of the 128-byte cell line) in one go, so all 19 (NEARBY18) probes of
// a query are in flight together and the dependent-load depth is 1 for voxels with <= 3 points,
// 2 otherwise.  Candidates inside the search radius are compacted with __ballot_sync into a
// per-warp shared-memory list; the K best are then peeled off with warp-wide min reductions
// (redux.sync) in canonical (d2, id) order.  Lane r ends up holding the r-th neighbour.
//
// Replaces IVox::GetClosestPoint (ivox3d.h:139-171) + IVoxNode::KNNPointByCondition
// (ivox3d_node.hpp:107-127), and — with the EXACT shell search — KD_TREE::Nearest_Search
// (ikd_Tree.cpp:367-397).
#pragma once
#include "lsd_common.cuh"

namespace lsd {

// Unity build (lsdreg.cu includes every .cu): one definition, visible to all kernels.
__constant__ Stencil c_stencils[5];  // CENTER, NEARBY6, NEARBY18, NEARBY26, NEARBY74
__host__ __device__ __forceinline__ int stencil_slot(int type) {
  return type == LSD_STENCIL_CENTER ? 0 : type == LSD_STENCIL_NEARBY6 ? 1 : type == LSD_STENCIL_NEARBY18 ? 2
       : type == LSD_STENCIL_NEARBY26 ? 3 : type == LSD_STENCIL_NEARBY74 ? 4 : -1;
}
// How far (voxels, Chebyshev in x-y) a search with this stencil reaches from the query's home voxel: the halo a tile-sharded
// map needs so that every voxel an owned query probes is held locally.  EXACT: knn_exact_warp's last shell.  -1: unknown.
__host__ __device__ __forceinline__ int stencil_reach(int type, float max_sq, float inv_res) {
  if (type == LSD_STENCIL_EXACT) return (int)ceilf(sqrtf(max_sq) * inv_res) + 1;
  const int s = stencil_slot(type);
  return s < 0 ? -1 : s == 0 ? 0 : s == 4 ? 2 : 1;
}

constexpr unsigned kFull = 0xffffffffu;
constexpr int kCandCap = 256;  // per-warp candidate list capacity (one 32-cell chunk adds <= 224)
constexpr unsigned kTaken = 0xffffffffu;

// per-warp candidate list in shared memory (SoA)
struct WarpList {
  unsigned* d;    // fp32 bits of d2 (d2 >= 0, so unsigned order == float order)
  int* id;
  unsigned* loc;  // line * 8 + slot (1..7)
  int n;          // warp-uniform
  unsigned char* cell = nullptr;  // optional: index of the stencil cell each candidate came from (reference-order export)
  int clipped = 0;                // the list was cut back to its K best at some point (list_compress): no longer every candidate
};
constexpr int kWarpListBytes = kCandCap * 12;

// the empty list of warp `warp` in a block's s_list[warps * kWarpListBytes]
__device__ __forceinline__ WarpList make_warp_list(unsigned char* s_list, int warp) {
  WarpList wl;
  wl.d = reinterpret_cast<unsigned*>(s_list + warp * kWarpListBytes);
  wl.id = reinterpret_cast<int*>(wl.d + kCandCap);
  wl.loc = reinterpret_cast<unsigned*>(wl.id + kCandCap);
  wl.n = 0;
  return wl;
}

#ifdef LSD_SIMT_EMU  // tests/simt: the host emulator has no PTX
__device__ __forceinline__ unsigned lanemask_lt() { return simt_lanemask_lt(); }
#else
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
#endif

// ballot-compact one candidate per lane into the list
// guarded (reference-order gather, which may not cut the list back): a push that would overflow is dropped and flagged
__device__ __forceinline__ void list_push(WarpList& wl, bool valid, float d2, int id, unsigned loc, int cell = 0, bool guarded = false) {
  const unsigned m = __ballot_sync(kFull, valid);
  if (guarded && wl.n + __popc(m) > kCandCap) { wl.clipped = 1; return; }
  if (valid) {
    const int pos = wl.n + __popc(m & lanemask_lt());
    wl.d[pos] = __float_as_uint(d2); wl.id[pos] = id; wl.loc[pos] = loc;
    if (wl.cell) wl.cell[pos] = (unsigned char)cell;
  }
  wl.n += __popc(m);
}

// lane r (r < n) receives the r-th best of the list in canonical (d2, id) order
struct Neighbor { float d2; int id; unsigned loc; };

template <int K>
__device__ __forceinline__ int list_select(WarpList& wl, Neighbor& out) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
  const int nf = min(wl.n, K);
  out.d2 = -1.0f; out.id = -1; out.loc = 0;
  if (wl.n <= 32) {
    // common case: one candidate per lane, selection entirely in registers (redux.sync)
    unsigned d = kTaken; int id = 0x7fffffff; unsigned loc = 0;
    if (lane < wl.n) { d = wl.d[lane]; id = wl.id[lane]; loc = wl.loc[lane]; }
    __syncwarp();  // every candidate is in a register now: the head of the list doubles as the output staging
#pragma unroll 1
    for (int r = 0; r < nf; r++) {
      const unsigned m = __reduce_min_sync(kFull, d);
      const unsigned eq = __ballot_sync(kFull, d == m);
      int win = __ffs(eq) - 1;
      if (eq & (eq - 1)) {  // equal distances: canonical order breaks ties by id
        const int mi = __reduce_min_sync(kFull, d == m ? id : 0x7fffffff);
        win = __ffs(__ballot_sync(kFull, d == m && id == mi)) - 1;
      }
      if (lane == win) { wl.d[r] = m; wl.id[r] = id; wl.loc[r] = loc; d = kTaken; }
    }
    __syncwarp();
    if (lane < nf) { out.d2 = __uint_as_float(wl.d[lane]); out.id = wl.id[lane]; out.loc = wl.loc[lane]; }
    __syncwarp();
    return nf;
  }
#pragma unroll 1
  for (int r = 0; r < nf; r++) {
    unsigned bd = kTaken; int bi = 0x7fffffff; int bp = 0;
    for (int p = lane; p < wl.n; p += 32) {
      const unsigned d = wl.d[p]; const int i = wl.id[p];
      if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; bp = p; }
    }
    const unsigned m = __reduce_min_sync(kFull, bd);
    const int mi = __reduce_min_sync(kFull, bd == m ? bi : 0x7fffffff);
    const unsigned wm = __ballot_sync(kFull, bd == m && bi == mi);
    const int win = __ffs(wm) - 1;
    unsigned wloc = 0;
    if (lane == win) { wloc = wl.loc[bp]; wl.d[bp] = kTaken; }
    wloc = __shfl_sync(kFull, wloc, win);
    if (lane == r) { out.d2 = __uint_as_float(m); out.id = mi; out.loc = wloc; }
    __syncwarp();
  }
  return nf;
}

// keep only the K best in the list
template <int K>
__device__ __forceinline__ void list_compress(WarpList& wl) {
  Neighbor nb;
  const int nf = list_select<K>(wl, nb);
  const int lane = threadIdx.x & 31;
  if (lane < nf) { wl.d[lane] = __float_as_uint(nb.d2); wl.id[lane] = nb.id; wl.loc[lane] = nb.loc; }
  wl.n = nf;
  wl.clipped = 1;
  __syncwarp();
}

// Each lane resolves ONE voxel (key == 0: none) and pushes its in-radius points.
// Phase A: header + points 0..2 (sectors 0,1) requested together; phase B: points 3..6 if needed;
// overflow levels (> 7 points in the voxel) are walked cooperatively afterwards.
template <int K>
__device__ __forceinline__ void warp_scan_cells(const MapView& mv, unsigned long long key, float qx, float qy, float qz,
                                                float max_sq, bool inclusive, WarpList& wl, int cell_base = 0, bool guarded = false) {
  const int my_cell = cell_base + (int)(threadIdx.x & 31);
  unsigned long long s = 0;
  const CellLine* ln = mv.lines;
  unsigned cnt = 0;
  {
    float4 p[3];
    p[0] = p[1] = p[2] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (key != 0ull) {
      // Walk the probe sequence in the TAG array (8 slots per 8-byte load, L2-resident): an absent
      // voxel is recognised without touching a line, a present one costs exactly one line access
      // (plus one per tag collision, 1/255 per occupied slot walked).
      constexpr unsigned long long k01 = 0x0101010101010101ull, k7f = 0x7f7f7f7f7f7f7f7full;
      const unsigned long long hh = hash_key(key);
      const unsigned long long tagv = (unsigned long long)slot_tag(hh) * k01;
      s = hh & mv.mask;
      bool present = false;
      for (unsigned walked = 0; walked < kMaxProbe && !present;) {
        const unsigned pos = (unsigned)(s & 7ull), nv = 8u - pos;
        const unsigned long long v = __ldg(reinterpret_cast<const unsigned long long*>(mv.tags + (s & ~7ull))) >> (8u * pos);
        // exact zero-byte flags (bit 7 of each zero byte); bytes shifted in above nv are zero, so fe <= nv
        const unsigned long long ze = ~(((v & k7f) + k7f) | v | k7f);
        const unsigned long long x = v ^ tagv;
        unsigned long long zm = ~(((x & k7f) + k7f) | x | k7f);
        const unsigned fe = ze ? (unsigned)(__ffsll((long long)ze) - 1) >> 3 : 8u;
        while (zm) {
          const unsigned fm = (unsigned)(__ffsll((long long)zm) - 1) >> 3;
          if (fm >= fe) break;  // the probe sequence ends at the first empty slot
          zm &= zm - 1ull;
          const unsigned long long c = (s + fm) & mv.mask;
          const CellLine* cl = mv.lines + c;
          const uint4 h = ldg_u4(cl);
          const float4 a0 = ldg_f4(&cl->pts[0]), a1 = ldg_f4(&cl->pts[1]), a2 = ldg_f4(&cl->pts[2]);
          if (((unsigned long long)h.x | ((unsigned long long)h.y << 32)) == key) {
            present = true; s = c; ln = cl; cnt = h.z; p[0] = a0; p[1] = a1; p[2] = a2;
            break;
          }
        }
        if (present || fe < nv) break;
        walked += nv;
        s = (s + nv) & mv.mask;
      }
    }
#pragma unroll
    for (int j = 0; j < 3; j++) {
      bool valid = (unsigned)j < cnt;
      float d2 = 0.f;
      if (valid) {
        d2 = dist2(qx, qy, qz, p[j].x, p[j].y, p[j].z);
        valid = inclusive ? (d2 <= max_sq) : (d2 < max_sq);
      }
      list_push(wl, valid, d2, __float_as_int(p[j].w), (unsigned)(s * 8 + j + 1), my_cell, guarded);
    }
  }
  if (__any_sync(kFull, cnt > 3u)) {  // phase B: sectors 2,3 of the lines that need them
    const unsigned n0 = min(cnt, (unsigned)kPtsPerLine);
    float4 p[4];
    p[0] = p[1] = p[2] = p[3] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n0 > 3) { p[0] = ldg_f4(&ln->pts[3]); p[1] = ldg_f4(&ln->pts[4]); p[2] = ldg_f4(&ln->pts[5]); p[3] = ldg_f4(&ln->pts[6]); }
#pragma unroll
    for (int j = 3; j < kPtsPerLine; j++) {
      bool valid = (unsigned)j < n0;
      float d2 = 0.f;
      if (valid) {
        d2 = dist2(qx, qy, qz, p[j - 3].x, p[j - 3].y, p[j - 3].z);
        valid = inclusive ? (d2 <= max_sq) : (d2 < max_sq);
      }
      list_push(wl, valid, d2, __float_as_int(p[j - 3].w), (unsigned)(s * 8 + j + 1), my_cell, guarded);
    }
  }
  // overflow levels: voxels with more than 7 points (rare in a 0.5 m-thinned map)
  unsigned ovf = __ballot_sync(kFull, cnt > (unsigned)kPtsPerLine);
  while (ovf) {
    const int src = __ffs(ovf) - 1;
    ovf &= ovf - 1;
    const unsigned long long okey = __shfl_sync(kFull, key, src);
    const unsigned ocnt = __shfl_sync(kFull, cnt, src);
    const int levels = min((int)((ocnt - 1) / kPtsPerLine), kMaxLevel);
    for (int L = 1; L <= levels; L++) {
      const unsigned long long kl = okey | ((unsigned long long)L << 57);
      unsigned long long sl = hash_key(kl) & mv.mask;
      bool found = false;
      for (unsigned probe = 0; probe < kMaxProbe; probe++) {  // warp-uniform probe
        const uint4 hh = ldg_u4(mv.lines + sl);
        const unsigned long long k2 = (unsigned long long)hh.x | ((unsigned long long)hh.y << 32);
        if (k2 == kl) { found = true; break; }
        if (k2 == 0ull) break;
        sl = (sl + 1) & mv.mask;
      }
      if (!found) continue;
      const int n = (int)min(ocnt - (unsigned)(L * kPtsPerLine), (unsigned)kPtsPerLine);
      const int lane = threadIdx.x & 31;
      bool valid = lane < n;
      float d2 = 0.f; float4 q = make_float4(0, 0, 0, 0);
      if (valid) {
        q = ldg_f4(&(mv.lines + sl)->pts[lane]);
        d2 = dist2(qx, qy, qz, q.x, q.y, q.z);
        valid = inclusive ? (d2 <= max_sq) : (d2 < max_sq);
      }
      if (!guarded && wl.n + 7 > kCandCap) list_compress<K>(wl);
      list_push(wl, valid, d2, __float_as_int(q.w), (unsigned)(sl * 8 + lane + 1), cell_base + src, guarded);
    }
  }
}

// The stencil offsets a lane is responsible for (cell c*32 + lane of the stencil), loaded once per
// kernel: constant-memory reads indexed by the lane would otherwise be replayed 32 ways per query.
struct LaneStencil {
  int n_chunks;
  int off[3];  // packed (dx, dy, dz) + valid flag per 32-cell chunk
};
__device__ __forceinline__ LaneStencil lane_stencil(int st_slot) {
  LaneStencil ls;
  ls.n_chunks = 0;
  ls.off[0] = ls.off[1] = ls.off[2] = 0;
  if (st_slot < 0) return ls;
  const Stencil& st = c_stencils[st_slot];
  const int lane = threadIdx.x & 31;
  ls.n_chunks = (st.n + 31) >> 5;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const int idx = c * 32 + lane;
    if (idx < st.n)
      ls.off[c] = 0x1000000 | ((st.off[idx][0] & 0xff) << 16) | ((st.off[idx][1] & 0xff) << 8) | (st.off[idx][2] & 0xff);
  }
  return ls;
}

// Fixed-stencil search (IVox NEARBY*).  32 stencil cells per pass.
template <int K>
__device__ __forceinline__ int knn_stencil_warp(const MapView& mv, const LaneStencil& ls, float qx, float qy, float qz,
                                                float max_sq, WarpList& wl, Neighbor& out) {
  const int3 c = pos2grid(qx, qy, qz, mv.inv_res);
  wl.n = 0;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    if (ch < ls.n_chunks) {
      if (ch > 0 && wl.n > kCandCap - 7 * 32) list_compress<K>(wl);
      unsigned long long key = 0ull;
      const int o = ls.off[ch];
      if (o) {
        const int x = c.x + (int)(signed char)(o >> 16), y = c.y + (int)(signed char)(o >> 8), z = c.z + (int)(signed char)o;
        if (coord_ok(x, y, z)) key = pack_key(x, y, z, 0);
      }
      warp_scan_cells<K>(mv, key, qx, qy, qz, max_sq, false, wl);
    }
  }
  return list_select<K>(wl, out);
}

// The gather half of knn_stencil_warp on its own: every in-range point of the stencil cells in the list, tagged with its cell
// (wl.cell must be set).  wl.clipped != 0 afterwards: more than kCandCap candidates, the list is incomplete.
template <int K>
__device__ __forceinline__ void knn_stencil_gather(const MapView& mv, const LaneStencil& ls, float qx, float qy, float qz,
                                                   float max_sq, WarpList& wl) {
  const int3 c = pos2grid(qx, qy, qz, mv.inv_res);
  wl.n = 0; wl.clipped = 0;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    if (ch < ls.n_chunks) {
      unsigned long long key = 0ull;
      const int o = ls.off[ch];
      if (o) {
        const int x = c.x + (int)(signed char)(o >> 16), y = c.y + (int)(signed char)(o >> 8), z = c.z + (int)(signed char)o;
        if (coord_ok(x, y, z)) key = pack_key(x, y, z, 0);
      }
      warp_scan_cells<K>(mv, key, qx, qy, qz, max_sq, false, wl, ch * 32, true);
    }
  }
  __syncwarp();
}

// Exact k-NN with d2 <= max_sq by Chebyshev shells around the query's voxel; stops as soon as the
// K-th best distance is below the lower bound of every unseen shell.
template <int K>
__device__ __forceinline__ int knn_exact_warp(const MapView& mv, float qx, float qy, float qz, float max_sq, WarpList& wl,
                                              Neighbor& out) {
  const int lane = threadIdx.x & 31;
  const int3 c = pos2grid(qx, qy, qz, mv.inv_res);
  const int rmax = (int)ceilf(sqrtf(max_sq) * mv.inv_res) + 1;
  wl.n = 0;
  int nf = 0;
  out.d2 = -1.0f; out.id = -1; out.loc = 0;
  for (int r = 0; r <= rmax; r++) {
    if (r >= 1 && nf == K) {
      // a point in shell >= r is at least (r-1)*res away along one axis (voxels are centred on
      // integer multiples of res, the query is anywhere inside its own voxel)
      const float kth = __shfl_sync(kFull, out.d2, K - 1);
      const float lo = (float)(r - 1) * mv.res * (1.0f - 1e-5f);
      if (kth < lo * lo) break;
    }
    const int side = 2 * r + 1;
    const int ncell = side * side * side;
    for (int t0 = 0; t0 < ncell; t0 += 32) {
      if (wl.n > kCandCap - 7 * 32) list_compress<K>(wl);
      const int t = t0 + lane;
      unsigned long long key = 0ull;
      if (t < ncell) {
        const int i = t / (side * side) - r, j = (t / side) % side - r, l = t % side - r;
        if (max(max(abs(i), abs(j)), abs(l)) == r) {
          const int x = c.x + i, y = c.y + j, z = c.z + l;
          if (coord_ok(x, y, z)) key = pack_key(x, y, z, 0);
        }
      }
      if (__any_sync(kFull, key != 0ull)) warp_scan_cells<K>(mv, key, qx, qy, qz, max_sq, true, wl);
    }
    // top-K so far (needed for the stopping rule); the list is cut back to those K
    nf = list_select<K>(wl, out);
    if (lane < nf) { wl.d[lane] = __float_as_uint(out.d2); wl.id[lane] = out.id; wl.loc[lane] = out.loc; }
    wl.n = nf;
    __syncwarp();
  }
  return nf;
}

// `ls` = lane_stencil(stencil_slot(stencil_type)), hoisted out of the caller's query loop
template <int K>
__device__ __forceinline__ int knn_search_warp(const MapView& mv, int stencil_type, const LaneStencil& ls, float qx, float qy,
                                               float qz, float max_sq, WarpList& wl, Neighbor& out) {
  if (stencil_type == LSD_STENCIL_EXACT) return knn_exact_warp<K>(mv, qx, qy, qz, max_sq, wl, out);
  return knn_stencil_warp<K>(mv, ls, qx, qy, qz, max_sq, wl, out);
}

// coordinates of a stored neighbour from its location code
__device__ __forceinline__ float4 load_loc(const MapView& mv, unsigned loc) {
  const CellLine* ln = mv.lines + (loc >> 3);
  return ldg_f4(&ln->pts[(loc & 7) - 1]);
}

}  // namespace lsd
