// brick.cuh — the brick layout of the hash-voxel map and the TMA-staged batched k-NN over it (K3, batch shape).
//
// Why: a hash of 128-byte voxel lines costs every query its own DRAM trips (tag -> line, per stencil cell), with most lanes
// of a warp idle.  Here the same points are ALSO stored brick by brick: a brick is 8 x 8 x 4 voxels (4 x 4 x 2 m at 0.5 m) and its
// page holds every point of those voxels PLUS a one-voxel halo (a point near a brick face is stored in up to 8 pages), so
// the 19-cell NEARBY18 stencil of any query whose home voxel lies in the brick is answered from that ONE page.  A batch
// is binned by brick (three small kernels), then a persistent CTA per work item pulls the page into shared memory with
// ONE cp.async.bulk (TMA, mbarrier completion) and answers up to 128 queries from it: a page is read once per ~20
// queries instead of ~7 lines per query, and every dependent load of the search is a shared-memory load.
//
// Page (kPageBytes = 4608, 128-byte aligned), one per directory slot:
//   [  0,  16)  reserved (brick key, for debugging)
//   [ 16, 616)  u8 head[600]    first point (index + 1) of each of the 10 x 10 x 6 region cells, 0 = empty
//   [616, 848)  u8 next[232]    next point (index + 1) of the same cell, 0 = end of list
//   [848,4560)  float4 pts[232] (x, y, z, id)
// Directory: open addressing over `keys` (u64: level:7 | bx:19 | by:19 | bz:19, 0 = empty) with the point counter of every
// brick in the parallel array `totals` (4 B per slot: the whole array stays in L2, so inserts and the planner never touch a
// page to learn its fill).  Points beyond 232 go to pages keyed (brick, level >= 1) found by hashing — the same
// no-linked-list, no-spin rule as the voxel lines (lsd_common.cuh).  Inserts are lock-free: atomicAdd slot claim, one
// float4 store, byte exchange on the cell's list head.  List order depends on arrival; results do not (canonical (d2, id)
// selection, the same candidate set as IVox::GetClosestPoint, ivox3d.h:139-171 — bit-identical to the line-based kernels).
// The vertical brick origin is shifted by one voxel (kBrickZOff) so that the z = 0 layer — the ground of a map that starts
// at the sensor — is not a brick boundary (it would double the replication of the most populated layer).
#pragma once
#include "lsd_common.cuh"

namespace lsd {

constexpr int kBrickXY = 8, kBrickZ = 4, kBrickZOff = 1;
constexpr int kRegXY = kBrickXY + 2, kRegZ = kBrickZ + 2;
constexpr int kRegCells = kRegXY * kRegXY * kRegZ;   // 600
constexpr int kBrickCap = 232;                        // points per page (u8 indices: <= 255)
constexpr int kPageHead = 16;
constexpr int kPageNext = kPageHead + kRegCells;      // 616
constexpr int kPagePts = kPageNext + kBrickCap;       // 848
constexpr int kPageBytes = 4608;
constexpr int kBrickQC = 32;                          // queries per work item: one WARP answers an item, one query per lane
constexpr int kBrickWarps = 4;                        // warps per CTA of the query kernel (two page buffers each)
static_assert(kPagePts % 16 == 0 && kPagePts + 16 * kBrickCap <= kPageBytes && kPageBytes % 128 == 0, "page layout");

// A query in brick order, in one of two formats chosen per batch (brick_batch_is_ordered):
//   32 bytes (x, y, z, w, index, pad) — one full sector per entry: a SHUFFLED batch scatters its entries all over the list, and a
//     16-byte store into a sector somebody else completes later costs a read-modify-write;
//   16 bytes (x, y, z, index) — a batch that arrives in spatial order fills both halves of a sector within one warp, and then
//     half the bytes are simply half the bytes.
struct __align__(32) BrickQuery { float4 p; int qi; int pad[3]; };
__device__ __forceinline__ void brick_query_store(BrickQuery* list, int pos, float4 q, int i, bool compact) {
  if (compact) reinterpret_cast<float4*>(list)[pos] = make_float4(q.x, q.y, q.z, __int_as_float(i));
  else { BrickQuery e; e.p = q; e.qi = i; e.pad[0] = e.pad[1] = e.pad[2] = 0; list[pos] = e; }
}
__device__ __forceinline__ void brick_query_load(const BrickQuery* list, int pos, bool compact, float4* p, int* qi) {
  if (compact) { const float4 v = __ldg(reinterpret_cast<const float4*>(list) + pos); *p = v; *qi = __float_as_int(v.w); }
  else { *p = __ldg(&list[pos].p); *qi = __ldg(&list[pos].qi); }
}
// A batch counts as spatially ordered when, in the sampled blocks of the bin kernel (one in eight), at least a quarter of the
// queries share their home brick with their predecessor (ctr[3]): neighbours in the batch are then neighbours in the list, and
// a warp's stores complete whole sectors.  (A shuffled batch of 2 M queries over 218 k bricks: 1e-4; the benchmark's
// voxel-sorted batch: 0.5-0.65.)
__device__ __forceinline__ bool brick_batch_is_ordered(const unsigned* ctr, int nq) {
  const unsigned sampled = (unsigned)((((nq + 255) / 256 + 7) / 8) * 256);
  return 4u * __ldcg(ctr + 3) >= sampled;
}
struct __align__(8) BrickWork { int slot, qbase, qn; unsigned total; unsigned long long key; };   // one (brick page, <= 32 queries) unit of the search

// ------------------------------------------------------------------ directory
__device__ __forceinline__ long long brick_find(const BrickView& bv, unsigned long long key) {
  unsigned long long s = hash_key(key) & bv.mask;
  for (unsigned probe = 0; probe < kMaxProbe; probe++) {
    const unsigned long long cur = __ldcg(bv.keys + s);
    if (cur == key) return (long long)s;
    if (cur == 0ull) return -1;
    s = (s + 1) & bv.mask;
  }
  return -1;
}
__device__ __forceinline__ long long brick_find_or_claim(const BrickView& bv, unsigned long long key) {
  unsigned long long s = hash_key(key) & bv.mask;
  for (unsigned probe = 0; probe < kMaxProbe; probe++) {
    unsigned long long* kp = bv.keys + s;
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(kp);
    if (cur == key) return (long long)s;
    if (cur == 0ull) {
      const unsigned long long old = atomicCAS(kp, 0ull, key);
      if (old == 0ull) { atomicAdd(&bv.counters[0], 1ull); return (long long)s; }
      if (old == key) return (long long)s;
    }
    s = (s + 1) & bv.mask;
  }
  return -1;
}

// brick of a voxel, and the voxel's coordinates inside the brick's own 8 x 8 x 4 range
__device__ __forceinline__ void brick_of(int cx, int cy, int cz, int3* b, int3* l) {
  b->x = floor_div(cx, kBrickXY); b->y = floor_div(cy, kBrickXY); b->z = floor_div(cz + kBrickZOff, kBrickZ);
  l->x = cx - b->x * kBrickXY; l->y = cy - b->y * kBrickXY; l->z = cz + kBrickZOff - b->z * kBrickZ;
}

// exchange one byte of a u8 array (32-bit CAS on the containing word): returns the previous value
__device__ __forceinline__ unsigned byte_exch(unsigned char* addr, unsigned v) {
  unsigned* w = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned long long>(addr) & ~3ull);
  const unsigned sh = (unsigned)(reinterpret_cast<unsigned long long>(addr) & 3ull) * 8u;
  unsigned old = *reinterpret_cast<volatile unsigned*>(w), assumed;
  do {
    assumed = old;
    old = atomicCAS(w, assumed, (assumed & ~(0xffu << sh)) | (v << sh));
  } while (old != assumed);
  return (old >> sh) & 0xffu;
}

// Store one point (already accepted by the voxel lines) in the page of every brick whose region contains its voxel.
__device__ __forceinline__ void brick_insert_point(const BrickView& bv, int cx, int cy, int cz, float4 p) {
  int3 b0, l;
  brick_of(cx, cy, cz, &b0, &l);
#pragma unroll 1
  for (int dz = -1; dz <= 1; dz++) {
    if ((dz < 0 && l.z != 0) || (dz > 0 && l.z != kBrickZ - 1)) continue;
#pragma unroll 1
    for (int dy = -1; dy <= 1; dy++) {
      if ((dy < 0 && l.y != 0) || (dy > 0 && l.y != kBrickXY - 1)) continue;
#pragma unroll 1
      for (int dx = -1; dx <= 1; dx++) {
        if ((dx < 0 && l.x != 0) || (dx > 0 && l.x != kBrickXY - 1)) continue;
        const int rc = ((l.z - dz * kBrickZ + 1) * kRegXY + (l.y - dy * kBrickXY + 1)) * kRegXY + (l.x - dx * kBrickXY + 1);
        const unsigned long long key = pack_key(b0.x + dx, b0.y + dy, b0.z + dz, 0);
        long long s = brick_find_or_claim(bv, key);
        if (s < 0) { atomicAdd(&bv.counters[2], 1ull); continue; }
        const unsigned idx = atomicAdd(bv.totals + s, 1u);
        const unsigned L = idx / kBrickCap, j = idx % kBrickCap;
        if (L > 0) {
          if (L > (unsigned)kMaxLevel) { atomicAdd(&bv.counters[2], 1ull); continue; }
          s = brick_find_or_claim(bv, key | ((unsigned long long)L << 57));
          if (s < 0) { atomicAdd(&bv.counters[2], 1ull); continue; }
        }
        unsigned char* page = bv.pages + (size_t)s * kPageBytes;
        reinterpret_cast<float4*>(page + kPagePts)[j] = p;
        page[kPageNext + j] = (unsigned char)byte_exch(page + kPageHead + rc, j + 1u);
        atomicAdd(&bv.counters[1], 1ull);
      }
    }
  }
}

// ------------------------------------------------------------------ TMA page load (cp.async.bulk + mbarrier)
__device__ __forceinline__ unsigned smem_u32(const void* p) {
#ifdef LSD_SIMT_EMU
  return 0u;
#else
  return (unsigned)__cvta_generic_to_shared(p);
#endif
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar) {
#ifdef LSD_SIMT_EMU
  *bar = 0ull;
#else
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
}
// One thread: arm the barrier with the byte count and issue the two bulk copies of a page holding n points
// (head + next block, then the points actually stored).  Every byte lands in shared memory without passing a register.
__device__ __forceinline__ void page_load_issue(unsigned char* smem_page, unsigned long long* bar, const unsigned char* gpage, unsigned n) {
#ifdef LSD_SIMT_EMU
  memcpy(smem_page, gpage, kPagePts);
  if (n) memcpy(smem_page + kPagePts, gpage + kPagePts, 16u * n);
#else
  const unsigned bytes_b = 16u * n;
  const unsigned dst = smem_u32(smem_page), b = smem_u32(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"((unsigned)kPagePts + bytes_b) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(gpage), "r"((unsigned)kPagePts), "r"(b) : "memory");
  if (bytes_b)
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst + (unsigned)kPagePts), "l"(gpage + kPagePts), "r"(bytes_b), "r"(b) : "memory");
#endif
}
// Every thread: wait until the bytes of the current phase have landed.
__device__ __forceinline__ void page_load_wait(unsigned long long* bar, unsigned phase) {
#ifdef LSD_SIMT_EMU
  __syncwarp();
#else
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LSD_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LSD_DONE;\n"
      "bra LSD_WAIT;\n"
      "LSD_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
#endif
}

// ------------------------------------------------------------------ batch binning
// K-A: home brick of every query; queries whose brick does not exist are answered here (nothing within reach).
__global__ void __launch_bounds__(256) brick_bin_kernel(BrickView bv, float inv_res, const float4* __restrict__ q, int nq, int k,
                                                        int* __restrict__ q_slot, int* __restrict__ q_rank, unsigned* __restrict__ bin_count,
                                                        int* __restrict__ out_idx, float* __restrict__ out_d2, int* __restrict__ out_cnt,
                                                        unsigned* __restrict__ ctr3) {
  __shared__ unsigned s_same;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool sample = (blockIdx.x & 7) == 0;       // one block in eight tells whether the batch arrives in spatial order
  if (sample && threadIdx.x == 0) s_same = 0u;
  if (sample) __syncthreads();
  long long s = -1;
  if (i < nq) {
    const float4 p = __ldg(q + i);
    const int3 c = pos2grid(p.x, p.y, p.z, inv_res);
    // beyond +-(2^18) no stencil cell is a valid voxel (coord_ok): nothing can be near
    if (abs(c.x) <= kCoordBias && abs(c.y) <= kCoordBias && abs(c.z) <= kCoordBias) {
      int3 b, l;
      brick_of(c.x, c.y, c.z, &b, &l);
      s = brick_find(bv, pack_key(b.x, b.y, b.z, 0));
    }
  }
  if (sample) {     // block-uniform: every lane takes part in the shuffle; one shared atomic per warp, one global per sampled block
    const long long prev = __shfl_up_sync(0xffffffffu, s, 1);
    const unsigned same = __ballot_sync(0xffffffffu, (threadIdx.x & 31) != 0 && s >= 0 && prev == s);
    if ((threadIdx.x & 31) == 0 && same) atomicAdd(&s_same, (unsigned)__popc(same));
    __syncthreads();
    if (threadIdx.x == 0 && s_same) atomicAdd(ctr3, s_same);
  }
  if (i >= nq) return;
  q_slot[i] = (int)s;
  if (s < 0) {
    for (int r = 0; r < k; r++) { out_idx[(size_t)i * k + r] = -1; out_d2[(size_t)i * k + r] = -1.0f; }
    out_cnt[i] = 0;
    return;
  }
  q_rank[i] = (int)atomicAdd(bin_count + s, 1u);
}

// K-B: one thread per directory slot: a contiguous range of the sorted query list for every brick that has queries, cut
// into work items of <= kBrickQC queries.  ctr[0] = queries placed, ctr[1] = work items.  Leaves bin_count zeroed.
// The two running totals are claimed once per BLOCK (block-wide exclusive scan, then one atomicAdd each): one atomic per
// occupied slot on the same two words serialises the whole kernel.
__device__ __forceinline__ unsigned block_excl_scan_256(unsigned v, unsigned* warp_tot, unsigned* total) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (unsigned)o) inc += t; }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  unsigned woff = 0, tot = 0;
  for (unsigned k = 0; k < 8; k++) { const unsigned t = warp_tot[k]; if (k < warp) woff += t; tot += t; }
  __syncthreads();
  *total = tot;
  return woff + inc - v;
}
__global__ void __launch_bounds__(256) brick_plan_kernel(BrickView bv, unsigned long long n_slots, unsigned* __restrict__ bin_count,
                                                         int* __restrict__ bin_base, BrickWork* __restrict__ work, unsigned* __restrict__ ctr) {
  __shared__ unsigned warp_tot[8];
  __shared__ unsigned s_base[2];
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned c = 0;
  if (s < n_slots) { c = bin_count[s]; if (c) bin_count[s] = 0u; }
  const unsigned nch = (c + kBrickQC - 1) / kBrickQC;      // items of <= 32 queries; a small last item spreads each query over 2 / 4 / 8 lanes
  unsigned tot_c, tot_w;
  const unsigned off_c = block_excl_scan_256(c, warp_tot, &tot_c);
  const unsigned off_w = block_excl_scan_256(nch, warp_tot, &tot_w);
  if (threadIdx.x == 0) { s_base[0] = tot_c ? atomicAdd(ctr + 0, tot_c) : 0u; s_base[1] = tot_w ? atomicAdd(ctr + 1, tot_w) : 0u; }
  __syncthreads();
  if (!c) return;
  const unsigned base = s_base[0] + off_c, w0 = s_base[1] + off_w;
  bin_base[s] = (int)base;
  const unsigned total = __ldcg(bv.totals + s);
  const unsigned long long key = __ldcg(bv.keys + s);
  for (unsigned ch = 0; ch < nch; ch++) {
    BrickWork w;
    w.slot = (int)s; w.qbase = (int)(base + ch * kBrickQC); w.qn = (int)min((unsigned)kBrickQC, c - ch * kBrickQC); w.total = total; w.key = key;
    work[w0 + ch] = w;
  }
}

// K-C: the batch in brick order: query + its index in the caller's batch, one 32-byte sector each, so that the search
// reads its queries with one contiguous load instead of index -> query (two dependent DRAM trips)
__global__ void __launch_bounds__(256) brick_scatter_kernel(const float4* __restrict__ q, const int* __restrict__ q_slot,
                                                            const int* __restrict__ q_rank, const int* __restrict__ bin_base, int nq,
                                                            BrickQuery* __restrict__ sorted, const unsigned* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const int s = q_slot[i];
  if (s < 0) return;
  brick_query_store(sorted, bin_base[s] + q_rank[i], __ldg(q + i), i, brick_batch_is_ordered(ctr, nq));
}

// ------------------------------------------------------------------ K-D: the search
// Persistent warps, one work item at a time: (brick page, <= 32 queries).  Every warp owns a page buffer and an mbarrier:
// lane 0 claims the next item and issues the page's bulk copies, the lanes load their queries meanwhile, the warp waits
// on the barrier and answers the item's queries from shared memory.
//
// What the instruction profile of the first two versions asked for (issue-bound with a minority of the 32 lanes active,
// half of the instructions in a branchy insertion running a few lanes wide):
//  * lane groups — a brick of the benchmark batch has ~13 queries, so an item of qn queries gives each query
//    g = 32 / pow2ceil(qn) lanes (1, 2, 4 or 8); lane `sub` of a group takes stencil cells sub, sub + g, ...
//  * a FLAT walk — phase 1 collects the heads of the lane's non-empty cells into a 28-byte queue in shared memory (uniform
//    19 / g iterations, predicated stores); phase 2 is ONE loop that handles one stored point per iteration, hopping to the
//    next queued cell when a list ends, so lanes diverge only in their total point count, not per cell;
//  * a branch-free top-K — candidates are 64-bit keys (fp32 bits of d2 << 32 | id: d2 >= 0, so integer order is the
//    canonical (d2, id) order) inserted by K min / max stages, no early-outs;
//  * a merge of the group's sorted lists by log2(g) butterfly steps: min(A[i], B[K-1-i]) keeps the K smallest of the union
//    (a bitonic sequence), a 9-comparator network sorts them again.
// Any split of the candidate set gives the same K best, so results stay bit-identical to the line-based kernels.
struct KeyTop5 {
  unsigned long long k[5];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < 5; i++) k[i] = ~0ull;
  }
  __device__ __forceinline__ void insert(unsigned long long x) {
#pragma unroll
    for (int i = 0; i < 5; i++) { const unsigned long long lo = min(k[i], x); x = max(k[i], x); k[i] = lo; }
  }
  __device__ __forceinline__ static void cx(unsigned long long& a, unsigned long long& b) { const unsigned long long lo = min(a, b); b = max(a, b); a = lo; }
  // K smallest of this (sorted) and the partner lane's (sorted) list, sorted again
  __device__ __forceinline__ void merge_xor(int x) {
    unsigned long long o[5];
#pragma unroll
    for (int i = 0; i < 5; i++) o[i] = __shfl_xor_sync(0xffffffffu, k[i], x);
#pragma unroll
    for (int i = 0; i < 5; i++) k[i] = min(k[i], o[4 - i]);
    // optimal 9-comparator sorting network for 5 keys
    cx(k[0], k[1]); cx(k[3], k[4]); cx(k[2], k[4]); cx(k[2], k[3]); cx(k[0], k[3]); cx(k[0], k[2]); cx(k[1], k[4]); cx(k[1], k[3]); cx(k[1], k[2]);
  }
};

template <int K>
__global__ void __launch_bounds__(kBrickWarps * 32) brick_knn_kernel(BrickView bv, float inv_res, int st_slot, float max_sq,
                                                                     const BrickQuery* __restrict__ sorted, int nq,
                                                                     const BrickWork* __restrict__ work, unsigned* __restrict__ ctr,
                                                                     int* __restrict__ out_idx, float* __restrict__ out_d2, int* __restrict__ out_cnt) {
  // Two page buffers per warp: while item N is answered from one, item N + 1's page lands in the other, its queries sit in
  // registers and item N + 2's descriptor is on its way — after the prologue no item waits for a memory round trip.
  __shared__ __align__(128) unsigned char pages[kBrickWarps][2][kPageBytes];
  __shared__ __align__(8) unsigned long long bars[kBrickWarps][2];
  __shared__ unsigned char cellq[kBrickWarps][32][28];   // per lane: heads of its non-empty stencil cells (<= 27: NEARBY26)
  __shared__ int s_off[32];                              // the stencil as region-index offsets
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { mbar_init(&bars[warp][0]); mbar_init(&bars[warp][1]); }
  const Stencil& st = c_stencils[st_slot];
  const int n_cells = st.n;                              // <= 27 for the stencils served here
  if (threadIdx.x < 32) s_off[threadIdx.x] = (int)threadIdx.x < n_cells ? (st.off[threadIdx.x][2] * kRegXY + st.off[threadIdx.x][1]) * kRegXY + st.off[threadIdx.x][0] : 0;
  __syncthreads();
  const unsigned n_work = __ldcg(ctr + 1);
  const bool compact = brick_batch_is_ordered(ctr, nq);   // the list's entry format (warp-uniform)
  unsigned char* myq = cellq[warp][lane];
  unsigned phase = 0u;                                   // bit b = parity the next wait on buffer b expects
  const BrickWork none = {0, 0, 0, 0u, 0ull};

  auto claim = [&]() { unsigned w = 0; if (lane == 0) w = atomicAdd(ctr + 2, 1u); return __shfl_sync(0xffffffffu, w, 0); };
  auto lanes_log2 = [](int qn) { return qn <= 4 ? 3 : qn <= 8 ? 2 : qn <= 16 ? 1 : 0; };   // lanes per query: 8 / 4 / 2 / 1
  auto load_query = [&](const BrickWork& it, float4* p, int* qi) {
    const int t = lane >> lanes_log2(it.qn);
    *qi = -1; *p = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < it.qn) brick_query_load(sorted, it.qbase + t, compact, p, qi);
  };

  // prologue: item 0 in flight, item 1 described
  unsigned w = claim();
  BrickWork it = w < n_work ? work[w] : none;
  float4 p; int qi;
  int b = 0;
  if (w < n_work) {
    if (lane == 0) page_load_issue(pages[warp][0], &bars[warp][0], bv.pages + (size_t)it.slot * kPageBytes, min(it.total, (unsigned)kBrickCap));
    load_query(it, &p, &qi);
  }
  unsigned w1 = w < n_work ? claim() : n_work;
  BrickWork it1 = w1 < n_work ? work[w1] : none;

  while (w < n_work) {
    // next item: page into the other buffer, queries into registers; the one after: descriptor
    float4 p1 = make_float4(0.f, 0.f, 0.f, 0.f); int qi1 = -1;
    if (w1 < n_work) {
      if (lane == 0) page_load_issue(pages[warp][b ^ 1], &bars[warp][b ^ 1], bv.pages + (size_t)it1.slot * kPageBytes, min(it1.total, (unsigned)kBrickCap));
      load_query(it1, &p1, &qi1);
    }
    const unsigned w2 = w1 < n_work ? claim() : n_work;
    const BrickWork it2 = w2 < n_work ? work[w2] : none;

    unsigned char* page = pages[warp][b];
    unsigned long long* bar = &bars[warp][b];
    const int lg = lanes_log2(it.qn);
    const int g = 1 << lg, sub = lane & (g - 1);
    const bool active = qi >= 0;
    int rc0 = 0;
    const unsigned long long key = it.key;
    if (active) {
      const int3 c = pos2grid(p.x, p.y, p.z, inv_res);
      const int bx = (int)((key >> 38) & 0x7ffffull) - kCoordBias, by = (int)((key >> 19) & 0x7ffffull) - kCoordBias,
                bz = (int)(key & 0x7ffffull) - kCoordBias;
      const int rx = c.x - bx * kBrickXY + 1, ry = c.y - by * kBrickXY + 1, rz = c.z + kBrickZOff - bz * kBrickZ + 1;   // 1..8, 1..8, 1..4
      rc0 = (rz * kRegXY + ry) * kRegXY + rx;
    }
    KeyTop5 best;
    best.init();
    int found = 0;
    const unsigned levels = it.total ? (it.total + kBrickCap - 1) / kBrickCap : 1u;
    for (unsigned L = 0; L < levels && L <= (unsigned)kMaxLevel; L++) {
      if (L > 0) {   // points 232 L .. of a crowded brick: their page is found by hashing (brick, L); loaded in place
        __syncwarp();                          // every lane is done with the previous page
        long long sl = -1;
        if (lane == 0) {
          sl = brick_find(bv, key | ((unsigned long long)L << 57));
          if (sl >= 0) page_load_issue(page, bar, bv.pages + (size_t)sl * kPageBytes, min(it.total - L * kBrickCap, (unsigned)kBrickCap));
        }
        sl = __shfl_sync(0xffffffffu, sl, 0);
        if (sl < 0) continue;
      }
      page_load_wait(bar, (phase >> b) & 1u);
      phase ^= 1u << b;
      if (active) {
        const unsigned char* head = page + kPageHead;
        const unsigned char* next = page + kPageNext;
        const float4* pts = reinterpret_cast<const float4*>(page + kPagePts);
        // phase 1: heads of this lane's non-empty cells
        int nc = 0;
#pragma unroll 1
        for (int o = sub; o < n_cells; o += g) {
          const unsigned char j = head[rc0 + s_off[o]];
          myq[nc] = j;
          nc += j != 0;
        }
        // phase 2: one stored point per iteration
        int qp = 1;
        unsigned j = nc ? myq[0] : 0u;
        while (j) {
          const float4 a = pts[j - 1];
          const float d2 = dist2(p.x, p.y, p.z, a.x, a.y, a.z);
          if (d2 < max_sq) {
            found++;
            best.insert(((unsigned long long)__float_as_uint(d2) << 32) | ((unsigned)__float_as_int(a.w) ^ 0x80000000u));   // signed id order
          }
          j = next[j - 1];
          if (j == 0u && qp < nc) j = myq[qp++];
        }
      }
    }
    // merge the group's lists: after step s every lane holds the K best of 2^(s+1) lanes' candidates
#pragma unroll 1
    for (int s = 0; s < lg; s++) {
      best.merge_xor(1 << s);
      found += __shfl_xor_sync(0xffffffffu, found, 1 << s);
    }
    if (active) {
      const int nf = min(found, K);
#pragma unroll
      for (int r = 0; r < K; r++) {
        if ((r & (g - 1)) == sub) {                          // the group's lanes share the K stores
          out_idx[(size_t)qi * K + r] = r < nf ? (int)((unsigned)(best.k[r] & 0xffffffffull) ^ 0x80000000u) : -1;
          out_d2[(size_t)qi * K + r] = r < nf ? __uint_as_float((unsigned)(best.k[r] >> 32)) : -1.0f;
        }
      }
      if (sub == 0) out_cnt[qi] = nf;
    }
    __syncwarp();   // this page buffer and the cell queues are free for the item after next
    w = w1; it = it1; p = p1; qi = qi1;
    w1 = w2; it1 = it2;
    b ^= 1;
  }
}

// ------------------------------------------------------------------ box delete on the pages (KD_TREE::Delete_Point_Boxes)
// Same rule as map_delete_boxes_kernel: a deleted point keeps its slot and gets NaN coordinates.  Unused slots hold zeros
// or older points of no list; rewriting them is harmless.
struct BrickBoxes { int n; float b[16][6]; };
__global__ void __launch_bounds__(256) brick_delete_boxes_kernel(BrickView bv, unsigned long long n_slots, BrickBoxes bx) {
  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long s = t / 8;           // 8 threads per page
  if (s >= n_slots || bv.keys[s] == 0ull) return;
  float4* pts = reinterpret_cast<float4*>(bv.pages + (size_t)s * kPageBytes + kPagePts);
  for (int j = (int)(t & 7); j < kBrickCap; j += 8) {
    const float4 p = pts[j];
    bool inside = false;
    for (int b = 0; b < bx.n && !inside; b++)
      inside = bx.b[b][0] <= p.x && bx.b[b][3] > p.x && bx.b[b][1] <= p.y && bx.b[b][4] > p.y && bx.b[b][2] <= p.z && bx.b[b][5] > p.z;
    if (inside) pts[j] = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000), p.w);
  }
}

}  // namespace lsd
