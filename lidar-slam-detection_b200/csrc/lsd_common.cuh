// lsd_common.cuh — shared device/host helpers for liblsdreg (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/lsdreg.h"

namespace lsd {

// SMs of the H100 SXM: persistent and grid-stride launches are sized in multiples of it
constexpr int kNumSms = 132;

// ------------------------------------------------------------------ errors
void set_error(const char* fmt, ...);
lsd_status_t cuda_fail(cudaError_t e, const char* what, const char* file, int line);
lsd_status_t ensure_device();

#define LSD_CUDA(call)                                                        \
  do {                                                                        \
    cudaError_t _e = (call);                                                  \
    if (_e != cudaSuccess) return lsd::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

// ------------------------------------------------------------------ hash-voxel map layout
// One 128-byte line per (voxel, level): header + 7 points.  A query resolves a voxel with ONE
// 32-byte sector read (header + first point) and no pointer chase; sectors 1..3 hold points 1..6.
// Level L > 0 lines hold points 7L .. 7L+6 of voxels with more than 7 points and are found by
// hashing (cell, L) — no linked lists, so inserts never wait on each other.
struct __align__(128) CellLine {
  unsigned long long key;  // packed (level, x, y, z); 0 = empty
  unsigned int count;      // level-0 line: total points in the voxel (all levels)
  unsigned int pad;
  float4 pts[7];           // (x, y, z, id as int bits)
};
static_assert(sizeof(CellLine) == 128, "CellLine must be one 128-byte line");

constexpr int kPtsPerLine = 7;
constexpr int kMaxLevel = 127;
constexpr int kCoordBias = 1 << 18;  // voxel coordinates in (-2^18, 2^18)
constexpr unsigned kMaxProbe = 4096;
// key of a retired line (LRU eviction): never 0 (probe chains run through it), never a voxel's (x + bias = 0 is outside coord_ok)
constexpr unsigned long long kTombKey = 1ull;

// Brick layout of the same points (brick.cuh): directory + one 4608-byte page per slot.  keys == nullptr: not enabled.
struct BrickView {
  unsigned long long* keys;      // [n_slots] level:7 | bx:19 | by:19 | bz:19, 0 = empty
  unsigned* totals;              // [n_slots] points stored in the brick (all levels), level-0 slot only
  unsigned char* pages;          // [n_slots] x kPageBytes
  unsigned long long mask;       // n_slots - 1
  unsigned long long* counters;  // [0] pages in use, [1] point replicas stored, [2] dropped (directory full / > 127 levels)
};

struct MapView {
  CellLine* lines;
  unsigned char* tags;      // one byte per line: 0 = empty, else slot_tag(hash) — the query-side filter (L2-resident)
  unsigned long long mask;  // n_lines - 1
  float res, inv_res;
  unsigned long long* counters;  // [0] cells, [1] points, [2] dropped
  // tile sharding (SURVEY.md §8e): world == 1 -> everything is local
  int shard_rank, shard_world, shard_tile, shard_reach;
  BrickView bricks;              // lsd_map_enable_bricks: every accepted point is also stored brick by brick
};

// Tile ownership: x-y tiles of `tile` voxels, owner = hash(tile) mod world.  A voxel is RELEVANT to a
// rank when any voxel within `reach` (Chebyshev, x-y) of it is owned by that rank: relevant points are
// replicated (halo), so the owner of a query's home voxel holds every point its stencil can touch.
__host__ __device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
__host__ __device__ __forceinline__ int tile_owner(int cx, int cy, int tile, int world) {
  const unsigned tx = (unsigned)floor_div(cx, tile), ty = (unsigned)floor_div(cy, tile);
  unsigned h = tx * 73856093u ^ ty * 19349663u;
  h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
  return (int)(h % (unsigned)world);
}
__host__ __device__ __forceinline__ bool shard_owns(const MapView& mv, int cx, int cy) {
  return mv.shard_world <= 1 || tile_owner(cx, cy, mv.shard_tile, mv.shard_world) == mv.shard_rank;
}
__host__ __device__ __forceinline__ bool shard_relevant(const MapView& mv, int cx, int cy) {
  if (mv.shard_world <= 1) return true;
  const int r = mv.shard_reach;
  return tile_owner(cx - r, cy - r, mv.shard_tile, mv.shard_world) == mv.shard_rank ||
         tile_owner(cx + r, cy - r, mv.shard_tile, mv.shard_world) == mv.shard_rank ||
         tile_owner(cx - r, cy + r, mv.shard_tile, mv.shard_world) == mv.shard_rank ||
         tile_owner(cx + r, cy + r, mv.shard_tile, mv.shard_world) == mv.shard_rank;
}

__host__ __device__ __forceinline__ bool coord_ok(int x, int y, int z) {
  return x > -kCoordBias && x < kCoordBias && y > -kCoordBias && y < kCoordBias && z > -kCoordBias && z < kCoordBias;
}
__host__ __device__ __forceinline__ unsigned long long pack_key(int x, int y, int z, int level) {
  return ((unsigned long long)level << 57) | ((unsigned long long)(x + kCoordBias) << 38) |
         ((unsigned long long)(y + kCoordBias) << 19) | (unsigned long long)(z + kCoordBias);
}
__host__ __device__ __forceinline__ unsigned long long hash_key(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}

// Tag of an occupied line: 1..255 from hash bits the slot index does not use.  Queries read the tag
// array (1 B/line: 32 MB for a 4 GB table, L2-resident) instead of the 128-byte lines to learn that a
// voxel is absent or where its line is, so only voxels that exist cost a DRAM access.
__host__ __device__ __forceinline__ unsigned slot_tag(unsigned long long h) { return (unsigned)(((h >> 56) * 255ull) >> 8) + 1u; }

// Pos2Grid (ivox3d.h:258-261): round-half-away-from-zero of p * inv_res, in fp32
__device__ __forceinline__ int3 pos2grid(float x, float y, float z, float inv_res) {
  return make_int3((int)roundf(x * inv_res), (int)roundf(y * inv_res), (int)roundf(z * inv_res));
}

// distance2 (ivox3d_node.hpp:11-14): (dx*dx + dy*dy) + dz*dz, fp32, no FMA (built with -fmad=false)
__device__ __forceinline__ float dist2(float ax, float ay, float az, float bx, float by, float bz) {
  float dx = bx - ax, dy = by - ay, dz = bz - az;
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ uint4 ldg_u4(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ float4 ldg_f4(const void* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// warp-level double sum
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// NV (9..32) per-lane values -> lane j returns the warp total of vals[j] (lanes >= NV return 0).  A transposed butterfly:
// at offset 16 a lane keeps one half of its values and sends the other half to its partner, then 8, 4, 2, 1 — 31 double
// shuffles and adds instead of NV x 5.  Every total is formed by the SAME pairing tree as warp_sum (partners l, l^16, then
// ^8, ...; IEEE addition is commutative), so the sums are bit-identical to NV calls of warp_sum.
template <int NV>
__device__ __forceinline__ double warp_sum_to_lane(const double (&vals)[NV]) {
  static_assert(NV > 8 && NV <= 32, "use warp_sum for a handful of values");
  const int lane = threadIdx.x & 31;
  double a[16], b[8], c[4], d[2];
  {
    const bool up = lane & 16;
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const double lo = (j < NV) ? vals[j < NV ? j : 0] : 0.0;
      const double hi = (j + 16 < NV) ? vals[j + 16 < NV ? j + 16 : 0] : 0.0;
      a[j] = (up ? hi : lo) + __shfl_xor_sync(0xffffffffu, up ? lo : hi, 16);
    }
  }
  {
    const bool up = lane & 8;
#pragma unroll
    for (int j = 0; j < 8; j++) b[j] = (up ? a[j + 8] : a[j]) + __shfl_xor_sync(0xffffffffu, up ? a[j] : a[j + 8], 8);
  }
  {
    const bool up = lane & 4;
#pragma unroll
    for (int j = 0; j < 4; j++) c[j] = (up ? b[j + 4] : b[j]) + __shfl_xor_sync(0xffffffffu, up ? b[j] : b[j + 4], 4);
  }
  {
    const bool up = lane & 2;
#pragma unroll
    for (int j = 0; j < 2; j++) d[j] = (up ? c[j + 2] : c[j]) + __shfl_xor_sync(0xffffffffu, up ? c[j] : c[j + 2], 2);
  }
  const bool up = lane & 1;
  return (up ? d[1] : d[0]) + __shfl_xor_sync(0xffffffffu, up ? d[0] : d[1], 1);
}

// ------------------------------------------------------------------ programmatic dependent launch (sm_90+)
// A scan is a chain of ~15 short kernels (5-40 us each) on one stream; between two dependent kernels the GPU idles for
// the grid drain plus the next grid's launch latency.  With the programmatic-stream-serialization attribute the next
// kernel's blocks are scheduled as soon as every block of the running one has passed pdl_trigger(), and park in
// pdl_wait() until that grid has completed and its memory is visible.  Every kernel of the chain executes
// pdl_wait() as its FIRST statement, on every thread, before touching global memory: the ordering the stream gave is
// kept link by link (B's completion implies its wait returned, hence A's completion), only the launch latency is hidden.
// Both instructions are no-ops in a kernel launched without the attribute (the default: lsd_lio_set_pdl).
__device__ __forceinline__ void pdl_wait() {
#ifndef LSD_SIMT_EMU
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_trigger() {
#ifndef LSD_SIMT_EMU
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_enter() { pdl_wait(); pdl_trigger(); }

#ifdef LSD_SIMT_EMU
#define LSD_LAUNCH(pdl, kern, g, b, st, ...) kern<<<g, b, 0, st>>>(__VA_ARGS__)
#else
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kern)(KArgs...), dim3 g, dim3 b, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = g; cfg.blockDim = b; cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);  // errors surface through cudaGetLastError, as for a plain launch
}
// Launch on `st`; pdl != 0 adds the programmatic-serialization attribute (the kernel must start with pdl_enter()).
#define LSD_LAUNCH(pdl, kern, g, b, st, ...)                                    \
  do {                                                                          \
    if (pdl) lsd::launch_pdl(kern, dim3(g), dim3(b), st, __VA_ARGS__);          \
    else kern<<<g, b, 0, st>>>(__VA_ARGS__);                                    \
  } while (0)
#endif

// ------------------------------------------------------------------ stencils (ivox3d.h:178-215)
constexpr int kStencilMax = 75;
struct Stencil { int n; signed char off[kStencilMax][3]; };
const Stencil* host_stencil(int type);  // nullptr for EXACT / unknown

}  // namespace lsd
