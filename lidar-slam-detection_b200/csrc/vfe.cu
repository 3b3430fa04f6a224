// vfe.cu — detection front-end voxelizer (config 5): multi-frame accumulate + hash voxelisation + mean
// voxel feature encoder output (fp16), feeding the CenterPoint-VoxelNet sparse 3D-CNN.
//
// Replaces (reference: sensor_driver/inference/voxelize):
//   PreprocessImplement::forward + transform_kernel      preprocess_kernel.cu:6-20,56-101
//   VoxelizationImplement::forward                        voxelization_kernel.cu:225-255
//     build_hash_table_kernel :73-92, voxelization_kernel :107-156, reduce_mean_kernel :158-180
// The reference's result depends on thread arrival order twice: voxel ids come from an atomicAdd
// counter, and a voxel with more than max_points_per_voxel points keeps whichever 5 arrive first.
// Here both follow the SEQUENTIAL order of the same code (ascending point index): voxel ids by first
// point, the 5 lowest-index points per voxel (kept by a chain of atomicMin registers in the claim pass), summed in
// index order — one of the outcomes the reference can produce, and the same one every run.  No 30 MB memset of the voxel scratch
// (:229-232) and no host synchronisation between the passes (:248).
#include <cuda_fp16.h>

#include <climits>

#include "lsd_common.cuh"

namespace lsd {

constexpr unsigned kVfeEmpty = 0xffffffffu;
struct __align__(32) VfeSlot { unsigned key, count, sel[5], vid; };  // sel[r] = r-th smallest point index of the voxel
static_assert(sizeof(VfeSlot) == 32, "VfeSlot must be 32 bytes");

struct VfeGrid { float mn[3], mx[3], vs[3]; int gs[3]; int max_ppv, max_voxels, nf; };

__device__ __forceinline__ unsigned vfe_hash(unsigned k) {  // murmur3 fmix32, voxelization_kernel.cu:29-36
  k ^= k >> 16; k *= 0x85ebca6bu; k ^= k >> 13; k *= 0xc2b2ae35u; k ^= k >> 16;
  return k;
}

// transform_kernel (preprocess_kernel.cu:6-20): older frames re-projected by the 3x4 motion, time + 0.1.
// The reference is compiled with nvcc's default FMA contraction; its SASS for m0*x + m1*y + m2*z + m3 is
// FMUL m1*y; FFMA m0*x + .; FFMA m2*z + .; FADD m3 — spelt out so this build (-fmad=false) produces the same bits
// (pinned against the recompiled reference kernel, tests/test_gpu_ref_cuda.py).  Features past z are carried over and
// the time channel (feature 4) gets + 0.1; the reference copies features 3 and 4 whatever num_feature is.
__global__ void __launch_bounds__(256) vfe_transform_kernel(int n, const float* __restrict__ src, float* __restrict__ dst, int nf,
                                                            const float* __restrict__ m) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float px = src[nf * i], py = src[nf * i + 1], pz = src[nf * i + 2];
  dst[nf * i + 0] = __fadd_rn(__fmaf_rn(m[2], pz, __fmaf_rn(m[0], px, __fmul_rn(m[1], py))), m[3]);
  dst[nf * i + 1] = __fadd_rn(__fmaf_rn(m[6], pz, __fmaf_rn(m[4], px, __fmul_rn(m[5], py))), m[7]);
  dst[nf * i + 2] = __fadd_rn(__fmaf_rn(m[10], pz, __fmaf_rn(m[8], px, __fmul_rn(m[9], py))), m[11]);
  for (int f = 3; f < nf; f++) dst[nf * i + f] = f == 4 ? (float)((double)src[nf * i + 4] + 0.1) : src[nf * i + f];
}

// floor((p - mn) / vs) as an int; NaN gives 0, as the reference's float-to-int conversion on the device does
__device__ __forceinline__ int vfe_cell(float p, float mn, float vs) {
  const float c = floorf((p - mn) / vs);
  return c == c ? (int)c : 0;
}

__device__ __forceinline__ unsigned vfe_voxel_offset(const VfeGrid& g, float px, float py, float pz, int* ix, int* iy, int* iz) {
  if (px < g.mn[0] || px >= g.mx[0] || py < g.mn[1] || py >= g.mx[1] || pz < g.mn[2] || pz >= g.mx[2]) return kVfeEmpty;  // NaN passes
  const int x = vfe_cell(px, g.mn[0], g.vs[0]), y = vfe_cell(py, g.mn[1], g.vs[1]), z = vfe_cell(pz, g.mn[2], g.vs[2]);
  if (x < 0 || x >= g.gs[0] || y < 0 || y >= g.gs[1] || z < 0 || z >= g.gs[2]) return kVfeEmpty;
  *ix = x; *iy = y; *iz = z;
  return (unsigned)((z * g.gs[1] + y) * g.gs[0] + x);
}

// pass 1: claim the voxel's slot, count it, and insert the point index into the voxel's sorted list of the max_ppv
// LOWEST indices.  sel[r] is an atomicMin register; a thread offers its index to sel[0], carries the larger of
// (what was there, what it offered) on to sel[1], and so on.  Whatever the interleaving, the values offered to
// register r are all indices except the r smallest, so it ends holding the (r+1)-th smallest: deterministic, one pass.
// next_vid != nullptr (unordered ids, lsd_vfe_params_t::unordered_ids): the thread that opens a slot also numbers the voxel,
// in atomic order like the reference's voxelization_kernel (voxelization_kernel.cu:119-126) — no scan pass needed.
__global__ void __launch_bounds__(256) vfe_claim_kernel(int n, const float* __restrict__ pts, VfeGrid g, VfeSlot* __restrict__ tab,
                                                        unsigned mask, int* __restrict__ pslot, int* __restrict__ next_vid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x, y, z;
  const unsigned key = vfe_voxel_offset(g, pts[g.nf * i], pts[g.nf * i + 1], pts[g.nf * i + 2], &x, &y, &z);
  int slot = -1;
  if (key != kVfeEmpty) {
    unsigned s = vfe_hash(key) & mask;
    for (unsigned probe = 0; probe <= mask; probe++) {
      const unsigned pre = atomicCAS(&tab[s].key, kVfeEmpty, key);
      if (pre == kVfeEmpty && next_vid) tab[s].vid = (unsigned)atomicAdd(next_vid, 1);
      if (pre == kVfeEmpty || pre == key) { slot = (int)s; break; }
      s = (s + 1) & mask;
    }
    if (slot >= 0) {
      atomicAdd(&tab[slot].count, 1u);
      unsigned x = (unsigned)i;
#pragma unroll
      for (int r = 0; r < 5; r++) {
        if (r >= g.max_ppv) break;
        const unsigned old = atomicMin(&tab[slot].sel[r], x);
        x = max(old, x);
        if (x == kVfeEmpty) break;  // carrying the "empty" sentinel: nothing left to place
      }
    }
  }
  pslot[i] = slot;
}

// voxel ids in order of first point: exclusive scan of "point i opens its voxel" over the points
__global__ void __launch_bounds__(1024) vfe_scan_kernel(int n, const VfeSlot* __restrict__ tab, const int* __restrict__ pslot,
                                                        int* __restrict__ local, int* __restrict__ block_sum,
                                                        unsigned* __restrict__ done, int* __restrict__ total) {
  __shared__ int warp_tot[32];
  __shared__ bool is_last;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int f = 0;
  if (i < n) { const int s = pslot[i]; f = (s >= 0 && tab[s].sel[0] == (unsigned)i) ? 1 : 0; }
  int inc = f;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= o) inc += t; }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
  __syncthreads();
  int woff = 0;
  for (int k = 0; k < (int)(threadIdx.x >> 5); k++) woff += warp_tot[k];
  if (i < n) local[i] = f ? woff + inc - 1 : -1;
  if (threadIdx.x == blockDim.x - 1) block_sum[blockIdx.x] = woff + inc;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < (int)gridDim.x; base += 1024) {
    const int b = base + threadIdx.x;
    const int v = b < (int)gridDim.x ? __ldcg(block_sum + b) : 0;
    int in2 = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, in2, o); if ((threadIdx.x & 31) >= o) in2 += t; }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = in2;
    __syncthreads();
    int w2 = 0;
    for (int k = 0; k < (int)(threadIdx.x >> 5); k++) w2 += warp_tot[k];
    const int c = carry;
    if (b < (int)gridDim.x) block_sum[b] = c + w2 + in2 - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + w2 + in2;
    __syncthreads();
  }
  if (threadIdx.x == 0) { *total = carry; *done = 0u; }
}

// voxelization_kernel + reduce_mean_kernel: the opening point of each voxel (its smallest point index) writes its row and
// returns the slot to its idle state (no separate reset pass: nobody else reads the slot in this kernel).
// ORDERED: voxel id = rank of the opening point among the opening points (vfe_scan_kernel); else the id taken at claim time.
template <bool ZYX, bool ORDERED>
__global__ void __launch_bounds__(256) vfe_emit_kernel(int n, const float* __restrict__ pts, VfeGrid g, VfeSlot* __restrict__ tab,
                                                       const int* __restrict__ pslot, const int* __restrict__ local,
                                                       const int* __restrict__ block_off, __half* __restrict__ feat,
                                                       uint4* __restrict__ idx, unsigned* __restrict__ npts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int sl = pslot[i];
  if (sl < 0) return;
  int vid;
  if (ORDERED) {
    const int l = local[i];
    if (l < 0) return;
    vid = block_off[i >> 10] + l;
  } else {
    if (*reinterpret_cast<volatile unsigned*>(&tab[sl].sel[0]) != (unsigned)i) return;
    vid = -1;
  }
  const VfeSlot s = tab[sl];
  if (!ORDERED) vid = (int)s.vid;
  {  // slot back to idle
    uint4* p = reinterpret_cast<uint4*>(tab + sl);
    p[0] = make_uint4(kVfeEmpty, 0u, kVfeEmpty, kVfeEmpty);
    p[1] = make_uint4(kVfeEmpty, kVfeEmpty, kVfeEmpty, 0u);
  }
  if (vid >= g.max_voxels) return;  // voxelization_kernel.cu:135-137
  const int cnt = (int)min(s.count, (unsigned)g.max_ppv);
  float acc[8];
  for (int f = 0; f < g.nf; f++) acc[f] = pts[g.nf * (size_t)s.sel[0] + f];
  for (int k = 1; k < cnt; k++)
    for (int f = 0; f < g.nf; f++) acc[f] += pts[g.nf * (size_t)s.sel[k] + f];
  for (int f = 0; f < g.nf; f++) feat[(size_t)vid * g.nf + f] = __float2half(acc[f] / (float)cnt);
  int x, y, z;
  vfe_voxel_offset(g, pts[g.nf * i], pts[g.nf * i + 1], pts[g.nf * i + 2], &x, &y, &z);
  idx[vid] = ZYX ? make_uint4(0u, (unsigned)z, (unsigned)y, (unsigned)x) : make_uint4(0u, (unsigned)x, (unsigned)y, (unsigned)z);
  npts[vid] = (unsigned)cnt;
}

}  // namespace lsd

struct lsd_vfe {
  lsd_vfe_params_t p{};
  lsd::VfeGrid grid{};
  int device = 0;
  cudaStream_t stream = nullptr;
  float* pts[2] = {nullptr, nullptr};  // A/B sliding-window buffers (preprocess_kernel.cu:44-49), rows() rows each
  int cur = 0;
  std::vector<int> frame_pts;
  int total = 0;
  float* d_motion = nullptr;
  lsd::VfeSlot* tab = nullptr;
  unsigned mask = 0;
  int *pslot = nullptr, *local = nullptr, *block_sum = nullptr, *d_total = nullptr;
  unsigned* d_done = nullptr;
  __half* feat = nullptr;
  uint4* idx = nullptr;
  unsigned* npts = nullptr;
  int num_voxels = 0;
  long long launches = 0;
  // The window's row bound.  The reference's arithmetic (kept: the totals are its totals) gives an incoming frame at
  // least one row even when the remaining frames already fill max_points, and a frame slot that was never filled pops 0
  // rows, so the total can reach max_points + max_frame_num - 1 (e.g. frames of max_points rows: max_points,
  // max_points + 1, ..., then back to max_points once a full frame leaves).
  size_t rows() const { return (size_t)p.max_points + (size_t)p.max_frame_num - 1; }
};

using namespace lsd;

extern "C" {

void lsd_vfe_default_params(lsd_vfe_params_t* p) {
  if (!p) return;
  // sensor_inference/cfgs/detection_object.yaml:7-16, sensor_driver/inference/inference.h:16-38
  const float mn[3] = {-64.f, -64.f, -2.f}, mx[3] = {64.f, 64.f, 4.f}, vs[3] = {0.1f, 0.1f, 0.15f};
  for (int i = 0; i < 3; i++) { p->min_range[i] = mn[i]; p->max_range[i] = mx[i]; p->voxel_size[i] = vs[i]; }
  p->max_points_per_voxel = 5; p->max_voxels = 300000; p->max_points = 500000; p->num_feature = 5; p->max_frame_num = 2; p->unordered_ids = 0;
}

lsd_status_t lsd_vfe_create(lsd_vfe_t** out, const lsd_vfe_params_t* p) {
  if (!out || !p || p->num_feature < 4 || p->num_feature > 8 || p->max_points_per_voxel < 1 || p->max_points_per_voxel > 5 ||
      p->max_points < 1 || p->max_voxels < 1 || p->max_frame_num < 1 || (long long)p->max_points + p->max_frame_num - 1 > INT_MAX) {
    set_error("lsd_vfe_create: bad params"); return LSD_ERR_INVALID;
  }
  int gs[3];
  for (int i = 0; i < 3; i++) gs[i] = (int)std::round((p->max_range[i] - p->min_range[i]) / p->voxel_size[i]);  // compute_grid_size, :182-189
  if ((long long)gs[0] * gs[1] * gs[2] >= (1ll << 31)) {  // voxel keys (z * gs1 + y) * gs0 + x are 32-bit ints
    set_error("lsd_vfe_create: grid of 2^31 cells or more"); return LSD_ERR_INVALID;
  }
  lsd_status_t s = ensure_device();
  if (s) return s;
  lsd_vfe* v = new lsd_vfe();
  v->p = *p;
  cudaGetDevice(&v->device);
  for (int i = 0; i < 3; i++) {
    v->grid.mn[i] = p->min_range[i]; v->grid.mx[i] = p->max_range[i]; v->grid.vs[i] = p->voxel_size[i];
    v->grid.gs[i] = gs[i];
  }
  v->grid.max_ppv = p->max_points_per_voxel; v->grid.max_voxels = p->max_voxels; v->grid.nf = p->num_feature;
  v->frame_pts.assign(p->max_frame_num, 0);
  const size_t N = v->rows();
  size_t cap = 1024;
  while (cap < N * 2) cap <<= 1;
  v->mask = (unsigned)(cap - 1);
  cudaError_t e = cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking);
  auto A = [&](void** ptr, size_t b) { if (e == cudaSuccess) e = cudaMalloc(ptr, b); if (e == cudaSuccess) e = cudaMemset(*ptr, 0, b); };
  A((void**)&v->pts[0], N * p->num_feature * 4);
  A((void**)&v->pts[1], N * p->num_feature * 4);
  A((void**)&v->d_motion, 64);
  A((void**)&v->tab, cap * sizeof(VfeSlot));
  A((void**)&v->pslot, N * 4);
  A((void**)&v->local, N * 4);
  A((void**)&v->block_sum, (N / 1024 + 2) * 4);
  A((void**)&v->d_total, 64);
  A((void**)&v->d_done, 64);
  A((void**)&v->feat, (size_t)p->max_voxels * p->num_feature * 2);
  A((void**)&v->idx, (size_t)p->max_voxels * 16);
  A((void**)&v->npts, (size_t)p->max_voxels * 4);
  if (e == cudaSuccess) {  // idle state of a slot: key empty, count 0, sel = +inf
    std::vector<unsigned> init(cap * 8);
    for (size_t i = 0; i < cap; i++) { unsigned* q = &init[i * 8]; q[0] = kVfeEmpty; q[1] = 0; for (int k = 2; k < 7; k++) q[k] = kVfeEmpty; q[7] = 0; }
    e = cudaMemcpy(v->tab, init.data(), init.size() * 4, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) { lsd_status_t r = cuda_fail(e, "lsd_vfe_create", __FILE__, __LINE__); lsd_vfe_destroy(v); return r; }
  *out = v;
  return LSD_OK;
}

lsd_status_t lsd_vfe_destroy(lsd_vfe_t* v) {
  if (!v) return LSD_OK;
  cudaSetDevice(v->device);
  if (v->stream) cudaStreamSynchronize(v->stream);
  void* ptrs[] = {v->pts[0], v->pts[1], v->d_motion, v->tab, v->pslot, v->local, v->block_sum, v->d_total, v->d_done, v->feat, v->idx, v->npts};
  for (void* q : ptrs) cudaFree(q);
  if (v->stream) cudaStreamDestroy(v->stream);
  delete v;
  return LSD_OK;
}

// PreprocessImplement::forward (preprocess_kernel.cu:56-101)
lsd_status_t lsd_vfe_accumulate(lsd_vfe_t* v, const float* points_host, int num_points, const float* motion16_host, int realtime,
                                int* total_points) {
  if (!v || (!points_host && num_points > 0) || num_points < 0 || (realtime && !motion16_host)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(v->device));
  cudaStream_t st = v->stream;
  const int nf = v->p.num_feature;
  // the one row the reference counts for an empty realtime frame (and copies from the caller's empty array): far out,
  // finite, outside every range box after any rigid motion
  float far_row[8] = {1e30f, 1e30f, 1e30f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (realtime && num_points == 0) points_host = far_row;
  if (realtime) {
    LSD_CUDA(cudaMemcpyAsync(v->d_motion, motion16_host, 64, cudaMemcpyHostToDevice, st));
    v->total -= v->frame_pts.back();
    num_points = std::min(num_points, v->p.max_points - v->total);
    num_points = std::max(num_points, 1);
    for (size_t i = v->frame_pts.size() - 1; i >= 1; i--) v->frame_pts[i] = v->frame_pts[i - 1];
    const float* src = v->pts[v->cur];
    v->cur ^= 1;
    float* dst = v->pts[v->cur];
    if (v->total > 0) {
      vfe_transform_kernel<<<(v->total + 255) / 256, 256, 0, st>>>(v->total, src, dst + (size_t)num_points * nf, nf, v->d_motion);
      LSD_CUDA(cudaGetLastError());
      v->launches++;
    }
  } else {
    v->frame_pts.assign(v->p.max_frame_num, 0);
    v->total = 0;
    v->cur = 0;
    num_points = std::min(num_points, v->p.max_points);
  }
  v->frame_pts[0] = num_points;
  v->total += num_points;
  if (num_points > 0) LSD_CUDA(cudaMemcpyAsync(v->pts[v->cur], points_host, (size_t)num_points * nf * 4, cudaMemcpyHostToDevice, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  if (total_points) *total_points = v->total;
  return LSD_OK;
}

// VoxelizationImplement::forward (voxelization_kernel.cu:225-255) on the accumulated window
lsd_status_t lsd_vfe_voxelize(lsd_vfe_t* v, int order_zyx, int* num_voxels) {
  if (!v) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(v->device));
  cudaStream_t st = v->stream;
  const int n = v->total;
  v->num_voxels = 0;
  if (n > 0) {
    const float* pts = v->pts[v->cur];
    const int nb = (n + 255) / 256;
    if (v->p.unordered_ids) {   // the reference's contract: voxel ids in atomic order — two kernels
      LSD_CUDA(cudaMemsetAsync(v->d_total, 0, 4, st));
      vfe_claim_kernel<<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->mask, v->pslot, v->d_total);
      if (order_zyx) vfe_emit_kernel<true, false><<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->pslot, v->local, v->block_sum, v->feat, v->idx, v->npts);
      else vfe_emit_kernel<false, false><<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->pslot, v->local, v->block_sum, v->feat, v->idx, v->npts);
      v->launches += 2;
    } else {                    // deterministic ids (order of first point): + the scan
      vfe_claim_kernel<<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->mask, v->pslot, nullptr);
      vfe_scan_kernel<<<(n + 1023) / 1024, 1024, 0, st>>>(n, v->tab, v->pslot, v->local, v->block_sum, v->d_done, v->d_total);
      if (order_zyx) vfe_emit_kernel<true, true><<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->pslot, v->local, v->block_sum, v->feat, v->idx, v->npts);
      else vfe_emit_kernel<false, true><<<nb, 256, 0, st>>>(n, pts, v->grid, v->tab, v->pslot, v->local, v->block_sum, v->feat, v->idx, v->npts);
      v->launches += 3;
    }
    LSD_CUDA(cudaGetLastError());
    int h = 0;
    LSD_CUDA(cudaMemcpyAsync(&h, v->d_total, 4, cudaMemcpyDeviceToHost, st));
    LSD_CUDA(cudaStreamSynchronize(st));
    v->num_voxels = std::min(h, v->p.max_voxels);
  }
  if (num_voxels) *num_voxels = v->num_voxels;
  return LSD_OK;
}

// Voxelization::get_output: device pointers for the engine, or host copies.
lsd_status_t lsd_vfe_get_output_dev(lsd_vfe_t* v, const void** features_fp16, const unsigned** indices, const unsigned** num_points) {
  if (!v) return LSD_ERR_INVALID;
  if (features_fp16) *features_fp16 = v->feat;
  if (indices) *indices = reinterpret_cast<const unsigned*>(v->idx);
  if (num_points) *num_points = v->npts;
  return LSD_OK;
}
lsd_status_t lsd_vfe_get_output(lsd_vfe_t* v, void* features_fp16_host, unsigned* indices_host, unsigned* num_points_host) {
  if (!v) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(v->device));
  const size_t V = (size_t)v->num_voxels;
  if (V == 0) return LSD_OK;
  if (features_fp16_host) LSD_CUDA(cudaMemcpyAsync(features_fp16_host, v->feat, V * v->p.num_feature * 2, cudaMemcpyDeviceToHost, v->stream));
  if (indices_host) LSD_CUDA(cudaMemcpyAsync(indices_host, v->idx, V * 16, cudaMemcpyDeviceToHost, v->stream));
  if (num_points_host) LSD_CUDA(cudaMemcpyAsync(num_points_host, v->npts, V * 4, cudaMemcpyDeviceToHost, v->stream));
  LSD_CUDA(cudaStreamSynchronize(v->stream));
  return LSD_OK;
}
lsd_status_t lsd_vfe_get_points(lsd_vfe_t* v, float* points_host, int cap, int* total) {
  if (!v) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(v->device));
  if (total) *total = v->total;
  const int c = std::min(cap, v->total);
  if (points_host && c > 0) LSD_CUDA(cudaMemcpy(points_host, v->pts[v->cur], (size_t)c * v->p.num_feature * 4, cudaMemcpyDeviceToHost));
  return LSD_OK;
}

}  // extern "C"
