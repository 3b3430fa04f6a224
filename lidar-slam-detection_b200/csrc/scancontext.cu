// scancontext.cu — ScanContext descriptor, database and candidate retrieval on the device (row N4 of SURVEY.md 8f).
//
// Replaces (reference: slam/common/Scancontext/Scancontext.cpp, call sites slam/common/keyframe.cpp:165-167,
// slam/localization/src/global_localization.cpp:104-118,365-398,439, slam/localization/include/global_alignment.hpp:206-237):
//   SCManager::makeScancontext(cloud, dx, dy)            -> sc_bin_kernel + sc_finish_kernel (all search_trans offsets of one
//                                                          cloud in ONE pass: blockIdx.y = offset)
//   makeRingkey / makeSectorkeyFromScancontext           -> sc_finish_kernel / sc_keys_kernel
//   buildRingKeyKDTree + nanoflann findNeighbors (k=10)  -> sc_ring_knn_kernel (exact brute force over the float ring keys)
//   distanceBtnScanContext (fastAlignUsingVkey + 7 x distDirectSC) -> sc_pair_kernel (one warp per (query, candidate))
//   detectClosestMatch / detectCandidateMatch            -> lsd_sc_query + a few host lines
// The arithmetic lives in sc_math.h (shared with the CPU pin, tests/sc_host_harness.cpp).  Everything is double / float
// exactly where the reference is; the descriptor is bit-exact (a max is order independent), keys and distances follow
// Eigen's reduction order.  The database stays in HBM: 1200 doubles + keys per key frame (10.6 KB; 100 k key frames ~ 1 GB).
#include <vector>

#include "lsd_common.cuh"
#include "sc_math.h"

namespace lsd {

using namespace sc;

constexpr int kScMaxQueries = 64;   // descriptors made / queried per call (the reference uses 9 offsets)
constexpr int kScBinBlock = 256;

struct ScSet {             // a set of descriptors with their keys, device resident
  double* desc = nullptr;    // [cap][1200] column-major
  double* ringkey = nullptr; // [cap][20]
  float* ringkey_f = nullptr;  // [cap][20]  eig2stdvec(ringkey)
  double* vkey = nullptr;    // [cap][60] sector key
  double* norm = nullptr;    // [cap][60] column norms
  int cap = 0;
};

}  // namespace lsd

struct lsd_sc {
  int device = 0;
  cudaStream_t stream = nullptr;
  lsd::ScSet db, q;
  int db_n = 0, q_n = 0;
  int* d_enc = nullptr;      // [kScMaxQueries][1200] encoded max heights
  double* d_off = nullptr;   // [kScMaxQueries][2]
  float4* d_cloud = nullptr; int cloud_cap = 0;
  float* d_d2 = nullptr;     // [kScMaxQueries][db.cap] ring-key distances (scratch)
  int* d_cand = nullptr;     // [kScMaxQueries][10] candidate index (-1 padded)
  int* d_ncand = nullptr;    // [kScMaxQueries]
  double* d_dist = nullptr;  // [kScMaxQueries * 10]
  int* d_shift = nullptr;    // [kScMaxQueries * 10]
  lsd::ScSet pa, pb;         // scratch for lsd_sc_distance: two sets of kScMaxQueries descriptors
  long long launches = 0;
};

namespace lsd {

__global__ void sc_fill_kernel(int* __restrict__ enc, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) enc[i] = enc_z(kNoPoint);
}

// makeScancontext, the per-point loop: block-local maxima in shared memory, then one atomicMax per touched bin.
__global__ void __launch_bounds__(kScBinBlock) sc_bin_kernel(const float4* __restrict__ pts, int n, const double* __restrict__ off,
                                                            int* __restrict__ enc) {
  __shared__ int s_enc[kDesc];
  const int init = enc_z(kNoPoint);
  for (int i = threadIdx.x; i < kDesc; i += blockDim.x) s_enc[i] = init;
  __syncthreads();
  const double dx = off[2 * blockIdx.y], dy = off[2 * blockIdx.y + 1];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(pts + i);
    int bin; float z;
    if (point_bin(p.x, p.y, p.z, dx, dy, &bin, &z)) atomicMax(&s_enc[bin], enc_z(z));
  }
  __syncthreads();
  int* g = enc + (size_t)blockIdx.y * kDesc;
  for (int i = threadIdx.x; i < kDesc; i += blockDim.x)
    if (s_enc[i] > init) atomicMax(&g[i], s_enc[i]);
}

// keys of descriptor set entries [first, first + gridDim.x): ring key (double + float), sector key, column norms
__device__ __forceinline__ void sc_keys_block(const double* d, double* ringkey, float* ringkey_f, double* vkey, double* norm) {
  for (int t = threadIdx.x; t < kRing + 2 * kSector; t += blockDim.x) {
    if (t < kRing) { const double m = ring_mean(d, t); ringkey[t] = m; ringkey_f[t] = (float)m; }
    else if (t < kRing + kSector) vkey[t - kRing] = sector_mean(d, t - kRing);
    else norm[t - kRing - kSector] = sector_norm(d, t - kRing - kSector);
  }
}
__global__ void __launch_bounds__(128) sc_keys_kernel(ScSet s, int first) {
  const int e = first + blockIdx.x;
  sc_keys_block(s.desc + (size_t)e * kDesc, s.ringkey + (size_t)e * kRing, s.ringkey_f + (size_t)e * kRing, s.vkey + (size_t)e * kSector,
                s.norm + (size_t)e * kSector);
}
// "reset no points to zero" (Scancontext.cpp:195-199) + keys; one block per offset
__global__ void __launch_bounds__(128) sc_finish_kernel(const int* __restrict__ enc, ScSet s) {
  const int e = blockIdx.x;
  double* d = s.desc + (size_t)e * kDesc;
  for (int i = threadIdx.x; i < kDesc; i += blockDim.x) {
    const float z = dec_z(enc[(size_t)e * kDesc + i]);
    d[i] = z == kNoPoint ? 0.0 : (double)z;
  }
  __syncthreads();
  sc_keys_block(d, s.ringkey + (size_t)e * kRing, s.ringkey_f + (size_t)e * kRing, s.vkey + (size_t)e * kSector, s.norm + (size_t)e * kSector);
}

// The 10 database entries nearest to each query's ring key, ascending (d2, index).  One block per query: every thread
// evaluates a strided share of the database into the scratch row, then ten rounds of block-wide argmin.
constexpr int kScKnnBlock = 256;
__global__ void __launch_bounds__(kScKnnBlock) sc_ring_knn_kernel(ScSet db, int db_n, ScSet q, float* __restrict__ d2_scratch, int d2_stride,
                                                                 int* __restrict__ cand, int* __restrict__ n_cand) {
  __shared__ float s_key[kRing];
  __shared__ float s_bd[kScKnnBlock / 32];
  __shared__ int s_bi[kScKnnBlock / 32];
  const int qi = blockIdx.x;
  if (threadIdx.x < kRing) s_key[threadIdx.x] = q.ringkey_f[(size_t)qi * kRing + threadIdx.x];
  __syncthreads();
  float* row = d2_scratch + (size_t)qi * d2_stride;
  for (int i = threadIdx.x; i < db_n; i += blockDim.x) row[i] = ring_d2(s_key, db.ringkey_f + (size_t)i * kRing);
  __syncthreads();
  const int k = min(kCand, db_n);
  for (int r = 0; r < kCand; r++) {
    if (r >= k) { if (threadIdx.x == 0) cand[qi * kCand + r] = -1; continue; }
    float bd = 3.0e38f; int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < db_n; i += blockDim.x) {
      const float d = row[i];
      if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; }   // taken entries hold +inf; NaN keys never win
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, bd, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_bd[threadIdx.x >> 5] = bd; s_bi[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kScKnnBlock / 32; w++)
        if (s_bd[w] < bd || (s_bd[w] == bd && s_bi[w] < bi)) { bd = s_bd[w]; bi = s_bi[w]; }
      const int win = bi == 0x7fffffff ? -1 : bi;
      cand[qi * kCand + r] = win;
      if (win >= 0) row[win] = __int_as_float(0x7f800000);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int c = 0;
    for (int r = 0; r < kCand; r++) c += cand[qi * kCand + r] >= 0;
    n_cand[qi] = c;
  }
}

// distanceBtnScanContext for one (a, b) pair per warp.  pair p compares a-set entry ia[p] with b-set entry ib[p]
// (ib < 0: no candidate -> dist = kBig, shift 0).
constexpr int kScPairWarps = 4;
__global__ void __launch_bounds__(kScPairWarps * 32) sc_pair_kernel(ScSet A, ScSet B, const int* __restrict__ ia_or_null, int a_div,
                                                                   const int* __restrict__ ib_or_null, int n_pairs,
                                                                   double* __restrict__ dist_out, int* __restrict__ shift_out) {
  __shared__ double s_sim[kScPairWarps][kSector];
  __shared__ unsigned char s_ok[kScPairWarps][kSector];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = blockIdx.x * kScPairWarps + warp;
  if (p >= n_pairs) return;
  const int ia = ia_or_null ? ia_or_null[p] : p / a_div;
  const int ib = ib_or_null ? ib_or_null[p] : p;
  if (ib < 0) { if (lane == 0) { dist_out[p] = kBig; shift_out[p] = 0; } return; }
  const double* a = A.desc + (size_t)ia * kDesc; const double* an = A.norm + (size_t)ia * kSector; const double* avk = A.vkey + (size_t)ia * kSector;
  const double* b = B.desc + (size_t)ib * kDesc; const double* bn = B.norm + (size_t)ib * kSector; const double* bvk = B.vkey + (size_t)ib * kSector;
  // 1. fastAlignUsingVkey: argmin over 60 shifts, the first minimum wins (strict <)
  double bd = vkey_diff_norm(avk, bvk, lane);
  int bs = lane;
  if (lane + 32 < kSector) {
    const double d = vkey_diff_norm(avk, bvk, lane + 32);
    if (d < bd) { bd = d; bs = lane + 32; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, bd, o); const int os = __shfl_xor_sync(0xffffffffu, bs, o);
    if (od < bd || (od == bd && os < bs)) { bd = od; bs = os; }
  }
  // 2. the 7 shifts around it, ascending; distDirectSC for each
  int space[2 * kSearchRadius + 1];
  search_space(bs, space);
  double best = kBig; int arg = 0;
  for (int t = 0; t < 2 * kSearchRadius + 1; t++) {
    const int shift = space[t];
    for (int j = lane; j < kSector; j += 32) {
      double sim = 0.0;
      const bool ok = sector_similarity(a, an, b, bn, j, shift, &sim);
      s_sim[warp][j] = sim; s_ok[warp][j] = ok ? 1 : 0;
    }
    __syncwarp();
    if (lane == 0) {
      double sum = 0.0; int num = 0;
      for (int j = 0; j < kSector; j++) if (s_ok[warp][j]) { sum = sum + s_sim[warp][j]; num = num + 1; }
      const double d = 1.0 - sum / (double)num;   // 0 / 0 = NaN when no sector counts: never below `best`
      if (d < best) { best = d; arg = shift; }
    }
    __syncwarp();
  }
  if (lane == 0) { dist_out[p] = best; shift_out[p] = arg; }
}

static lsd_status_t set_alloc(ScSet* s, int cap) {
  s->cap = cap;
  LSD_CUDA(cudaMalloc((void**)&s->desc, (size_t)cap * kDesc * 8));
  LSD_CUDA(cudaMalloc((void**)&s->ringkey, (size_t)cap * kRing * 8));
  LSD_CUDA(cudaMalloc((void**)&s->ringkey_f, (size_t)cap * kRing * 4));
  LSD_CUDA(cudaMalloc((void**)&s->vkey, (size_t)cap * kSector * 8));
  LSD_CUDA(cudaMalloc((void**)&s->norm, (size_t)cap * kSector * 8));
  return LSD_OK;
}
static void set_free(ScSet* s) {
  cudaFree(s->desc); cudaFree(s->ringkey); cudaFree(s->ringkey_f); cudaFree(s->vkey); cudaFree(s->norm);
  *s = ScSet();
}

// descriptors of the cloud at d_pts for n_off offsets -> the query set
static lsd_status_t sc_make_dev(lsd_sc* s, const float4* d_pts, int n, const double* offsets_xy, int n_off) {
  cudaStream_t st = s->stream;
  LSD_CUDA(cudaMemcpyAsync(s->d_off, offsets_xy, (size_t)n_off * 16, cudaMemcpyHostToDevice, st));
  sc_fill_kernel<<<(n_off * kDesc + 255) / 256, 256, 0, st>>>(s->d_enc, n_off * kDesc);
  if (n > 0) {
    const int nb = std::max(1, std::min((n + kScBinBlock * 4 - 1) / (kScBinBlock * 4), lsd::kNumSms));
    sc_bin_kernel<<<dim3(nb, n_off), kScBinBlock, 0, st>>>(d_pts, n, s->d_off, s->d_enc);
    s->launches++;
  }
  sc_finish_kernel<<<n_off, 128, 0, st>>>(s->d_enc, s->q);
  s->launches += 2;
  LSD_CUDA(cudaGetLastError());
  s->q_n = n_off;
  return LSD_OK;
}

static lsd_status_t copy_out_set(lsd_sc* s, const ScSet& set, int n, double* desc_out, double* ringkey_out, double* sectorkey_out) {
  cudaStream_t st = s->stream;
  if (desc_out) LSD_CUDA(cudaMemcpyAsync(desc_out, set.desc, (size_t)n * kDesc * 8, cudaMemcpyDeviceToHost, st));
  if (ringkey_out) LSD_CUDA(cudaMemcpyAsync(ringkey_out, set.ringkey, (size_t)n * kRing * 8, cudaMemcpyDeviceToHost, st));
  if (sectorkey_out) LSD_CUDA(cudaMemcpyAsync(sectorkey_out, set.vkey, (size_t)n * kSector * 8, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  return LSD_OK;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

lsd_status_t lsd_sc_destroy(lsd_sc_t* s);
static lsd_status_t sc_alloc_all(lsd_sc* s, int db_capacity) {
  lsd_status_t e;
  LSD_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
  if ((e = set_alloc(&s->db, db_capacity)) || (e = set_alloc(&s->q, kScMaxQueries)) || (e = set_alloc(&s->pa, kScMaxQueries)) ||
      (e = set_alloc(&s->pb, kScMaxQueries)))
    return e;
  LSD_CUDA(cudaMalloc((void**)&s->d_enc, (size_t)kScMaxQueries * kDesc * 4));
  LSD_CUDA(cudaMalloc((void**)&s->d_off, (size_t)kScMaxQueries * 16));
  LSD_CUDA(cudaMalloc((void**)&s->d_d2, (size_t)kScMaxQueries * db_capacity * 4));
  LSD_CUDA(cudaMalloc((void**)&s->d_cand, (size_t)kScMaxQueries * kCand * 4));
  LSD_CUDA(cudaMalloc((void**)&s->d_ncand, (size_t)kScMaxQueries * 4));
  LSD_CUDA(cudaMalloc((void**)&s->d_dist, (size_t)kScMaxQueries * kCand * 8));
  LSD_CUDA(cudaMalloc((void**)&s->d_shift, (size_t)kScMaxQueries * kCand * 4));
  return LSD_OK;
}

lsd_status_t lsd_sc_create(lsd_sc_t** out, int db_capacity) {
  if (!out || db_capacity < 1) return LSD_ERR_INVALID;
  *out = nullptr;
  lsd_status_t e = ensure_device();
  if (e) return e;
  lsd_sc* s = new lsd_sc();
  cudaGetDevice(&s->device);
  e = sc_alloc_all(s, db_capacity);
  if (e) { lsd_sc_destroy(s); return e; }
  *out = s;
  return LSD_OK;
}

lsd_status_t lsd_sc_destroy(lsd_sc_t* s) {
  if (!s) return LSD_OK;
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  set_free(&s->db); set_free(&s->q); set_free(&s->pa); set_free(&s->pb);
  cudaFree(s->d_enc); cudaFree(s->d_off); cudaFree(s->d_cloud); cudaFree(s->d_d2); cudaFree(s->d_cand); cudaFree(s->d_ncand);
  cudaFree(s->d_dist); cudaFree(s->d_shift);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
  return LSD_OK;
}

lsd_status_t lsd_sc_make_dev(lsd_sc_t* s, const float* xyzi_dev, int n, const double* offsets_xy, int n_off, double* desc_out,
                             double* ringkey_out, double* sectorkey_out) {
  static const double zero2[2] = {0.0, 0.0};
  if (!s || n < 0 || (n > 0 && !xyzi_dev) || n_off < 0 || n_off > kScMaxQueries) return LSD_ERR_INVALID;
  if (!offsets_xy) { offsets_xy = zero2; n_off = 1; }
  if (n_off == 0) return LSD_ERR_INVALID;
  cudaSetDevice(s->device);
  lsd_status_t e = sc_make_dev(s, reinterpret_cast<const float4*>(xyzi_dev), n, offsets_xy, n_off);
  if (e) return e;
  return copy_out_set(s, s->q, n_off, desc_out, ringkey_out, sectorkey_out);
}

lsd_status_t lsd_sc_make(lsd_sc_t* s, const float* xyzi_host, int n, const double* offsets_xy, int n_off, double* desc_out,
                         double* ringkey_out, double* sectorkey_out) {
  if (!s || n < 0 || (n > 0 && !xyzi_host)) return LSD_ERR_INVALID;
  cudaSetDevice(s->device);
  if (n > s->cloud_cap) {
    cudaFree(s->d_cloud); s->d_cloud = nullptr; s->cloud_cap = 0;
    LSD_CUDA(cudaMalloc((void**)&s->d_cloud, (size_t)n * 16));
    s->cloud_cap = n;
  }
  if (n > 0) LSD_CUDA(cudaMemcpyAsync(s->d_cloud, xyzi_host, (size_t)n * 16, cudaMemcpyHostToDevice, s->stream));
  return lsd_sc_make_dev(s, reinterpret_cast<const float*>(s->d_cloud), n, offsets_xy, n_off, desc_out, ringkey_out, sectorkey_out);
}

lsd_status_t lsd_sc_db_clear(lsd_sc_t* s) {
  if (!s) return LSD_ERR_INVALID;
  s->db_n = 0;
  return LSD_OK;
}

lsd_status_t lsd_sc_db_size(lsd_sc_t* s, int* n) {
  if (!s || !n) return LSD_ERR_INVALID;
  *n = s->db_n;
  return LSD_OK;
}

lsd_status_t lsd_sc_db_add(lsd_sc_t* s, const double* desc_host, int n) {
  if (!s || n < 0 || (n > 0 && !desc_host)) return LSD_ERR_INVALID;
  if (n == 0) return LSD_OK;
  if (s->db_n + n > s->db.cap) { set_error("lsd_sc_db_add: %d + %d descriptors exceed the capacity %d", s->db_n, n, s->db.cap); return LSD_ERR_CAPACITY; }
  cudaSetDevice(s->device);
  LSD_CUDA(cudaMemcpyAsync(s->db.desc + (size_t)s->db_n * kDesc, desc_host, (size_t)n * kDesc * 8, cudaMemcpyHostToDevice, s->stream));
  sc_keys_kernel<<<n, 128, 0, s->stream>>>(s->db, s->db_n);
  LSD_CUDA(cudaGetLastError());
  LSD_CUDA(cudaStreamSynchronize(s->stream));   // desc_host may be pageable and reused by the caller
  s->launches++;
  s->db_n += n;
  return LSD_OK;
}

lsd_status_t lsd_sc_db_add_made(lsd_sc_t* s, int slot) {
  if (!s || slot < 0 || slot >= s->q_n) return LSD_ERR_INVALID;
  if (s->db_n + 1 > s->db.cap) { set_error("lsd_sc_db_add_made: capacity %d reached", s->db.cap); return LSD_ERR_CAPACITY; }
  cudaSetDevice(s->device);
  cudaStream_t st = s->stream;
  const size_t e = (size_t)s->db_n, q = (size_t)slot;
  LSD_CUDA(cudaMemcpyAsync(s->db.desc + e * kDesc, s->q.desc + q * kDesc, kDesc * 8, cudaMemcpyDeviceToDevice, st));
  LSD_CUDA(cudaMemcpyAsync(s->db.ringkey + e * kRing, s->q.ringkey + q * kRing, kRing * 8, cudaMemcpyDeviceToDevice, st));
  LSD_CUDA(cudaMemcpyAsync(s->db.ringkey_f + e * kRing, s->q.ringkey_f + q * kRing, kRing * 4, cudaMemcpyDeviceToDevice, st));
  LSD_CUDA(cudaMemcpyAsync(s->db.vkey + e * kSector, s->q.vkey + q * kSector, kSector * 8, cudaMemcpyDeviceToDevice, st));
  LSD_CUDA(cudaMemcpyAsync(s->db.norm + e * kSector, s->q.norm + q * kSector, kSector * 8, cudaMemcpyDeviceToDevice, st));
  s->db_n++;
  return LSD_OK;
}

lsd_status_t lsd_sc_query(lsd_sc_t* s, const double* desc_host_or_null, int nq, int32_t* cand_idx, double* cand_dist, int32_t* cand_shift,
                          int32_t* n_cand) {
  if (!s || nq < 1 || nq > kScMaxQueries || !cand_idx || !cand_dist || !cand_shift || !n_cand) return LSD_ERR_INVALID;
  if (!desc_host_or_null && nq > s->q_n) { set_error("lsd_sc_query: %d queries asked, the last lsd_sc_make made %d", nq, s->q_n); return LSD_ERR_INVALID; }
  cudaSetDevice(s->device);
  cudaStream_t st = s->stream;
  if (desc_host_or_null) {
    LSD_CUDA(cudaMemcpyAsync(s->q.desc, desc_host_or_null, (size_t)nq * kDesc * 8, cudaMemcpyHostToDevice, st));
    sc_keys_kernel<<<nq, 128, 0, st>>>(s->q, 0);
    s->launches++;
    s->q_n = nq;
  }
  if (s->db_n == 0) {   // `if (polarcontexts_.size() <= 0) return` (Scancontext.cpp:270-273,335-337)
    LSD_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < nq; i++) n_cand[i] = 0;
    for (int i = 0; i < nq * kCand; i++) { cand_idx[i] = -1; cand_dist[i] = kBig; cand_shift[i] = 0; }
    return LSD_OK;
  }
  sc_ring_knn_kernel<<<nq, kScKnnBlock, 0, st>>>(s->db, s->db_n, s->q, s->d_d2, s->db.cap, s->d_cand, s->d_ncand);
  const int n_pairs = nq * kCand;
  sc_pair_kernel<<<(n_pairs + kScPairWarps - 1) / kScPairWarps, kScPairWarps * 32, 0, st>>>(s->q, s->db, nullptr, kCand, s->d_cand, n_pairs,
                                                                                            s->d_dist, s->d_shift);
  s->launches += 2;
  LSD_CUDA(cudaGetLastError());
  LSD_CUDA(cudaMemcpyAsync(cand_idx, s->d_cand, (size_t)n_pairs * 4, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaMemcpyAsync(cand_dist, s->d_dist, (size_t)n_pairs * 8, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaMemcpyAsync(cand_shift, s->d_shift, (size_t)n_pairs * 4, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaMemcpyAsync(n_cand, s->d_ncand, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  return LSD_OK;
}

lsd_status_t lsd_sc_distance(lsd_sc_t* s, const double* desc_a_host, const double* desc_b_host, int n_pairs, double* dist, int32_t* shift) {
  if (!s || n_pairs < 0 || (n_pairs > 0 && (!desc_a_host || !desc_b_host || !dist || !shift))) return LSD_ERR_INVALID;
  cudaSetDevice(s->device);
  cudaStream_t st = s->stream;
  for (int p0 = 0; p0 < n_pairs; p0 += kScMaxQueries) {
    const int m = std::min(kScMaxQueries, n_pairs - p0);
    LSD_CUDA(cudaMemcpyAsync(s->pa.desc, desc_a_host + (size_t)p0 * kDesc, (size_t)m * kDesc * 8, cudaMemcpyHostToDevice, st));
    LSD_CUDA(cudaMemcpyAsync(s->pb.desc, desc_b_host + (size_t)p0 * kDesc, (size_t)m * kDesc * 8, cudaMemcpyHostToDevice, st));
    sc_keys_kernel<<<m, 128, 0, st>>>(s->pa, 0);
    sc_keys_kernel<<<m, 128, 0, st>>>(s->pb, 0);
    sc_pair_kernel<<<(m + kScPairWarps - 1) / kScPairWarps, kScPairWarps * 32, 0, st>>>(s->pa, s->pb, nullptr, 1, nullptr, m, s->d_dist, s->d_shift);
    s->launches += 3;
    LSD_CUDA(cudaGetLastError());
    LSD_CUDA(cudaMemcpyAsync(dist + p0, s->d_dist, (size_t)m * 8, cudaMemcpyDeviceToHost, st));
    LSD_CUDA(cudaMemcpyAsync(shift + p0, s->d_shift, (size_t)m * 4, cudaMemcpyDeviceToHost, st));
    LSD_CUDA(cudaStreamSynchronize(st));
  }
  return LSD_OK;
}

// SCManager::detectClosestMatch for query `slot` of the last lsd_sc_make / lsd_sc_query (Scancontext.cpp:268-331)
lsd_status_t lsd_sc_detect_closest(lsd_sc_t* s, int slot, double dist_thres, int32_t* loop_id, float* yaw_rad, double* score) {
  if (!s || slot < 0 || slot >= s->q_n || !loop_id || !yaw_rad || !score) return LSD_ERR_INVALID;
  *loop_id = -1; *yaw_rad = 0.0f;
  if (s->db_n == 0) return LSD_OK;   // the reference returns before touching `score`
  std::vector<int32_t> idx((size_t)s->q_n * kCand), sh((size_t)s->q_n * kCand), nc(s->q_n);
  std::vector<double> d((size_t)s->q_n * kCand);
  lsd_status_t e = lsd_sc_query(s, nullptr, s->q_n, idx.data(), d.data(), sh.data(), nc.data());
  if (e) return e;
  double min_dist = kBig; int align = 0, nn = 0;
  for (int c = 0; c < nc[slot]; c++) {
    const size_t at = (size_t)slot * kCand + c;
    if (d[at] < min_dist) { min_dist = d[at]; align = sh[at]; nn = idx[at]; }
  }
  *score = min_dist;
  if (min_dist < dist_thres) *loop_id = nn;
  *yaw_rad = shift_to_yaw(align);
  return LSD_OK;
}

// SCManager::detectCandidateMatch (Scancontext.cpp:333-367): candidates below the threshold, in candidate order
lsd_status_t lsd_sc_detect_candidates(lsd_sc_t* s, int slot, double dist_thres, int32_t* idx10, float* yaw10, float* dist10, int32_t* n) {
  if (!s || slot < 0 || slot >= s->q_n || !idx10 || !yaw10 || !dist10 || !n) return LSD_ERR_INVALID;
  *n = 0;
  if (s->db_n == 0) return LSD_OK;
  std::vector<int32_t> idx((size_t)s->q_n * kCand), sh((size_t)s->q_n * kCand), nc(s->q_n);
  std::vector<double> d((size_t)s->q_n * kCand);
  lsd_status_t e = lsd_sc_query(s, nullptr, s->q_n, idx.data(), d.data(), sh.data(), nc.data());
  if (e) return e;
  for (int c = 0; c < nc[slot]; c++) {
    const size_t at = (size_t)slot * kCand + c;
    if (d[at] < dist_thres) { idx10[*n] = idx[at]; yaw10[*n] = shift_to_yaw(sh[at]); dist10[*n] = (float)d[at]; (*n)++; }
  }
  return LSD_OK;
}

}  // extern "C"
